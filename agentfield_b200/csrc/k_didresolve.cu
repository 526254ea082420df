// DIDs resolved and DID documents served on the device (afc_did_resolve_batch, include/afcrypto.h; afc_didresolve.cuh).
//
// Reference call sites replaced (relative to the reference's control-plane/):
//   k_dres_probe               ResolveDID's scan of the registry (a directory probe)   internal/services/did_service.go:368-473
//   k_dres_probe / k_dres_emit the handlers' c.JSON, json.Unmarshal of the stored JWK  internal/handlers/did_handlers.go:73-94, 368-429
//
// At attach (afc_did_directory_set_identities) k_dres_entries runs one thread per directory entry: both body lengths, or 0 for HOST, the
// directory's largest body, and the length of the canonical JWK text when the stored one is not canonical; the existing scan turns those
// into offsets and k_dres_canon writes the canonical texts, so that no request re-marshals a JWK.  Per call, k_dres_probe runs one thread
// per request (the probe, the state, the body length from the entry's cached lengths, or the escaped length of the request for a 404
// document), the existing scan lays the bodies out and k_dres_emit writes each one from the directory's columns through ByteWriter.
#include "afc_didresolve.cuh"
#include "afc_launch.h"

namespace afc {

static constexpr int DRES_THREADS = 128;

__device__ __forceinline__ DresStr dres_span(const uint8_t* base, uint64_t a, uint64_t b) {
    DresStr s; s.p = base + a; s.len = b - a;
    return s;
}
__device__ __forceinline__ DresStr dres_did(const launch::DresDir& D, uint32_t k) { return dres_span(D.dids, D.did_off[k], D.did_off[k + 1]); }
__device__ __forceinline__ DresStr dres_col(const launch::DresDir& D, uint32_t k, uint32_t c) {
    return dres_span(D.icols, D.icol_off[DRES_COLUMNS * k + c], D.icol_off[DRES_COLUMNS * k + c + 1]);
}
// entry k's jv_emit tape: icol_off[3 k + 2] / 2 + k leaves each entry jwk.len / 2 + 1 entries before the next one's
__device__ __forceinline__ uint32_t* dres_tape(const launch::DresDir& D, uint32_t* tape, uint32_t k) {
    return tape + D.icol_off[DRES_COLUMNS * k + DRES_COL_JWK] / 2 + k;
}

// at 48 registers (what ptxas picks under __launch_bounds__(128)) the jv_emit walk spills; attach runs once per directory
__global__ void __maxnreg__(96)
k_dres_entries(const launch::DresDir D, uint32_t* __restrict__ tape, uint32_t* __restrict__ largest) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= D.n) return;
    const DresEntry e = dres_entry(D.kind[k], dres_did(D, k), dres_col(D, k, DRES_COL_PATH), dres_col(D, k, DRES_COL_FUNCTION),
                                   dres_col(D, k, DRES_COL_JWK), dres_tape(D, tape, k));
    D.rlen[k] = e.rlen;
    D.dlen[k] = e.dlen;
    D.side_off[k + 1] = e.side;
    atomicMax(largest, max(e.rlen, e.dlen));
}

__global__ void __launch_bounds__(DRES_THREADS)
k_dres_canon(const launch::DresDir D, uint32_t* __restrict__ tape) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= D.n || D.side_off[k + 1] == D.side_off[k]) return;
    const DresStr jwk = dres_col(D, k, DRES_COL_JWK);
    ByteWriter w; w.init(D.side + D.side_off[k]);
    jv_emit(w, jwk.p, (uint32_t)jwk.len, dres_tape(D, tape, k));
    w.finish();
}

__global__ void __launch_bounds__(DRES_THREADS)
k_dres_ends(const uint64_t* __restrict__ req_off, uint32_t n, unsigned long long* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) { out[0] = req_off[0]; out[1] = req_off[n]; }
    if (i >= n) return;
    const uint64_t a = req_off[i], b = req_off[i + 1];
    const unsigned long long f = (b < a ? 1ull : 0ull) | (b >= a && b - a > DRES_REQ_MAX ? 2ull : 0ull);
    if (f) atomicOr(out + 2, f);
}

__global__ void __launch_bounds__(DRES_THREADS)
k_dres_probe(const launch::DresDir D, const uint8_t* __restrict__ kinds, const uint8_t* __restrict__ reqs, const uint64_t* __restrict__ req_off,
             uint32_t n, uint8_t* __restrict__ state, uint32_t* __restrict__ ent, uint64_t* __restrict__ body_off) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t kind = kinds[i];
    const DresStr req = dres_span(reqs, req_off[i], req_off[i + 1]);
    uint32_t st, k = 0xffffffffu;
    uint64_t len;
    if (kind > DRES_DOCUMENT) {
        st = DRES_HOST; len = 0;
    } else if (req.len == 0) {
        st = DRES_BAD_REQUEST; len = DRES_BAD_REQUEST_LEN;
    } else {
        k = vcj_resolve(req.p, (uint32_t)req.len, D.dids, D.did_off, D.slots, D.mask);
        if (k == 0xffffffffu) {
            ByteCounter c; c.init();
            dres_not_found(c, kind, req);
            st = DRES_NOT_FOUND; len = c.n;
        } else {
            len = kind == DRES_RESOLVE ? D.rlen[k] : D.dlen[k];
            st = len ? DRES_FOUND : DRES_HOST;
        }
    }
    state[i] = (uint8_t)st;
    ent[i] = k;
    body_off[i + 1] = len;
}

__global__ void __launch_bounds__(DRES_THREADS)
k_dres_emit(const launch::DresDir D, const uint8_t* __restrict__ kinds, const uint8_t* __restrict__ reqs, const uint64_t* __restrict__ req_off,
            uint32_t n, const uint8_t* __restrict__ state, const uint32_t* __restrict__ ent, const uint64_t* __restrict__ body_off,
            uint8_t* __restrict__ bodies) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t st = state[i], kind = kinds[i];
    if (st == DRES_HOST) return;
    ByteWriter w; w.init(bodies + body_off[i]);
    if (st == DRES_BAD_REQUEST) {
        vci_put_text(w, DRES_BAD_REQUEST_BODY);
    } else if (st == DRES_NOT_FOUND) {
        dres_not_found(w, kind, dres_span(reqs, req_off[i], req_off[i + 1]));
    } else {
        const uint32_t k = ent[i];
        if (kind == DRES_RESOLVE) {
            dres_resolve(w, D.kind[k], dres_did(D, k), dres_col(D, k, DRES_COL_PATH), dres_col(D, k, DRES_COL_FUNCTION), dres_col(D, k, DRES_COL_JWK));
        } else {
            const uint64_t s0 = D.side_off[k], s1 = D.side_off[k + 1];
            dres_document(w, dres_did(D, k), s1 > s0 ? dres_span(D.side, s0, s1) : dres_col(D, k, DRES_COL_JWK));
        }
    }
    w.finish();
}

namespace launch {

static inline uint32_t dres_blocks(uint64_t n) { return (uint32_t)((n + DRES_THREADS - 1) / DRES_THREADS); }

cudaError_t dres_entries(const DresDir& D, uint32_t* tape, uint32_t* largest, cudaStream_t s, LaunchLog* lg) {
    if (D.n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_dres_entries", s, k_dres_entries<<<dres_blocks(D.n), DRES_THREADS, 0, s>>>(D, tape, largest));
    return cudaGetLastError();
}
cudaError_t dres_canon(const DresDir& D, uint32_t* tape, cudaStream_t s, LaunchLog* lg) {
    if (D.n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_dres_canon", s, k_dres_canon<<<dres_blocks(D.n), DRES_THREADS, 0, s>>>(D, tape));
    return cudaGetLastError();
}
cudaError_t dres_ends(const uint64_t* req_off, uint32_t n, uint64_t* out, cudaStream_t s, LaunchLog* lg) {
    AFC_LAUNCH(lg, "k_dres_ends", s, k_dres_ends<<<dres_blocks(n > 0 ? n : 1), DRES_THREADS, 0, s>>>(req_off, n, (unsigned long long*)out));
    return cudaGetLastError();
}
cudaError_t dres_probe(const DresDir& D, const uint8_t* kinds, const uint8_t* reqs, const uint64_t* req_off, uint32_t n, uint8_t* state,
                       uint32_t* ent, uint64_t* body_off, uint64_t* scan, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_dres_probe", s, k_dres_probe<<<dres_blocks(n), DRES_THREADS, 0, s>>>(D, kinds, reqs, req_off, n, state, ent, body_off));
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    return offsets_from_lengths(body_off, n, scan, s, lg);
}
cudaError_t dres_emit(const DresDir& D, const uint8_t* kinds, const uint8_t* reqs, const uint64_t* req_off, uint32_t n, const uint8_t* state,
                      const uint32_t* ent, const uint64_t* body_off, uint8_t* bodies, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_dres_emit", s, k_dres_emit<<<dres_blocks(n), DRES_THREADS, 0, s>>>(D, kinds, reqs, req_off, n, state, ent, body_off, bodies));
    return cudaGetLastError();
}
uint64_t dres_request_fixed() { return DRES_DOC404_FIXED; }

}  // namespace launch
}  // namespace afc
