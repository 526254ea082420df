// VC verification requests answered on the device (afc_vc_verify_request_batch, include/afcrypto.h; afc_vcreq.cuh).
//
// Reference call sites replaced (relative to the reference's control-plane/):
//   k_vrq_bind               c.ShouldBindJSON(&types.VCVerificationRequest)   internal/handlers/did_handlers.go:99, ui/did.go:444
//   (vc_stored_enqueue)      VCService.VerifyVC on the vc_document bytes      internal/services/vc_service.go:242-289
//   k_vrq_sizes / k_vrq_emit c.JSON(status, response)                         internal/handlers/did_handlers.go:100-110
//
// k_vrq_bind runs one request per thread: Go's scanner over the first value, its type, the span of the winning vc_document value and,
// for a null one, whether the key set holds the DID "".  The scan lays the object values out, k_vrq_gather copies them into one buffer
// (a warp per value), and the json-verify path of afc_vc_verify_json_batch runs on that buffer unchanged.  k_vrq_sizes writes each
// request's state and body length (re-walking the rare VC_BAD_ENCODING documents for proofValue's span, which `fields` does not carry),
// the scan lays the bodies out and k_vrq_emit writes them.
#include "afc_launch.h"
#include "afc_vcreq.cuh"

namespace afc {

static constexpr int VRQ_THREADS = 128;

// ptxas gives the scanner 32 registers under __launch_bounds__(VRQ_THREADS) and spills its state
__global__ void __maxnreg__(64)
k_vrq_bind(const uint8_t* __restrict__ reqs, const uint64_t* __restrict__ req_off, uint32_t n, const uint8_t* __restrict__ dids,
           const uint32_t* __restrict__ did_off, const uint32_t* __restrict__ slots, uint32_t slot_mask, uint8_t* __restrict__ bind,
           uint32_t* __restrict__ span, uint64_t* __restrict__ val_len) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t a = req_off[i];
    VrqBind b = vrq_bind(reqs + a, req_off[i + 1] - a);
    // ResolveDID("") of the zero VCDocument: not found unless the key set holds the empty DID, whose verify the host runs
    if (b.kind == VRB_NULL_DOC && vcj_resolve(reqs, 0, dids, did_off, slots, slot_mask) != 0xffffffffu) b.kind = VRB_HOST;
    bind[i] = (uint8_t)b.kind;
    span[i] = b.off;
    val_len[i] = b.len;
}

// a warp per request: its object value to docs + doc_off[i]
__global__ void __launch_bounds__(VRQ_THREADS)
k_vrq_gather(const uint8_t* __restrict__ reqs, const uint64_t* __restrict__ req_off, uint32_t n, const uint32_t* __restrict__ span,
             const uint64_t* __restrict__ doc_off, uint8_t* __restrict__ docs) {
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= n) return;
    const uint64_t d0 = doc_off[i], len = doc_off[i + 1] - d0;
    const uint8_t* src = reqs + req_off[i] + span[i];
    for (uint64_t k = lane; k < len; k += 32) docs[d0 + k] = src[k];
}

// at 48 registers (what ptxas picks under __launch_bounds__(128)) the vcj_walk of the rare VC_BAD_ENCODING documents spills
__global__ void __maxnreg__(64)
k_vrq_sizes(const VcjSchema* __restrict__ schema, const uint8_t* __restrict__ bind, const uint8_t* __restrict__ status,
            const uint32_t* __restrict__ fields, const uint8_t* __restrict__ docs, const uint64_t* __restrict__ doc_off, uint32_t n,
            uint32_t* __restrict__ b64_at, uint8_t* __restrict__ state, uint64_t* __restrict__ body_len) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t bk = bind[i], st = status[i];
    const uint8_t* doc = docs + doc_off[i];
    uint32_t at = 0;
    if (bk == VRB_OBJECT && st == VC_BAD_ENCODING) {
        VcjParse r;
        ByteCounter c; c.init();
        vcj_walk<true>(*schema, doc, doc_off[i + 1] - doc_off[i], c, r);
        at = vrq_b64_error_at(doc + r.pv_off, r.pv_len);
    }
    ByteCounter c; c.init();
    const uint32_t s = vrq_body(c, bk, st, doc, fields + 4 * (size_t)i, at);
    b64_at[i] = at;
    state[i] = (uint8_t)s;
    body_len[i] = c.n;
}

__global__ void __launch_bounds__(VRQ_THREADS)
k_vrq_emit(const uint8_t* __restrict__ bind, const uint8_t* __restrict__ status, const uint32_t* __restrict__ fields,
           const uint8_t* __restrict__ docs, const uint64_t* __restrict__ doc_off, uint32_t n, const uint32_t* __restrict__ b64_at,
           const uint64_t* __restrict__ body_off, uint8_t* __restrict__ bodies) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || body_off[i + 1] == body_off[i]) return;
    ByteWriter w; w.init(bodies + body_off[i]);
    vrq_body(w, bind[i], status[i], docs + doc_off[i], fields + 4 * (size_t)i, b64_at[i]);
    w.finish();
}

namespace launch {

static inline uint32_t vrq_blocks(uint64_t threads) { return (uint32_t)((threads + VRQ_THREADS - 1) / VRQ_THREADS); }

cudaError_t vrq_bind(const uint8_t* reqs, const uint64_t* req_off, uint32_t n, const uint8_t* dids, const uint32_t* did_off, const uint32_t* slots,
                     uint32_t slot_mask, uint8_t* bind, uint32_t* span, uint64_t* doc_off, uint64_t* scan, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vrq_bind", s, k_vrq_bind<<<vrq_blocks(n), VRQ_THREADS, 0, s>>>(reqs, req_off, n, dids, did_off, slots, slot_mask, bind, span,
                                                                                    doc_off + 1));
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    return offsets_from_lengths(doc_off, n, scan, s, lg);
}
cudaError_t vrq_gather(const uint8_t* reqs, const uint64_t* req_off, uint32_t n, const uint32_t* span, const uint64_t* doc_off, uint8_t* docs,
                       cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vrq_gather", s, k_vrq_gather<<<vrq_blocks(32ull * n), VRQ_THREADS, 0, s>>>(reqs, req_off, n, span, doc_off, docs));
    return cudaGetLastError();
}
cudaError_t vrq_sizes(const void* schema, const uint8_t* bind, const uint8_t* status, const uint32_t* fields, const uint8_t* docs,
                      const uint64_t* doc_off, uint32_t n, uint32_t* b64_at, uint8_t* state, uint64_t* body_off, uint64_t* scan, cudaStream_t s,
                      LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vrq_sizes", s, k_vrq_sizes<<<vrq_blocks(n), VRQ_THREADS, 0, s>>>((const VcjSchema*)schema, bind, status, fields, docs, doc_off, n,
                                                                                      b64_at, state, body_off + 1));
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    return offsets_from_lengths(body_off, n, scan, s, lg);
}
cudaError_t vrq_emit(const uint8_t* bind, const uint8_t* status, const uint32_t* fields, const uint8_t* docs, const uint64_t* doc_off, uint32_t n,
                     const uint32_t* b64_at, const uint64_t* body_off, uint8_t* bodies, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vrq_emit", s, k_vrq_emit<<<vrq_blocks(n), VRQ_THREADS, 0, s>>>(bind, status, fields, docs, doc_off, n, b64_at, body_off, bodies));
    return cudaGetLastError();
}
uint64_t vrq_request_fixed() { return VRQ_FIXED; }

}  // namespace launch
}  // namespace afc
