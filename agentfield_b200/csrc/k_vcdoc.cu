// Stored credential documents verified on the device (afc_vc_verify_stored_batch, include/afcrypto.h).
//
// Reference call sites replaced (relative to /root/reference/control-plane):
//   k_vc_parse / k_vc_emit   json.Unmarshal + json.Marshal with a zero Proof   internal/services/vc_service.go:250-251, 469-476
//                                                                               internal/services/vc_service.go:1589-1597
//                                                                               internal/cli/vc_verification_enhanced.go:418-454
//                            ResolveDID of the issuer                          internal/services/vc_service.go:259
//                            base64.RawURLEncoding.DecodeString(proofValue)    internal/services/vc_service.go:498
//   (then the keyed verify of k_ed25519.cu, unchanged, and k_vc_fold)
//
// k_vc_parse: one document per thread through the schema (afc_vcdoc.cuh); the schema — ops and literal pool, 1.3 KB — is staged
// in shared memory, where the divergent literal positions of a warp's 32 documents cost bank conflicts at worst, not the
// serialisation constant memory imposes on different addresses.  Writes the status so far, the signing-message length, the
// decoded signature, the key index and the field spans.  After the scan, k_vc_emit copies D[0:p] and appends the zero-proof text
// (32-byte sector stores through ByteWriter).
//
// The audit (afc_vc_audit_stored_batch) runs k_vc_parse_capture, the same walk that also records the spans of the members the
// ExecutionVC record's columns are compared with and what @context / type hold, then k_vc_crosscheck (record columns against those
// spans, status, timestamp, structure and compliance rules: VerifyExecutionVCComprehensive, internal/services/vc_service.go:926-1005,
// 1008-1359), then the same scan / emit / keyed verify / fold.
#include "afc_launch.h"
#include "afc_vcdoc.cuh"

namespace afc {

static constexpr int VC_THREADS = 128;

__device__ __forceinline__ void vc_stage_schema(VcSchema& S, const VcSchema* __restrict__ g) {
    const uint32_t* src = (const uint32_t*)g;
    uint32_t* dst = (uint32_t*)&S;
    for (uint32_t k = threadIdx.x; k < sizeof(VcSchema) / 4; k += blockDim.x) dst[k] = __ldg(src + k);
    __syncthreads();
}

// One document of k_vc_parse; with CAPTURE also its audit capture (caps: VC_CAP_WORDS words per document)
template <bool CAPTURE>
__device__ __forceinline__ void vc_parse_one(const VcSchema& S, const uint8_t* __restrict__ docs, const uint64_t* __restrict__ doc_off, uint32_t i,
                                             const uint8_t* __restrict__ dids, const uint32_t* __restrict__ did_off, const uint32_t* __restrict__ slots,
                                             uint32_t slot_mask, uint8_t* __restrict__ status, uint64_t* __restrict__ len_out, uint32_t* __restrict__ sigs,
                                             uint32_t* __restrict__ key_index, uint32_t* __restrict__ fields, uint32_t* __restrict__ caps) {
    const uint64_t o0 = doc_off[i];
    const uint8_t* d = docs + o0;
    const uint64_t len = doc_off[i + 1] - o0;
    VcParse r;
    vc_parse_doc_t<CAPTURE>(S, d, len, r, CAPTURE ? caps + (size_t)i * VC_CAP_WORDS : nullptr);
    uint32_t st = VC_HOST, key = 0;
    if (r.ok) {
        // resolve the issuer: hash of its bytes, probe, confirm byte for byte
        ByteWindow w; w.init(d + r.iss_off, r.iss_len);
        uint32_t h = 2166136261u;
        while (w.rem) { w.fill(); h = vc_did_hash_byte(h, w.peek(0)); w.skip(1); }
        st = VC_UNRESOLVED;
        for (uint32_t s = h & slot_mask;; s = (s + 1) & slot_mask) {
            const uint32_t k = slots[s];
            if (k == 0xffffffffu) break;
            const uint32_t k0 = did_off[k], kl = did_off[k + 1] - k0;
            if (kl != r.iss_len) continue;
            uint32_t j = 0;
            while (j < kl && dids[k0 + j] == d[r.iss_off + j]) ++j;
            if (j == kl) { st = VC_VALID; key = k; break; }
        }
        if (st == VC_VALID) st = vc_b64_signature(d + r.pv_off, r.pv_len, sigs + (size_t)i * 16);
    }
    const bool cand = st == VC_VALID;              // verified next; the fold turns it into VALID / INVALID
    status[i] = (uint8_t)st;
    len_out[i] = cand ? (uint64_t)r.proof_at + S.tail_len : 0;
    key_index[i] = cand ? key : 0;
    if (!cand) { uint4* z = (uint4*)(sigs + (size_t)i * 16); const uint4 zero = {0, 0, 0, 0}; z[0] = zero; z[1] = zero; z[2] = zero; z[3] = zero; }
    if (fields) {
        uint4 f = {0, 0, 0, 0};
        if (r.ok) f = make_uint4(r.iss_off, r.iss_len, r.date_off, r.date_len);
        ((uint4*)fields)[i] = f;
    }
}

__global__ void __launch_bounds__(VC_THREADS)
k_vc_parse(const VcSchema* __restrict__ schema, const uint8_t* __restrict__ docs, const uint64_t* __restrict__ doc_off, uint32_t n,
           const uint8_t* __restrict__ dids, const uint32_t* __restrict__ did_off, const uint32_t* __restrict__ slots, uint32_t slot_mask,
           uint8_t* __restrict__ status, uint64_t* __restrict__ len_out, uint32_t* __restrict__ sigs, uint32_t* __restrict__ key_index,
           uint32_t* __restrict__ fields) {
    __shared__ VcSchema S;
    vc_stage_schema(S, schema);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    vc_parse_one<false>(S, docs, doc_off, i, dids, did_off, slots, slot_mask, status, len_out, sigs, key_index, fields, nullptr);
}

// k_vc_parse that also writes each document's audit capture (afc_vc_audit_stored_batch).  This kernel and k_vc_crosscheck take a
// register budget instead of launch bounds: under __launch_bounds__(VC_THREADS) ptxas holds them to 40 registers and spills.
__global__ void __maxnreg__(64)
k_vc_parse_capture(const VcSchema* __restrict__ schema, const uint8_t* __restrict__ docs, const uint64_t* __restrict__ doc_off, uint32_t n,
                   const uint8_t* __restrict__ dids, const uint32_t* __restrict__ did_off, const uint32_t* __restrict__ slots, uint32_t slot_mask,
                   uint8_t* __restrict__ status, uint64_t* __restrict__ len_out, uint32_t* __restrict__ sigs, uint32_t* __restrict__ key_index,
                   uint32_t* __restrict__ caps) {
    __shared__ VcSchema S;
    vc_stage_schema(S, schema);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    vc_parse_one<true>(S, docs, doc_off, i, dids, did_off, slots, slot_mask, status, len_out, sigs, key_index, nullptr, caps);
}

// The record's columns against the captured document: one credential per thread, a uint32 issue mask (0 for HOST documents, which
// the caller audits itself).  col_off: AFC_AUDIT_COLUMNS per record + 1, absolute offsets into cols (nullptr for workflow documents).
__global__ void __maxnreg__(64)
k_vc_crosscheck(int kind, const uint8_t* __restrict__ docs, const uint64_t* __restrict__ doc_off, uint32_t n, const uint32_t* __restrict__ caps,
                const uint8_t* __restrict__ status, const uint8_t* __restrict__ cols, const uint64_t* __restrict__ col_off,
                uint32_t* __restrict__ issues) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (status[i] == VC_HOST) { issues[i] = 0; return; }
    issues[i] = vc_audit_mask(kind, docs + doc_off[i], caps + (size_t)i * VC_CAP_WORDS, cols, col_off ? col_off + (size_t)i * VC_AUDIT_COLUMNS : nullptr);
}

__global__ void __launch_bounds__(VC_THREADS)
k_vc_emit(const VcSchema* __restrict__ schema, const uint8_t* __restrict__ docs, const uint64_t* __restrict__ doc_off, uint32_t n,
          const uint64_t* __restrict__ msg_off, uint8_t* __restrict__ msgs) {
    __shared__ VcSchema S;
    vc_stage_schema(S, schema);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t m0 = msg_off[i], mlen = msg_off[i + 1] - m0;
    if (mlen == 0) return;
    ByteWriter w; w.init(msgs + m0);
    json_copy_raw(w, docs + doc_off[i], mlen - S.tail_len);
    const uint32_t* t = S.pool + (S.tail_off >> 2);
    uint32_t k = 0;
    for (; k + 4 <= S.tail_len; k += 4) w.put4(t[k >> 2]);
    for (; k < S.tail_len; k++) w.put((t[k >> 2] >> (8 * (k & 3))) & 0xffu);
    w.finish();
}

__global__ void __launch_bounds__(256)
k_vc_fold(uint8_t* __restrict__ status, const uint8_t* __restrict__ ok, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (status[i] == VC_VALID) status[i] = ok[i] ? VC_VALID : VC_INVALID;
}

namespace launch {

static inline uint32_t vc_blocks(uint64_t n, uint32_t t) { return (uint32_t)((n + t - 1) / t); }

cudaError_t vc_parse(const void* schema, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, const uint8_t* dids, const uint32_t* did_off,
                     const uint32_t* slots, uint32_t slot_mask, uint8_t* status, uint64_t* len_out, uint8_t* sigs, uint32_t* key_index,
                     uint32_t* fields, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vc_parse", s, k_vc_parse<<<vc_blocks(n, VC_THREADS), VC_THREADS, 0, s>>>((const VcSchema*)schema, docs, doc_off, n, dids, did_off,
                                                                                              slots, slot_mask, status, len_out, (uint32_t*)sigs, key_index, fields));
    return cudaGetLastError();
}
cudaError_t vc_parse_capture(const void* schema, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, const uint8_t* dids, const uint32_t* did_off,
                             const uint32_t* slots, uint32_t slot_mask, uint8_t* status, uint64_t* len_out, uint8_t* sigs, uint32_t* key_index,
                             uint32_t* caps, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vc_parse_capture", s, k_vc_parse_capture<<<vc_blocks(n, VC_THREADS), VC_THREADS, 0, s>>>((const VcSchema*)schema, docs, doc_off, n,
                                                                                                              dids, did_off, slots, slot_mask, status, len_out,
                                                                                                              (uint32_t*)sigs, key_index, caps));
    return cudaGetLastError();
}
cudaError_t vc_crosscheck(int kind, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, const uint32_t* caps, const uint8_t* status,
                          const uint8_t* cols, const uint64_t* col_off, uint32_t* issues, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vc_crosscheck", s, k_vc_crosscheck<<<vc_blocks(n, VC_THREADS), VC_THREADS, 0, s>>>(kind, docs, doc_off, n, caps, status, cols,
                                                                                                        col_off, issues));
    return cudaGetLastError();
}
size_t vc_capture_bytes(uint32_t n) { return (size_t)n * VC_CAP_WORDS * 4; }
cudaError_t vc_emit(const void* schema, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, const uint64_t* msg_off, uint8_t* msgs,
                    cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vc_emit", s, k_vc_emit<<<vc_blocks(n, VC_THREADS), VC_THREADS, 0, s>>>((const VcSchema*)schema, docs, doc_off, n, msg_off, msgs));
    return cudaGetLastError();
}
cudaError_t vc_fold(uint8_t* status, const uint8_t* ok, uint32_t n, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vc_fold", s, k_vc_fold<<<vc_blocks(n, 256), 256, 0, s>>>(status, ok, n));
    return cudaGetLastError();
}
size_t vc_schema_bytes() { return sizeof(VcSchema); }
#if !AFC_DEVICE_CODE
int vc_schema_host(int kind, void* out) { return vc_schema_build(kind, (VcSchema*)out); }
#endif

}  // namespace launch
}  // namespace afc
