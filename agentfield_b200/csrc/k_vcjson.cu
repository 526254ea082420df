// Credential documents in any JSON spelling verified on the device (afc_vc_verify_json_batch, include/afcrypto.h).
//
// Reference call sites replaced (relative to AgentField's control-plane/):
//   k_vcj_parse / k_vcj_emit   json.Unmarshal + json.Marshal with a zero Proof   internal/services/vc_service.go:250-251, 469-476
//                                                                                 internal/handlers/did_handlers.go:97-111 (request bodies)
//                                                                                 internal/cli/vc.go:159 (af vc verify on a file)
//                              ResolveDID of the issuer                          internal/services/vc_service.go:259
//                              base64.RawURLEncoding.DecodeString(proofValue)    internal/services/vc_service.go:498
//   (then the scan, the keyed verify of k_ed25519.cu and k_vc_fold, unchanged)
//
// k_vcj_parse: one document per thread through the tolerant walk of afc_vcjson.cuh with a ByteCounter: status so far, the length of
// the canonical signing message, decoded signature, key index and field spans, in the layout k_vc_parse writes.  After the scan,
// k_vcj_emit walks each candidate again with a ByteWriter, stops at "proof": and appends the zero-proof text.  The schema (ops,
// literal pool and whitespace masks, 1.8 KB) is staged in shared memory, as k_vc_parse stages its own.
#include "afc_launch.h"
#include "afc_vcjson.cuh"

namespace afc {

static constexpr int VCJ_THREADS = 128;

// vc_stage_schema of k_vcdoc.cu for the larger VcjSchema: a deliberate copy, so that the existing kernels' machine code stays exactly
// as it was (a shared template would recompile them)
__device__ __forceinline__ void vcj_stage_schema(VcjSchema& S, const VcjSchema* __restrict__ g) {
    const uint32_t* src = (const uint32_t*)g;
    uint32_t* dst = (uint32_t*)&S;
    for (uint32_t k = threadIdx.x; k < sizeof(VcjSchema) / 4; k += blockDim.x) dst[k] = __ldg(src + k);
    __syncthreads();
}

// Both kernels take a register budget instead of launch bounds: under __launch_bounds__(VCJ_THREADS) ptxas holds them to 48 registers
// and spills.
__global__ void __maxnreg__(64)
k_vcj_parse(const VcjSchema* __restrict__ schema, const uint8_t* __restrict__ docs, const uint64_t* __restrict__ doc_off, uint32_t n,
            const uint8_t* __restrict__ dids, const uint32_t* __restrict__ did_off, const uint32_t* __restrict__ slots, uint32_t slot_mask,
            uint8_t* __restrict__ status, uint64_t* __restrict__ len_out, uint32_t* __restrict__ sigs, uint32_t* __restrict__ key_index,
            uint32_t* __restrict__ fields) {
    __shared__ VcjSchema S;
    vcj_stage_schema(S, schema);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t o0 = doc_off[i];
    const uint8_t* d = docs + o0;
    const uint64_t len = doc_off[i + 1] - o0;
    VcjParse r;
    ByteCounter c; c.init();
    vcj_walk<true>(S, d, len, c, r);
    uint32_t st = VC_HOST, key = 0;
    if (r.ok) {
        key = vcj_resolve(d + r.iss_off, r.iss_len, dids, did_off, slots, slot_mask);
        st = key == 0xffffffffu ? VC_UNRESOLVED : vc_b64_signature(d + r.pv_off, r.pv_len, sigs + (size_t)i * 16);
    }
    const bool cand = st == VC_VALID;              // verified next; the fold turns it into VALID / INVALID
    status[i] = (uint8_t)st;
    len_out[i] = cand ? (uint64_t)r.prefix + S.s.tail_len : 0;
    key_index[i] = cand ? key : 0;
    if (!cand) { uint4* z = (uint4*)(sigs + (size_t)i * 16); const uint4 zero = {0, 0, 0, 0}; z[0] = zero; z[1] = zero; z[2] = zero; z[3] = zero; }
    if (fields) {
        uint4 f = {0, 0, 0, 0};
        if (r.ok) f = make_uint4(r.iss_off, r.iss_len, r.date_off, r.date_len);
        ((uint4*)fields)[i] = f;
    }
}

__global__ void __maxnreg__(64)
k_vcj_emit(const VcjSchema* __restrict__ schema, const uint8_t* __restrict__ docs, const uint64_t* __restrict__ doc_off, uint32_t n,
           const uint64_t* __restrict__ msg_off, uint8_t* __restrict__ msgs) {
    __shared__ VcjSchema S;
    vcj_stage_schema(S, schema);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t m0 = msg_off[i], mlen = msg_off[i + 1] - m0;
    if (mlen == 0) return;
    const uint64_t o0 = doc_off[i];
    ByteWriter w; w.init(msgs + m0);
    VcjParse r;
    vcj_walk<false>(S, docs + o0, doc_off[i + 1] - o0, w, r);
    vcj_put_lit(w, S.s.pool, S.s.tail_off, S.s.tail_len);
    w.finish();
}

namespace launch {

static inline uint32_t vcj_blocks(uint64_t n, uint32_t t) { return (uint32_t)((n + t - 1) / t); }

cudaError_t vcj_parse(const void* schema, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, const uint8_t* dids, const uint32_t* did_off,
                      const uint32_t* slots, uint32_t slot_mask, uint8_t* status, uint64_t* len_out, uint8_t* sigs, uint32_t* key_index,
                      uint32_t* fields, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vcj_parse", s, k_vcj_parse<<<vcj_blocks(n, VCJ_THREADS), VCJ_THREADS, 0, s>>>((const VcjSchema*)schema, docs, doc_off, n, dids,
                                                                                                     did_off, slots, slot_mask, status, len_out,
                                                                                                     (uint32_t*)sigs, key_index, fields));
    return cudaGetLastError();
}
cudaError_t vcj_emit(const void* schema, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, const uint64_t* msg_off, uint8_t* msgs,
                     cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vcj_emit", s, k_vcj_emit<<<vcj_blocks(n, VCJ_THREADS), VCJ_THREADS, 0, s>>>((const VcjSchema*)schema, docs, doc_off, n, msg_off, msgs));
    return cudaGetLastError();
}
size_t vcj_schema_bytes() { return sizeof(VcjSchema); }
#if !AFC_DEVICE_CODE
int vcj_schema_host(int kind, void* out) { return vcj_schema_build(kind, (VcjSchema*)out); }
#endif

}  // namespace launch
}  // namespace afc
