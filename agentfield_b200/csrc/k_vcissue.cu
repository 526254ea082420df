// Execution credentials issued on the device (afc_vc_issue_execution_batch, include/afcrypto.h; afc_vcissue.cuh).
//
// Reference call sites replaced (relative to /root/reference/control-plane):
//   k_vci_hashdata           hashData(marshalDataOrNull(input / output))   internal/services/vc_service.go:146-147, 508-515, 1297-1306
//   k_vci_sizes / k_vci_fill createVCDocument + json.Marshal               internal/services/vc_service.go:374-431, 436-439
//                            json.Marshal(vcDoc) of the stored document    internal/services/vc_service.go:201
//   (then the expanded-key signing of k_ed25519.cu, unchanged)             internal/services/vc_service.go:460-463
//   k_vci_proof              base64.RawURLEncoding.EncodeToString(sig)     internal/services/vc_service.go:465
//
// One payload (k_vci_hashdata) or one credential (the others) per thread.  k_vci_sizes writes both lengths of each credential —
// the signing message and the stored document — and the existing scan turns them into offsets; k_vci_fill then writes both
// in one walk over the columns.  The program (constant text and column map, ~0.8 KB) is a kernel parameter staged in shared
// memory, as the stored-document schema is in k_vcdoc.cu.
#include "afc_launch.h"
#include "afc_vcissue.cuh"

namespace afc {

static constexpr int VCI_THREADS = 128;

__device__ __forceinline__ void vci_stage(VciProgram& S, const VciProgram& g) {
    const uint32_t* src = (const uint32_t*)&g;
    uint32_t* dst = (uint32_t*)&S;
    for (uint32_t k = threadIdx.x; k < sizeof(VciProgram) / 4; k += blockDim.x) dst[k] = src[k];
    __syncthreads();
}

__device__ __forceinline__ VciItem vci_item(const uint8_t* cols, const uint64_t* col_off, const int64_t* duration, const uint8_t* hashes,
                                           uint32_t i) {
    VciItem it;
    it.cols = cols; it.coff = col_off + (size_t)i * VCI_COLUMNS; it.duration = duration[i];
    it.hashes = hashes ? hashes + (size_t)i * 2 * VCI_HASH_CHARS : nullptr;
    return it;
}

// payload j of 2n (input i = 2i, output i = 2i + 1): 43 characters at hashes + 43 j
__global__ void __launch_bounds__(VCI_THREADS)
k_vci_hashdata(const uint8_t* __restrict__ payloads, const uint64_t* __restrict__ payload_off, const uint8_t* __restrict__ nil, uint32_t m,
               uint8_t* __restrict__ hashes) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint64_t o0 = payload_off[j];
    vci_hashdata_one(payloads + o0, payload_off[j + 1] - o0, nil[j] != 0, hashes + (size_t)j * VCI_HASH_CHARS);
}

__global__ void __launch_bounds__(VCI_THREADS)
k_vci_sizes(const __grid_constant__ VciProgram prog, const uint8_t* __restrict__ cols, const uint64_t* __restrict__ col_off,
            const int64_t* __restrict__ duration, const uint8_t* __restrict__ hashes, uint32_t n, uint64_t* __restrict__ msg_len,
            uint64_t* __restrict__ doc_len) {
    __shared__ VciProgram S;
    vci_stage(S, prog);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t ml, dl;
    vci_doc_sizes(S, vci_item(cols, col_off, duration, hashes, i), &ml, &dl);
    msg_len[i] = ml;
    doc_len[i] = dl;
}

__global__ void __launch_bounds__(VCI_THREADS)
k_vci_fill(const __grid_constant__ VciProgram prog, const uint8_t* __restrict__ cols, const uint64_t* __restrict__ col_off,
           const int64_t* __restrict__ duration, const uint8_t* __restrict__ hashes, uint32_t n, const uint64_t* __restrict__ msg_off,
           uint8_t* __restrict__ msgs, const uint64_t* __restrict__ doc_off, uint8_t* __restrict__ docs) {
    __shared__ VciProgram S;
    vci_stage(S, prog);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    vci_doc_fill(S, vci_item(cols, col_off, duration, hashes, i), msgs + msg_off[i], docs + doc_off[i]);
}

// the 86 proofValue characters: into the stored document (they end 3 bytes before it does: "}}) and into proof_values
__global__ void __launch_bounds__(VCI_THREADS)
k_vci_proof(const uint8_t* __restrict__ sigs, uint32_t n, const uint64_t* __restrict__ doc_off, uint8_t* __restrict__ docs,
            uint8_t* __restrict__ proof_values) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint4* s = (const uint4*)(sigs + (size_t)i * 64);
    uint32_t w[16];
#pragma unroll
    for (int q = 0; q < 4; q++) { const uint4 v = s[q]; w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w; }
    vci_proof_one(w, docs + doc_off[i + 1] - 3 - VCI_PV_CHARS, proof_values + (size_t)i * VCI_PV_CHARS);
}

namespace launch {

static inline uint32_t vci_blocks(uint64_t n) { return (uint32_t)((n + VCI_THREADS - 1) / VCI_THREADS); }
static const VciProgram& vci_program() {
    static const VciProgram P = [] { VciProgram p; vci_program_build(&p); return p; }();
    return P;
}

cudaError_t vci_hashdata(const uint8_t* payloads, const uint64_t* payload_off, const uint8_t* nil, uint32_t m, uint8_t* hashes, cudaStream_t s,
                         LaunchLog* lg) {
    if (m == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vci_hashdata", s, k_vci_hashdata<<<vci_blocks(m), VCI_THREADS, 0, s>>>(payloads, payload_off, nil, m, hashes));
    return cudaGetLastError();
}
cudaError_t vci_sizes(const uint8_t* cols, const uint64_t* col_off, const int64_t* duration, const uint8_t* hashes, uint32_t n, uint64_t* msg_len,
                      uint64_t* doc_len, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vci_sizes", s, k_vci_sizes<<<vci_blocks(n), VCI_THREADS, 0, s>>>(vci_program(), cols, col_off, duration, hashes, n, msg_len,
                                                                                      doc_len));
    return cudaGetLastError();
}
cudaError_t vci_fill(const uint8_t* cols, const uint64_t* col_off, const int64_t* duration, const uint8_t* hashes, uint32_t n, const uint64_t* msg_off,
                     uint8_t* msgs, const uint64_t* doc_off, uint8_t* docs, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vci_fill", s, k_vci_fill<<<vci_blocks(n), VCI_THREADS, 0, s>>>(vci_program(), cols, col_off, duration, hashes, n, msg_off, msgs,
                                                                                    doc_off, docs));
    return cudaGetLastError();
}
cudaError_t vci_proof(const uint8_t* sigs, uint32_t n, const uint64_t* doc_off, uint8_t* docs, uint8_t* proof_values, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vci_proof", s, k_vci_proof<<<vci_blocks(n), VCI_THREADS, 0, s>>>(sigs, n, doc_off, docs, proof_values));
    return cudaGetLastError();
}
uint64_t vci_literal_bytes() {
    static const uint64_t text = [] { VciProgram p; return (uint64_t)vci_program_build(&p); }();
    return text;
}

}  // namespace launch
}  // namespace afc
