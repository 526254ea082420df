// Workflow credentials issued on the device (afc_vc_issue_workflow_batch, include/afcrypto.h; afc_vcworkflow.cuh).
//
// Reference call sites replaced (relative to /root/reference/control-plane):
//   k_vcw_records / k_vcw_sizes   determineWorkflowStatus, countCompletedSteps, the start / end loop   internal/services/vc_service.go:531-563, 721-787
//   k_vcw_sizes / k_vcw_fill / k_vcw_ids   createWorkflowVCDocument + json.Marshal                 internal/services/vc_service.go:635-693, 611
//   (then the expanded-key signing of k_ed25519.cu, unchanged)                                       internal/services/vc_service.go:686-718
//   k_vcw_proof                   base64.RawURLEncoding of the signature into the stored proof      internal/services/vc_service.go:596-611
//
// k_vcw_records runs one thread per record: its status class, the validity of its time and the length of its escaped id.  k_vcw_sizes
// runs one thread per workflow over its records and writes both lengths of its credential; the existing scan turns the workflows' and
// the records' lengths into offsets.  k_vcw_fill writes each workflow's text around its componentVcIds array and k_vcw_ids writes every
// record's id into it, one thread per record, so a workflow of 4096 records does not hold one thread for 4096 ids.  k_vcw_proof is
// k_vci_proof that skips VCW_HOST workflows (their documents are empty) and zeroes their proof values.
#include "afc_launch.h"
#include "afc_vcworkflow.cuh"

namespace afc {

// __launch_bounds__(VCW_THREADS, 1): without the minimum, ptxas aims at a register count that makes k_vcw_fill spill its two writers
static constexpr int VCW_THREADS = 128;

__device__ __forceinline__ void vcw_stage(VcwProgram& S, const VcwProgram& g) {
    const uint32_t* src = (const uint32_t*)&g;
    uint32_t* dst = (uint32_t*)&S;
    for (uint32_t k = threadIdx.x; k < sizeof(VcwProgram) / 4; k += blockDim.x) dst[k] = src[k];
    __syncthreads();
}

// Record j of the batch (absolute index rec_off[0] + j): class into cls[j], vcw_id_bytes into id_len[j]
__global__ void __launch_bounds__(VCW_THREADS, 1)
k_vcw_records(const uint8_t* __restrict__ rec_cols, const uint64_t* __restrict__ rec_col_off, const int64_t* __restrict__ created_at,
              const uint64_t* __restrict__ rec_off, uint32_t m, uint8_t* __restrict__ cls, uint64_t* __restrict__ id_len) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint64_t r = rec_off[0] + j;
    const uint64_t* co = rec_col_off + 2 * r;
    const uint64_t a = co[0], b = co[1], c = co[2];
    cls[j] = (uint8_t)vcw_record_class(rec_cols + b, c - b, created_at[2 * r], created_at[2 * r + 1]);
    id_len[j] = vcw_id_bytes(rec_cols + a, b - a);
}

__device__ __forceinline__ VcwItem vcw_item(const uint8_t* cols, const uint64_t* col_off, const int64_t* created_at, const uint64_t* rec_off,
                                            const uint32_t* summary, uint64_t ids_bytes, uint32_t i) {
    VcwItem it;
    it.cols = cols; it.coff = col_off + (size_t)i * VCW_COLUMNS;
    const uint64_t r = rec_off[i];
    it.cnt = (uint32_t)(rec_off[i + 1] - r);
    it.status = summary[4 * i];
    const uint32_t s = summary[4 * i + 2], e = summary[4 * i + 3];
    it.start_sec = s != VCW_NONE ? created_at[2 * (r + s)] : 0;
    it.has_end = e != VCW_NONE;
    it.end_sec = it.has_end ? created_at[2 * (r + e)] : 0;
    it.ids_bytes = ids_bytes;
    return it;
}

// Workflow i: its plan (summary, state), both lengths, and where its array starts and how long it is (arr[2 i], arr[2 i + 1])
__global__ void __launch_bounds__(VCW_THREADS, 1)
k_vcw_sizes(const __grid_constant__ VcwProgram prog, const uint8_t* __restrict__ cols, const uint64_t* __restrict__ col_off,
            const uint64_t* __restrict__ rec_off, const int64_t* __restrict__ created_at, const uint8_t* __restrict__ cls,
            const uint64_t* __restrict__ id_len, uint32_t n, uint64_t* __restrict__ msg_len, uint64_t* __restrict__ doc_len,
            uint64_t* __restrict__ arr, uint32_t* __restrict__ summary, uint8_t* __restrict__ state) {
    __shared__ VcwProgram S;
    vcw_stage(S, prog);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t a = rec_off[i] - rec_off[0];
    const VcwPlan p = vcw_reduce(cls + a, id_len + a, created_at + 2 * rec_off[i], (uint32_t)(rec_off[i + 1] - rec_off[i]));
    state[i] = (uint8_t)p.state;
    if (p.state == VCW_HOST) {
        summary[4 * (size_t)i] = 0; summary[4 * (size_t)i + 1] = 0; summary[4 * (size_t)i + 2] = 0; summary[4 * (size_t)i + 3] = 0;
        msg_len[i] = 0; doc_len[i] = 0; arr[2 * (size_t)i] = 0; arr[2 * (size_t)i + 1] = 0;
        return;
    }
    summary[4 * (size_t)i] = p.status; summary[4 * (size_t)i + 1] = p.completed; summary[4 * (size_t)i + 2] = p.start;
    summary[4 * (size_t)i + 3] = p.end;
    uint64_t ml, dl, at;
    vcw_doc_sizes(S, vcw_item(cols, col_off, created_at, rec_off, summary, p.ids_bytes, i), &ml, &dl, &at);
    msg_len[i] = ml; doc_len[i] = dl;
    arr[2 * (size_t)i] = at; arr[2 * (size_t)i + 1] = p.ids_bytes;
}

__global__ void __launch_bounds__(VCW_THREADS, 1)
k_vcw_fill(const __grid_constant__ VcwProgram prog, const uint8_t* __restrict__ cols, const uint64_t* __restrict__ col_off,
           const uint64_t* __restrict__ rec_off, const int64_t* __restrict__ created_at, const uint32_t* __restrict__ summary,
           const uint8_t* __restrict__ state, const uint64_t* __restrict__ arr, uint32_t n, const uint64_t* __restrict__ msg_off,
           uint8_t* __restrict__ msgs, const uint64_t* __restrict__ doc_off, uint8_t* __restrict__ docs) {
    __shared__ VcwProgram S;
    vcw_stage(S, prog);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || state[i] != VCW_BUILT) return;
    vcw_doc_fill(S, vcw_item(cols, col_off, created_at, rec_off, summary, arr[2 * (size_t)i + 1], i), arr[2 * (size_t)i], msgs + msg_off[i],
                 docs + doc_off[i]);
}

// Record j: its id into both forms of its workflow's credential.  id_off: the scanned vcw_id_bytes of the batch's records.
__global__ void __launch_bounds__(VCW_THREADS, 1)
k_vcw_ids(const uint8_t* __restrict__ rec_cols, const uint64_t* __restrict__ rec_col_off, const uint64_t* __restrict__ rec_off, uint32_t n,
          uint32_t m, const uint8_t* __restrict__ state, const uint64_t* __restrict__ arr, const uint64_t* __restrict__ id_off,
          const uint64_t* __restrict__ msg_off, uint8_t* __restrict__ msgs, const uint64_t* __restrict__ doc_off, uint8_t* __restrict__ docs) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint64_t r0 = rec_off[0], r = r0 + j;
    uint32_t lo = 0, hi = n;                                      // the last workflow i with rec_off[i] <= r (it holds r: r < rec_off[n])
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (rec_off[mid] <= r) lo = mid; else hi = mid;
    }
    const uint32_t i = lo;
    if (state[i] != VCW_BUILT) return;
    const uint64_t first = rec_off[i] - r0;
    const uint64_t at = arr[2 * (size_t)i] + vcw_id_at(id_off[j] - id_off[first], (uint32_t)(j - first));
    const uint64_t a = rec_col_off[2 * r], b = rec_col_off[2 * r + 1];
    vcw_put_id(rec_cols + a, b - a, (uint32_t)(j - first), msgs + msg_off[i] + at, docs + doc_off[i] + at);
}

// the 86 proofValue characters into each built document (they end 3 bytes before it does: "}}) and into proof_values; zeros for VCW_HOST
__global__ void __launch_bounds__(VCW_THREADS, 1)
k_vcw_proof(const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ state, uint32_t n, const uint64_t* __restrict__ doc_off,
            uint8_t* __restrict__ docs, uint8_t* __restrict__ proof_values) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t* pv = proof_values + (size_t)i * VCI_PV_CHARS;
    if (state[i] != VCW_BUILT) {
        for (int k = 0; k < VCI_PV_CHARS; k++) pv[k] = 0;
        return;
    }
    const uint4* s = (const uint4*)(sigs + (size_t)i * 64);
    uint32_t w[16];
#pragma unroll
    for (int q = 0; q < 4; q++) { const uint4 v = s[q]; w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w; }
    vci_proof_one(w, docs + doc_off[i + 1] - 3 - VCI_PV_CHARS, pv);
}

namespace launch {

static inline uint32_t vcw_blocks(uint64_t n) { return (uint32_t)((n + VCW_THREADS - 1) / VCW_THREADS); }
static const VcwProgram& vcw_program() {
    static const VcwProgram P = [] { VcwProgram p; vcw_program_build(&p); return p; }();
    return P;
}

cudaError_t vcw_records(const uint8_t* rec_cols, const uint64_t* rec_col_off, const int64_t* created_at, const uint64_t* rec_off, uint32_t m,
                        uint8_t* cls, uint64_t* id_len, cudaStream_t s, LaunchLog* lg) {
    if (m == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vcw_records", s, k_vcw_records<<<vcw_blocks(m), VCW_THREADS, 0, s>>>(rec_cols, rec_col_off, created_at, rec_off, m, cls, id_len));
    return cudaGetLastError();
}
cudaError_t vcw_sizes(const uint8_t* cols, const uint64_t* col_off, const uint64_t* rec_off, const int64_t* created_at, const uint8_t* cls,
                      const uint64_t* id_len, uint32_t n, uint64_t* msg_len, uint64_t* doc_len, uint64_t* arr, uint32_t* summary, uint8_t* state,
                      cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vcw_sizes", s, k_vcw_sizes<<<vcw_blocks(n), VCW_THREADS, 0, s>>>(vcw_program(), cols, col_off, rec_off, created_at, cls, id_len,
                                                                                      n, msg_len, doc_len, arr, summary, state));
    return cudaGetLastError();
}
cudaError_t vcw_fill(const uint8_t* cols, const uint64_t* col_off, const uint64_t* rec_off, const int64_t* created_at, const uint32_t* summary,
                     const uint8_t* state, const uint64_t* arr, uint32_t n, const uint64_t* msg_off, uint8_t* msgs, const uint64_t* doc_off,
                     uint8_t* docs, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vcw_fill", s, k_vcw_fill<<<vcw_blocks(n), VCW_THREADS, 0, s>>>(vcw_program(), cols, col_off, rec_off, created_at, summary, state,
                                                                                    arr, n, msg_off, msgs, doc_off, docs));
    return cudaGetLastError();
}
cudaError_t vcw_ids(const uint8_t* rec_cols, const uint64_t* rec_col_off, const uint64_t* rec_off, uint32_t n, uint32_t m, const uint8_t* state,
                    const uint64_t* arr, const uint64_t* id_off, const uint64_t* msg_off, uint8_t* msgs, const uint64_t* doc_off, uint8_t* docs,
                    cudaStream_t s, LaunchLog* lg) {
    if (m == 0 || n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vcw_ids", s, k_vcw_ids<<<vcw_blocks(m), VCW_THREADS, 0, s>>>(rec_cols, rec_col_off, rec_off, n, m, state, arr, id_off, msg_off,
                                                                                  msgs, doc_off, docs));
    return cudaGetLastError();
}
cudaError_t vcw_proof(const uint8_t* sigs, const uint8_t* state, uint32_t n, const uint64_t* doc_off, uint8_t* docs, uint8_t* proof_values,
                      cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    AFC_LAUNCH(lg, "k_vcw_proof", s, k_vcw_proof<<<vcw_blocks(n), VCW_THREADS, 0, s>>>(sigs, state, n, doc_off, docs, proof_values));
    return cudaGetLastError();
}
uint64_t vcw_literal_bytes() {
    static const uint64_t text = [] { VcwProgram p; return (uint64_t)vcw_program_build(&p); }();
    return text;
}

}  // namespace launch
}  // namespace afc
