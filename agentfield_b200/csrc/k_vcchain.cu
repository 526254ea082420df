// Workflow VC chains served on the device (afc_vc_workflow_chain_batch, include/afcrypto.h; afc_vcchain.cuh).
//
// Reference call sites replaced (relative to /root/reference/control-plane):
//   (the workflow-credential passes of k_vcworkflow.cu, unchanged)   generateWorkflowVCDocument   internal/services/vc_service.go:525-632
//   k_vcc_records / k_vcc_distinct   collectDIDResolutionBundle: the DIDs, ResolveDID (a directory probe), the map's key order   :810-870
//   k_vcc_sizes / k_vcc_frame / k_vcc_emit_records / k_vcc_emit_entries / k_vcc_copy_doc   c.JSON(WorkflowVCChainResponse)
//                                                                   internal/handlers/ui/did.go:383, pkg/types/did_types.go:287-295
//
// Workflow i owns the DID occurrence slots [o_i, o_i + 3 cnt_i + 1), o_i = 3 (rec_off[i] - rec_off[0]) + i: the issuer, caller and target of
// each of its records, then the workflow credential's issuer.  k_vcc_records runs one thread per record: its state, its text's length and
// the directory rank of its three DIDs (VCC_NONE for a DID the bundle skips or the directory lacks).  k_vcc_distinct runs one CTA per
// workflow: a hash set of 2 x slots entries in scratch takes each rank once, the distinct ranks are merge-sorted (each element finds its
// place in the other run by binary search, O(d log^2 d) for d distinct ranks), in shared memory when they fit and in the hash set's
// scratch otherwise, and each bundle member's length is written.  The existing scan turns the record and member lengths into offsets;
// k_vcc_sizes lays out each body.  The emit passes write at final offsets through ByteWriter: the frame one thread per workflow, the
// records and their ids one thread per record, the bundle one thread per member, the stored credential one CTA per workflow.
#include "afc_launch.h"
#include "afc_vcchain.cuh"

namespace afc {

static constexpr int VCC_THREADS = 128;
static constexpr int VCC_CTA = 256;          // k_vcc_distinct, k_vcc_copy_doc
static constexpr uint32_t VCC_SORT_CAP = 2048;  // distinct ranks sorted in shared memory (2 x 8 KB)
enum { VCC_LAY = 9 };                        // per workflow: the five part starts, then the records, the ids' '[', the document, the bundle

__device__ __forceinline__ uint64_t vcc_occ_base(const uint64_t* rec_off, uint32_t i) { return 3 * (rec_off[i] - rec_off[0]) + i; }

// the workflow holding batch record j: the last i with rec_off[i] <= rec_off[0] + j
__device__ __forceinline__ uint32_t vcc_workflow_of_record(const uint64_t* rec_off, uint32_t n, uint64_t j) {
    const uint64_t r = rec_off[0] + j;
    uint32_t lo = 0, hi = n;
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (rec_off[mid] <= r) lo = mid; else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ uint32_t vcc_workflow_of_slot(const uint64_t* rec_off, uint32_t n, uint64_t s) {
    uint32_t lo = 0, hi = n;
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (vcc_occ_base(rec_off, mid) <= s) lo = mid; else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ VccStr vcc_col(const uint8_t* cols, const uint64_t* off, uint64_t k) {
    VccStr s; s.p = cols + off[k]; s.len = off[k + 1] - off[k];
    return s;
}

__device__ __forceinline__ VccRecord vcc_load_record(const launch::VccArgs& A, uint64_t r) {
    VccRecord x;
    x.vc_id = vcc_col(A.rec_cols, A.rec_col_off, 2 * r);
    x.status = vcc_col(A.rec_cols, A.rec_col_off, 2 * r + 1);
    x.cols = A.chain_rec_cols; x.coff = A.chain_rec_col_off + VCC_REC_COLUMNS * r;
    x.flags = A.rec_flags[r];
    x.doc_size = A.doc_size[r];
    x.sec = A.created_at[2 * r]; x.nsec = A.created_at[2 * r + 1]; x.zone = A.created_off[r];
    return x;
}

// the directory rank of a DID the bundle takes, VCC_NONE otherwise; a DID longer than VCC_DID_MAX that the bundle would take declines
// workflow i
__device__ __forceinline__ uint32_t vcc_rank(const launch::VccArgs& A, VccStr d, uint32_t i) {
    if (!vcc_did_wanted(d.p, d.len) || d.len >= 0xffffffffull) return VCC_NONE;
    const uint32_t k = vcj_resolve(d.p, (uint32_t)d.len, A.dir_dids, A.dir_off, A.dir_slots, A.dir_mask);
    if (k == 0xffffffffu) return VCC_NONE;
    if (d.len > VCC_DID_MAX) atomicOr(A.host + i, 1u);
    return A.dir_rank[k];
}

// Record j: its state (a HOST record marks its workflow), its text's length with the comma before it, its three DIDs' ranks
__global__ void __launch_bounds__(VCC_THREADS, 1)
k_vcc_records(const launch::VccArgs A) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= A.m) return;
    const uint32_t i = vcc_workflow_of_record(A.rec_off, A.n, j);
    const uint64_t r = A.rec_off[0] + j, k = r - A.rec_off[i];
    const VccRecord x = vcc_load_record(A, r);
    uint64_t len = 0;
    if (vcc_record_state(x) == VCC_HOST) {
        atomicOr(A.host + i, 1u);
    } else {
        ByteCounter c; c.init();
        vcc_record(c, x);
        len = c.n + (k ? 1 : 0);
    }
    A.rlen[j + 1] = len;
    uint32_t* rank = A.rank + vcc_occ_base(A.rec_off, i) + 3 * k;
    rank[0] = vcc_rank(A, x.col(VCC_R_ISSUER), i);
    rank[1] = vcc_rank(A, x.col(VCC_R_CALLER), i);
    rank[2] = vcc_rank(A, x.col(VCC_R_TARGET), i);
}

__device__ __forceinline__ bool vcc_insert(uint32_t* set, uint32_t size, uint32_t x) {
    uint32_t h = (uint32_t)(((uint64_t)(x * 0x9E3779B1u) * size) >> 32);
    for (;;) {
        const uint32_t old = atomicCAS(set + h, VCC_NONE, x);
        if (old == VCC_NONE) return true;
        if (old == x) return false;
        h = h + 1 == size ? 0 : h + 1;
    }
}

// Merge sort of nd distinct values, a -> b -> a ...: in each round an element's place in the merged pair of runs is its place in its own
// run plus the number of smaller elements in the other run.  Returns the buffer that holds the sorted values.
__device__ uint32_t* vcc_sort(uint32_t* a, uint32_t* b, uint32_t nd) {
    for (uint32_t w = 1; w < nd; w *= 2) {
        for (uint32_t j = threadIdx.x; j < nd; j += blockDim.x) {
            const uint32_t x = a[j], run = j / w, own = run * w, other = (run ^ 1) * w, pair = (run & ~1u) * w;
            uint32_t lo = 0, hi = other < nd ? min(w, nd - other) : 0;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) / 2;
                if (a[other + mid] < x) lo = mid + 1; else hi = mid;
            }
            b[pair + (j - own) + lo] = x;
        }
        __syncthreads();
        uint32_t* t = a; a = b; b = t;
    }
    return a;
}

// Workflow blockIdx.x: the credential issuer's rank, the distinct ranks in order at dlist + o_i, their count, each member's length
__global__ void __launch_bounds__(VCC_CTA, 1)
k_vcc_distinct(const launch::VccArgs A) {
    __shared__ uint32_t sa[VCC_SORT_CAP], sb[VCC_SORT_CAP];
    __shared__ uint32_t count;
    const uint32_t i = blockIdx.x;
    const uint64_t base = vcc_occ_base(A.rec_off, i), cnt = A.rec_off[i + 1] - A.rec_off[i];
    const uint32_t slots = (uint32_t)(3 * cnt + 1);
    uint32_t* set = A.hset + 2 * base;
    uint32_t* list = A.dlist + base;
    if (threadIdx.x == 0) {
        count = 0;
        A.rank[base + 3 * cnt] = vcc_rank(A, vcc_col(A.cols, A.col_off, (uint64_t)i * VCW_COLUMNS + VCW_COL_ISSUER), i);
    }
    __syncthreads();
    for (uint32_t s = threadIdx.x; s < slots; s += blockDim.x) {
        const uint32_t x = A.rank[base + s];
        if (x != VCC_NONE && vcc_insert(set, 2 * slots, x)) list[atomicAdd(&count, 1u)] = x;
    }
    __syncthreads();
    const uint32_t nd = count;
    if (nd <= VCC_SORT_CAP) {
        for (uint32_t k = threadIdx.x; k < nd; k += blockDim.x) sa[k] = list[k];
        __syncthreads();
        const uint32_t* sorted = vcc_sort(sa, sb, nd);
        for (uint32_t k = threadIdx.x; k < nd; k += blockDim.x) list[k] = sorted[k];
    } else {                                                      // the set's 2 x slots entries are free now: the second buffer
        const uint32_t* sorted = vcc_sort(list, set, nd);
        if (sorted != list)
            for (uint32_t k = threadIdx.x; k < nd; k += blockDim.x) list[k] = sorted[k];
    }
    __syncthreads();
    const VccStr resolved = vcc_col(A.chain_cols, A.chain_col_off, (uint64_t)i * VCC_COLUMNS + VCC_COL_RESOLVED_AT);
    const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (uint32_t k = threadIdx.x; k < slots; k += blockDim.x) {
        uint64_t len = 0;
        if (k < nd) {
            const uint32_t d = A.dir_order[list[k]];
            VccStr did; did.p = A.dir_dids + A.dir_off[d]; did.len = A.dir_off[d + 1] - A.dir_off[d];
            ByteCounter c; c.init();
            vcc_entry(c, did, zero, resolved);
            len = c.n + (k ? 1 : 0);
        }
        A.elen[base + k + 1] = len;
    }
    if (threadIdx.x == 0) A.ndist[i] = nd;
}

__device__ __forceinline__ VccFrame vcc_load_frame(const launch::VccArgs& A, uint32_t i) {
    VccFrame f;
    const uint64_t* co = A.col_off + (size_t)i * VCW_COLUMNS;
    f.workflow_id = vcc_col(A.cols, co, VCW_COL_WORKFLOW);
    f.session_id = vcc_col(A.cols, co, VCW_COL_SESSION);
    f.issuer = vcc_col(A.cols, co, VCW_COL_ISSUER);
    f.wf_vc_id = vcc_col(A.chain_cols, A.chain_col_off, (uint64_t)i * VCC_COLUMNS + VCC_COL_WF_VC_ID);
    const uint64_t r0 = A.rec_off[i];
    f.cnt = (uint32_t)(A.rec_off[i + 1] - r0);
    const uint32_t* sm = A.summary + 4 * (size_t)i;
    f.status = sm[0]; f.completed = sm[1];
    for (int t = 0; t < 3; t++) f.snap[t] = A.clock[3 * (size_t)i + t];
    if (f.cnt) {
        const uint64_t r = r0 + sm[2];
        f.start[0] = A.created_at[2 * r]; f.start[1] = A.created_at[2 * r + 1]; f.start[2] = A.created_off[r];
    } else {
        for (int t = 0; t < 3; t++) f.start[t] = f.snap[t];
    }
    f.has_end = sm[3] != VCW_NONE;
    const uint64_t e = r0 + (f.has_end ? sm[3] : 0);
    f.end[0] = f.has_end ? A.created_at[2 * e] : 0; f.end[1] = f.has_end ? A.created_at[2 * e + 1] : 0; f.end[2] = f.has_end ? A.created_off[e] : 0;
    f.has_bundle = A.ndist[i] != 0;
    f.proof_value = A.pv + (size_t)i * VCI_PV_CHARS;
    f.doc_len = A.doc_off[i + 1] - A.doc_off[i];
    return f;
}

// Workflow i: its state and body length, and where each part and region of its body starts
__global__ void __launch_bounds__(VCC_THREADS, 1)
k_vcc_sizes(const launch::VccArgs A) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= A.n) return;
    const VccFrame f = vcc_load_frame(A, i);
    const VccStr resolved = vcc_col(A.chain_cols, A.chain_col_off, (uint64_t)i * VCC_COLUMNS + VCC_COL_RESOLVED_AT);
    const bool host = A.wstate[i] != VCW_BUILT || A.host[i] || !vcc_time_ok(f.snap[0], f.snap[1], f.snap[2]) || resolved.len > VCC_RESOLVED_MAX;
    A.state[i] = (uint8_t)(host ? VCC_HOST : VCC_BUILT);
    if (host) { A.body_off[i + 1] = 0; return; }
    const uint64_t j0 = A.rec_off[i] - A.rec_off[0], o = vcc_occ_base(A.rec_off, i);
    const uint64_t recs = A.rlen[j0 + f.cnt] - A.rlen[j0], ents = A.elen[o + 3 * f.cnt + 1] - A.elen[o];
    uint64_t L[VCC_PARTS];
    for (uint32_t p = 0; p < VCC_PARTS; p++) { ByteCounter c; c.init(); vcc_frame(c, f, p); L[p] = c.n; }
    uint64_t* lay = A.lay + (size_t)i * VCC_LAY;
    lay[0] = 0;
    lay[5] = L[0];                                                // the records
    lay[1] = L[0] + recs;
    lay[6] = lay[1] + L[1] - 1;                                   // the ids' '['
    lay[2] = lay[6] + A.arr[2 * (size_t)i + 1] - 1;               // the ']' after them
    lay[7] = lay[2] + L[2];                                       // the stored document
    lay[3] = lay[7] + f.doc_len;
    lay[8] = lay[3] + L[3];                                       // the bundle's members
    lay[4] = lay[8] + ents;
    A.body_off[i + 1] = lay[4] + L[4];
}

__global__ void __launch_bounds__(VCC_THREADS, 1)
k_vcc_frame(const launch::VccArgs A) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= A.n || A.state[i] != VCC_BUILT) return;
    const VccFrame f = vcc_load_frame(A, i);
    const uint64_t* lay = A.lay + (size_t)i * VCC_LAY;
    uint8_t* body = A.bodies + A.body_off[i];
    for (uint32_t p = 0; p < VCC_PARTS; p++) {
        ByteWriter w; w.init(body + lay[p]);
        vcc_frame(w, f, p);
        w.finish();
    }
}

// Record j: its text in component_vcs and its id in the credential's component_vcs
__global__ void __launch_bounds__(VCC_THREADS, 1)
k_vcc_emit_records(const launch::VccArgs A) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= A.m) return;
    const uint32_t i = vcc_workflow_of_record(A.rec_off, A.n, j);
    if (A.state[i] != VCC_BUILT) return;
    const uint64_t r = A.rec_off[0] + j, k = r - A.rec_off[i], first = j - k;
    const uint64_t* lay = A.lay + (size_t)i * VCC_LAY;
    uint8_t* body = A.bodies + A.body_off[i];
    const VccRecord x = vcc_load_record(A, r);
    {
        ByteWriter w; w.init(body + lay[5] + A.rlen[j] - A.rlen[first]);
        if (k) w.put(',');
        vcc_record(w, x);
        w.finish();
    }
    ByteWriter w; w.init(body + lay[6] + vcw_id_at(A.id_off[j] - A.id_off[first], (uint32_t)k));
    if (k) w.put(',');
    w.put('"');
    go_json_escape(w, x.vc_id.p, x.vc_id.len);
    w.put('"');
    w.finish();
}

// Occurrence slot s: the bundle member it stands for, if its workflow has that many
__global__ void __launch_bounds__(VCC_THREADS, 1)
k_vcc_emit_entries(const launch::VccArgs A, uint64_t slots) {
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= slots) return;
    const uint32_t i = vcc_workflow_of_slot(A.rec_off, A.n, s);
    const uint64_t o = vcc_occ_base(A.rec_off, i), k = s - o;
    if (k >= A.ndist[i] || A.state[i] != VCC_BUILT) return;
    const uint32_t d = A.dir_order[A.dlist[s]];
    VccStr did; did.p = A.dir_dids + A.dir_off[d]; did.len = A.dir_off[d + 1] - A.dir_off[d];
    const uint4* q = (const uint4*)(A.dir_pks + 32 * (size_t)d);
    const uint4 q0 = q[0], q1 = q[1];
    const uint32_t pk[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
    ByteWriter w; w.init(A.bodies + A.body_off[i] + A.lay[(size_t)i * VCC_LAY + 8] + A.elen[s] - A.elen[o]);
    if (k) w.put(',');
    vcc_entry(w, did, pk, vcc_col(A.chain_cols, A.chain_col_off, (uint64_t)i * VCC_COLUMNS + VCC_COL_RESOLVED_AT));
    w.finish();
}

// Workflow blockIdx.x: its stored credential, byte for byte (json.Marshal wrote it compact and escaped, so appendCompact keeps it)
__global__ void __launch_bounds__(VCC_CTA, 1)
k_vcc_copy_doc(const launch::VccArgs A) {
    const uint32_t i = blockIdx.x;
    if (A.state[i] != VCC_BUILT) return;
    const uint8_t* src = A.docs + A.doc_off[i];
    uint8_t* dst = A.bodies + A.body_off[i] + A.lay[(size_t)i * VCC_LAY + 7];
    const uint64_t len = A.doc_off[i + 1] - A.doc_off[i];
    for (uint64_t b = threadIdx.x; b < len; b += blockDim.x) dst[b] = src[b];
}

namespace launch {

static inline uint32_t vcc_blocks(uint64_t n) { return (uint32_t)((n + VCC_THREADS - 1) / VCC_THREADS); }

size_t vcc_lay_words() { return VCC_LAY; }

cudaError_t vcc_sizes(const VccArgs& A, cudaStream_t s, LaunchLog* lg) {
    if (A.n == 0) return cudaSuccess;
    const uint64_t slots = 3 * (uint64_t)A.m + A.n;
    cudaError_t e = cudaMemsetAsync(A.hset, 0xff, 2 * slots * sizeof(uint32_t), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(A.host, 0, (size_t)A.n * sizeof(uint32_t), s);
    if (e != cudaSuccess) return e;
    if (A.m) {
        AFC_LAUNCH(lg, "k_vcc_records", s, k_vcc_records<<<vcc_blocks(A.m), VCC_THREADS, 0, s>>>(A));
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        if ((e = offsets_from_lengths(A.rlen, A.m, A.scan, s, lg)) != cudaSuccess) return e;
    } else if ((e = cudaMemsetAsync(A.rlen, 0, sizeof(uint64_t), s)) != cudaSuccess) {
        return e;
    }
    AFC_LAUNCH(lg, "k_vcc_distinct", s, k_vcc_distinct<<<A.n, VCC_CTA, 0, s>>>(A));
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if ((e = offsets_from_lengths(A.elen, (uint32_t)slots, A.scan, s, lg)) != cudaSuccess) return e;
    AFC_LAUNCH(lg, "k_vcc_sizes", s, k_vcc_sizes<<<vcc_blocks(A.n), VCC_THREADS, 0, s>>>(A));
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    return offsets_from_lengths(A.body_off, A.n, A.scan, s, lg);
}

cudaError_t vcc_emit(const VccArgs& A, cudaStream_t s, LaunchLog* lg) {
    if (A.n == 0) return cudaSuccess;
    const uint64_t slots = 3 * (uint64_t)A.m + A.n;
    AFC_LAUNCH(lg, "k_vcc_frame", s, k_vcc_frame<<<vcc_blocks(A.n), VCC_THREADS, 0, s>>>(A));
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && A.m) {
        AFC_LAUNCH(lg, "k_vcc_emit_records", s, k_vcc_emit_records<<<vcc_blocks(A.m), VCC_THREADS, 0, s>>>(A));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        AFC_LAUNCH(lg, "k_vcc_emit_entries", s, k_vcc_emit_entries<<<vcc_blocks(slots), VCC_THREADS, 0, s>>>(A, slots));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        AFC_LAUNCH(lg, "k_vcc_copy_doc", s, k_vcc_copy_doc<<<A.n, VCC_CTA, 0, s>>>(A));
        e = cudaGetLastError();
    }
    return e;
}

uint64_t vcc_frame_fixed() { return VCC_FRAME_FIXED; }
uint64_t vcc_record_fixed() { return VCC_RECORD_FIXED; }
uint64_t vcc_entry_fixed() { return VCC_ENTRY_FIXED; }

}  // namespace launch
}  // namespace afc
