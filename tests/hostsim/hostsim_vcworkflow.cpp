// TEST-ONLY CPU build of the workflow-credential routines (agentfield_b200/csrc/afc_vcworkflow.cuh): what the threads of k_vcw_records,
// k_vcw_sizes, k_vcw_fill and k_vcw_ids do for one workflow.  Compiled on its own by tests/test_vcworkflow_hostsim.py.
#define AFC_HOSTSIM 1
#include <vector>

#include "../../agentfield_b200/csrc/afc_vcworkflow.cuh"

using namespace afc;

extern "C" {

// time.Time.UTC().Format(time.RFC3339) of n Unix seconds: 20 characters each
void hs_vcw_times(const int64_t* sec, uint32_t n, uint8_t* out) {
    for (uint32_t i = 0; i < n; i++) {
        ByteWriter w; w.init(out + 20 * (size_t)i);
        vcw_put_time(w, sec[i]);
        w.finish();
    }
}

uint32_t hs_vcw_record_class(const uint8_t* status, uint64_t len, int64_t sec, int64_t nsec) { return vcw_record_class(status, len, sec, nsec); }

// One workflow: cols with VCW_COLUMNS + 1 absolute offsets; its cnt records' columns with 2 cnt + 1 absolute offsets and their (seconds,
// nanoseconds).  Writes summary[4] and *state as k_vcw_sizes does, the two lengths, and — when msg and doc are given (the lengths plus
// 32 bytes) — both byte strings as k_vcw_fill and k_vcw_ids write them, the stored proofValue a placeholder.
int hs_vcw_issue(const uint8_t* cols, const uint64_t* coff, const uint8_t* rec_cols, const uint64_t* rec_coff, const int64_t* created, uint32_t cnt,
                 uint32_t* summary, uint32_t* state, uint8_t* msg, uint64_t* msg_len, uint8_t* doc, uint64_t* doc_len) {
    static VcwProgram P;
    static bool built = false;
    if (!built) { if (!vcw_program_build(&P)) return -1; built = true; }
    std::vector<uint8_t> cls(cnt + 1);
    std::vector<uint64_t> id_len(cnt + 1);
    for (uint32_t k = 0; k < cnt; k++) {                          // k_vcw_records
        const uint64_t a = rec_coff[2 * k], b = rec_coff[2 * k + 1], c = rec_coff[2 * k + 2];
        cls[k] = (uint8_t)vcw_record_class(rec_cols + b, c - b, created[2 * k], created[2 * k + 1]);
        id_len[k] = vcw_id_bytes(rec_cols + a, b - a);
    }
    const VcwPlan p = vcw_reduce(cls.data(), id_len.data(), created, cnt);     // k_vcw_sizes
    *state = p.state;
    if (p.state == VCW_HOST) {
        summary[0] = summary[1] = summary[2] = summary[3] = 0;
        *msg_len = *doc_len = 0;
        return 0;
    }
    summary[0] = p.status; summary[1] = p.completed; summary[2] = p.start; summary[3] = p.end;
    VcwItem it;
    it.cols = cols; it.coff = coff; it.cnt = cnt; it.status = p.status;
    it.start_sec = p.start != VCW_NONE ? created[2 * p.start] : 0;
    it.has_end = p.end != VCW_NONE;
    it.end_sec = it.has_end ? created[2 * p.end] : 0;
    it.ids_bytes = p.ids_bytes;
    uint64_t arr_at;
    vcw_doc_sizes(P, it, msg_len, doc_len, &arr_at);
    if (!msg || !doc) return 0;
    vcw_doc_fill(P, it, arr_at, msg, doc);                        // k_vcw_fill
    uint64_t before = 0;
    for (uint32_t k = 0; k < cnt; k++) {                          // k_vcw_ids
        const uint64_t at = arr_at + vcw_id_at(before, k);
        vcw_put_id(rec_cols + rec_coff[2 * k], rec_coff[2 * k + 1] - rec_coff[2 * k], k, msg + at, doc + at);
        before += id_len[k];
    }
    return 0;
}

}  // extern "C"
