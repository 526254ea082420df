// TEST-ONLY CPU build of the audit logic of agentfield_b200/csrc/afc_vcdoc.cuh: what one thread of k_vc_parse_capture records for a
// document and what k_vc_crosscheck then decides for it against its record's columns, plus the three rules on their own.  Compiled
// on its own by tests/test_audit_hostsim.py.
#define AFC_HOSTSIM 1
#include "../../agentfield_b200/csrc/afc_vcdoc.cuh"

using namespace afc;

extern "C" {

// 1 and the capture (VC_CAP_WORDS words) if the document is canonical for the schema, 0 if the device would leave it to the host
int hs_audit_capture(int kind, const uint8_t* doc, uint64_t len, uint32_t* cap) {
    static VcSchema S[2];
    static bool built = false;
    if (!built) { if (vc_schema_build(VC_DOC_EXECUTION, &S[0]) || vc_schema_build(VC_DOC_WORKFLOW, &S[1])) return -1; built = true; }
    if (kind != VC_DOC_EXECUTION && kind != VC_DOC_WORKFLOW) return -1;
    VcParse r;
    vc_parse_doc_t<true>(S[kind], doc, len, r, cap);
    return r.ok ? 1 : 0;
}
// the issue mask of a captured document; col_off: the record's 11 offsets into cols (NULL for workflow documents)
uint32_t hs_audit_mask(int kind, const uint8_t* doc, const uint32_t* cap, const uint8_t* cols, const uint64_t* col_off) {
    return vc_audit_mask(kind, doc, cap, cols, col_off);
}
int hs_column_equals(const uint8_t* span, uint32_t span_len, const uint8_t* col, uint64_t col_len) {
    return vc_column_equals(span, span_len, col, col_len) ? 1 : 0;
}
// 0..7 (unknown, pending, queued, running, succeeded, failed, cancelled, timeout) or 255 (undecided)
uint32_t hs_status_class(const uint8_t* s, uint64_t n, int is_span) { return vc_status_class(s, n, is_span != 0); }
// 0 valid, 1 invalid, 255 undecided
uint32_t hs_rfc3339(const uint8_t* s, uint32_t n) { return vc_rfc3339(s, n); }
int hs_cap_words(void) { return VC_CAP_WORDS; }

}  // extern "C"
