// Execution webhook deliveries built and signed on the device (afc_webhook_sign_batch, include/afcrypto.h): the body
// json.Marshal(buildPayload(exec, determineWebhookEvent(exec.Status))) and the X-AgentField-Signature header of one delivery
// (internal/services/webhook_dispatcher.go:294-320, 394-419, 450-474; pkg/types/webhook.go:42-53).
//
//   wh_plan    the event (NormalizeExecutionStatus(status) == "succeeded", decided on printable-ASCII statuses as the audit path
//              does, vc_status_class; anything else is WH_HOST) and what the result member holds:
//                none     failed event, empty raw, or raw that decodes to null (omitempty drops a nil interface{})
//                value    json.Marshal(json.Unmarshal(raw)) (afc_jsonval.cuh); false, 0 and "" are written
//                string   raw that Unmarshal rejects by syntax: string(raw), invalid UTF-8 as U+FFFD byte by byte (go_json_escape)
//   wh_body    the constant text of ExecutionWebhookPayload interleaved with the escaped columns: event, execution_id,
//              workflow_id (RunID), status (raw, not normalised), target (node_id "." reasoner_id), type, duration_ms (*int64,
//              omitted when nil, 0 written), result (completed event only), error_message (failed event only, omitted when nil,
//              "" written), timestamp.  One template over the sink, like afc_vcissue.cuh.
//   wh_header_text  "sha256=" + hex(HMAC-SHA256(secret, body)), 71 characters; the HMAC is hmac_sha256_msg (keys over 64 bytes are
//              pre-hashed).
#pragma once
#include "afc_jsonval.cuh"
#include "afc_vcissue.cuh"

namespace afc {

enum {
    WH_COLUMNS = 8,          // execution_id, run_id, status, node_id, reasoner_id, target_type, timestamp, error_message (AFC_WEBHOOK_COLUMNS)
    WH_COL_EXEC = 0, WH_COL_RUN = 1, WH_COL_STATUS = 2, WH_COL_NODE = 3, WH_COL_REASONER = 4, WH_COL_TYPE = 5, WH_COL_TIMESTAMP = 6,
    WH_COL_ERROR = 7,
    WH_HEADER_CHARS = 71,
};
enum : uint32_t { WH_HAS_DURATION = 1, WH_HAS_ERROR_MESSAGE = 2, WH_HAS_SECRET = 4 };     // AFC_WEBHOOK_HAS_*
enum : uint32_t { WH_BUILT = 0, WH_HOST = 1 };                                            // AFC_WEBHOOK_BUILT / _HOST
// a delivery's plan, kept between the passes: WH_P_HOST, or the event bit and the result kind
enum : uint32_t { WH_P_HOST = 1, WH_P_COMPLETED = 2, WH_P_VALUE = 4, WH_P_STRING = 8 };

struct WhItem {
    const uint8_t* cols;
    const uint64_t* coff;       // its WH_COLUMNS + 1 absolute offsets into cols
    int64_t duration;
    uint32_t flags;
    const uint8_t* result;      // the raw result bytes (empty: nil)
    uint64_t result_len;
};

AFC_HD uint32_t wh_plan(const WhItem& it) {
    const uint64_t s0 = it.coff[WH_COL_STATUS];
    const uint32_t cls = vc_status_class(it.cols + s0, it.coff[WH_COL_STATUS + 1] - s0, false);
    if (cls == VC_UNDECIDED) return WH_P_HOST;
    if (cls != 4) return 0;                                     // execution.failed
    if (it.result_len == 0) return WH_P_COMPLETED;
    const uint32_t v = jv_validate(it.result, it.result_len);
    if (v == JV_HOST) return WH_P_HOST;
    if (v == JV_SYNTAX) return WH_P_COMPLETED | WH_P_STRING;
    const uint32_t p = jv_skip_ws(it.result, 0, (uint32_t)it.result_len);
    return it.result[p] == 'n' ? WH_P_COMPLETED : WH_P_COMPLETED | WH_P_VALUE;     // a null value is a nil interface{}
}

template <class Sink>
AFC_HD void wh_col(Sink& out, const WhItem& it, uint32_t c) { go_json_escape(out, it.cols + it.coff[c], it.coff[c + 1] - it.coff[c]); }

// The body of a delivery whose plan is not WH_P_HOST; false = the result declined (jv_emit).  tape: afc_jsonval.cuh.
template <class Sink>
AFC_HD bool wh_body(Sink& out, const WhItem& it, uint32_t plan, uint32_t* tape) {
    const bool completed = plan & WH_P_COMPLETED;
    vci_put_text(out, completed ? "{\"event\":\"execution.completed\",\"execution_id\":\"" : "{\"event\":\"execution.failed\",\"execution_id\":\"");
    wh_col(out, it, WH_COL_EXEC);
    vci_put_text(out, "\",\"workflow_id\":\"");
    wh_col(out, it, WH_COL_RUN);
    vci_put_text(out, "\",\"status\":\"");
    wh_col(out, it, WH_COL_STATUS);
    vci_put_text(out, "\",\"target\":\"");
    wh_col(out, it, WH_COL_NODE);
    out.put('.');
    wh_col(out, it, WH_COL_REASONER);
    vci_put_text(out, "\",\"type\":\"");
    wh_col(out, it, WH_COL_TYPE);
    out.put('"');
    if (it.flags & WH_HAS_DURATION) { vci_put_text(out, ",\"duration_ms\":"); vci_put_int(out, it.duration); }
    if (plan & WH_P_VALUE) {
        vci_put_text(out, ",\"result\":");
        if (!jv_emit(out, it.result, (uint32_t)it.result_len, tape)) return false;
    } else if (plan & WH_P_STRING) {
        vci_put_text(out, ",\"result\":\"");
        go_json_escape(out, it.result, it.result_len);
        out.put('"');
    } else if (!completed && (it.flags & WH_HAS_ERROR_MESSAGE)) {
        vci_put_text(out, ",\"error_message\":\"");
        wh_col(out, it, WH_COL_ERROR);
        out.put('"');
    }
    vci_put_text(out, ",\"timestamp\":\"");
    wh_col(out, it, WH_COL_TIMESTAMP);
    out.put('"'); out.put('}');
    return true;
}

// "sha256=" + 64 lower-case hex digits of a 32-byte HMAC-SHA256 (mac), or 71 zero bytes (mac == nullptr)
AFC_HD void wh_header_text(uint8_t* out, const uint8_t* mac) {
    if (!mac) { for (int k = 0; k < WH_HEADER_CHARS; k++) out[k] = 0; return; }
    out[0] = 's'; out[1] = 'h'; out[2] = 'a'; out[3] = '2'; out[4] = '5'; out[5] = '6'; out[6] = '=';
    for (int k = 0; k < 32; k++) {
        const uint32_t b = mac[k];
        out[7 + 2 * k] = (uint8_t)json_hex_digit(b >> 4);
        out[8 + 2 * k] = (uint8_t)json_hex_digit(b & 15u);
    }
}

// (host code) The constant text a body can hold at most (completed event, every optional member, a 20-character int64, the result's quotes):
// with 6 bytes per column and result byte it bounds the body (afc_webhook_bound)
static inline uint64_t wh_fixed_bytes() {
    static const char* const lits[] = {"{\"event\":\"execution.completed\",\"execution_id\":\"", "\",\"workflow_id\":\"", "\",\"status\":\"",
                                       "\",\"target\":\"", ".", "\",\"type\":\"", "\"", ",\"duration_ms\":", "-9223372036854775808",
                                       ",\"result\":\"\"", ",\"error_message\":\"\"", ",\"timestamp\":\"", "\"}"};
    uint64_t n = 0;
    for (const char* s : lits) n += strlen(s);
    return n;
}

}  // namespace afc
