// Stored credential documents read back on the device (SURVEY.md §8f N3, verify half).
//
// VCService.VerifyVC (internal/services/vc_service.go:242-289) verifies json.Marshal(Unmarshal(D) with Proof = VCProof{}).  When
// the stored bytes D are already exactly what json.Marshal writes for the struct, that message is D[0 : p] followed by the
// zero-proof text, p = the offset just after "proof":.  The parser below PROVES that D is in that form with local, conservative
// checks (fixed member layout, Go's string escaping, integers that round-trip, sorted metadata keys, ...) and declines (VC_HOST)
// whatever it cannot prove: the caller then re-marshals that document on the host, as before.  Accepting is exact, declining is
// only slower.  The string rules are those of afc_json.cuh (what go_json_escape writes), read in the other direction.
//
// A schema is a short program of operations over a literal pool; one document per thread walks it with a ByteWindow (aligned
// 32-bit loads), literals compared a word at a time, plain string bytes consumed four at a time (json_word_is_plain).
// Shared by the device kernels (k_vcdoc.cu) and the CPU build of the same logic in tests/hostsim.
#pragma once
#include "afc_json.cuh"

namespace afc {

// per-document verdicts (include/afcrypto.h AFC_VC_*)
enum { VC_INVALID = 0, VC_VALID = 1, VC_HOST = 2, VC_UNRESOLVED = 3, VC_BAD_ENCODING = 4 };
enum { VC_DOC_EXECUTION = 0, VC_DOC_WORKFLOW = 1 };

enum VcCode : uint8_t {
    VOP_LIT,            // constant text
    VOP_STR,            // string body (the quotes are literal text), escapes allowed
    VOP_ISSUER,         // string body without escapes; span recorded (it is looked up as the DID)
    VOP_ISSUANCE,       // string body; span recorded
    VOP_STRLIST,        // []string: null or [ "..." , ... ]
    VOP_INT,            // Go int: -?(0|[1-9][0-9]*), at most 18 digits, not -0
    VOP_OPT_STR,        // *string with omitempty: absent, or the member text, a string body and its closing quote ("" allowed)
    VOP_OPT_STR_NE,     // string with omitempty: absent, or present and non-empty
    VOP_ANY,            // map[string]interface{}: null or an object (sorted keys without escapes, nested up to VC_MAX_DEPTH)
    VOP_PROOF,          // marks p, the end of the signed prefix
    VOP_PROOFVALUE,     // string body without escapes; span recorded
    VOP_END             // nothing may follow
};
constexpr int VC_MAX_OPS = 64, VC_POOL_WORDS = 256, VC_MAX_DEPTH = 8;
struct VcOp { uint16_t off; uint8_t len; uint8_t code; };      // literal at pool byte `off` (a multiple of 4), `len` bytes
struct VcSchema {
    uint32_t n_ops, tail_off, tail_len, pad;                     // tail: the zero-proof text appended after D[0:p]
    VcOp ops[VC_MAX_OPS];
    uint32_t pool[VC_POOL_WORDS];                                // literals, each starting on a word, zero padded
};

struct VcParse {
    uint32_t ok;                          // 1 = the document is canonical for the schema
    uint32_t proof_at;                    // p
    uint32_t iss_off, iss_len, date_off, date_len, pv_off, pv_len;
};

AFC_HD uint32_t vc_mask(uint32_t m) { return m >= 4 ? 0xffffffffu : (1u << (8 * m)) - 1u; }

// the next `len` bytes equal the pool literal at byte `off`
AFC_HD bool vc_lit(ByteWindow& w, const uint32_t* pool, uint32_t off, uint32_t len) {
    for (uint32_t k = 0; k < len; k += 4) {
        w.fill();
        const uint32_t m = len - k < 4 ? len - k : 4;
        if (w.have < m || (((uint32_t)w.win ^ pool[(off + k) >> 2]) & vc_mask(m))) return false;
        w.skip(m);
    }
    return true;
}
// the next byte is c (consumed)
AFC_HD bool vc_byte(ByteWindow& w, uint32_t c) {
    w.fill();
    if (w.have == 0 || w.peek(0) != c) return false;
    w.skip(1);
    return true;
}
// the next m (<= 4) bytes are the little-endian word x (consumed)
AFC_HD bool vc_word(ByteWindow& w, uint32_t x, uint32_t m) {
    w.fill();
    if (w.have < m || (((uint32_t)w.win ^ x) & vc_mask(m))) return false;
    w.skip(m);
    return true;
}
AFC_HD bool vc_is_lower_hex(uint32_t c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'f'); }

// A string body exactly as Go's encoder writes it, up to (not including) the closing quote; *n = its length in bytes.
AFC_HD bool vc_str(ByteWindow& w, bool allow_escape, uint32_t* n) {
    uint32_t len = 0;
    for (;;) {
        w.fill();
        if (w.have >= 4 && json_word_is_plain((uint32_t)w.win)) { w.skip(4); len += 4; continue; }
        if (w.have == 0) return false;
        const uint32_t b = w.peek(0);
        if (b == '"') { *n = len; return true; }
        if (b < 0x20 || b == '<' || b == '>' || b == '&') return false;       // Go escapes these
        if (b == '\\') {
            if (!allow_escape || w.have < 2) return false;
            const uint32_t c = w.peek(1);
            if (c == '"' || c == '\\' || c == 'b' || c == 'f' || c == 'n' || c == 'r' || c == 't') { w.skip(2); len += 2; continue; }
            if (c != 'u') return false;                                           // \/ and friends: Go never writes them
            w.skip(2); w.fill();
            if (w.have < 4) return false;
            const uint32_t h0 = w.peek(0), h1 = w.peek(1), h2 = w.peek(2), h3 = w.peek(3);
            bool good;
            if (h0 == '0' && h1 == '0') {
                if (h2 == '0' || h2 == '1') {                                     // other control bytes: \u00XX, lowercase
                    const uint32_t v = ((h2 - '0') << 4) | (h3 <= '9' ? h3 - '0' : h3 - 'a' + 10);
                    good = vc_is_lower_hex(h3) && v != 0x08 && v != 0x09 && v != 0x0a && v != 0x0c && v != 0x0d;
                } else {
                    good = (h2 == '3' && (h3 == 'c' || h3 == 'e')) || (h2 == '2' && h3 == '6');     // < > &
                }
            } else {
                good = h0 == '2' && h1 == '0' && h2 == '2' && (h3 == '8' || h3 == '9');          // U+2028 / U+2029
            }
            if (!good) return false;                                              // includes �: Go does not round-trip it
            w.skip(4); len += 6;
            continue;
        }
        if (b < 0x80) { w.skip(1); ++len; continue; }
        const uint32_t k = utf8_valid_len(w, w.rem);
        if (k == 0) return false;
        if (k == 3 && b == 0xE2 && w.peek(1) == 0x80 && (w.peek(2) == 0xA8 || w.peek(2) == 0xA9)) return false;
        w.skip(k); len += k;
    }
}
// "..." including both quotes
AFC_HD bool vc_quoted(ByteWindow& w, bool allow_escape, uint32_t* n) {
    return vc_byte(w, '"') && vc_str(w, allow_escape, n) && vc_byte(w, '"');
}

// -?(0|[1-9][0-9]*) with at most max_digits digits; -0 only if allowed.  What follows is checked by the caller.
AFC_HD bool vc_int(ByteWindow& w, uint32_t max_digits, bool allow_neg_zero) {
    w.fill();
    if (w.have == 0) return false;
    const bool neg = w.peek(0) == '-';
    if (neg) { w.skip(1); w.fill(); if (w.have == 0) return false; }
    uint32_t d = w.peek(0);
    if (d < '0' || d > '9') return false;
    if (d == '0') { w.skip(1); return !neg || allow_neg_zero; }
    uint32_t count = 0;
    while (w.have && (d = w.peek(0)) >= '0' && d <= '9') {
        if (++count > max_digits) return false;
        w.skip(1); w.fill();
    }
    return true;
}

AFC_HD bool vc_strlist(ByteWindow& w) {
    w.fill();
    if (w.have && w.peek(0) == 'n') return vc_word(w, 0x6c6c756eu, 4);          // null
    if (!vc_byte(w, '[')) return false;
    w.fill();
    if (w.have && w.peek(0) == ']') { w.skip(1); return true; }
    for (;;) {
        uint32_t n;
        if (!vc_quoted(w, true, &n)) return false;
        w.fill();
        if (w.have == 0) return false;
        const uint32_t c = w.peek(0);
        w.skip(1);
        if (c == ']') return true;
        if (c != ',') return false;
    }
}

// the key at [co, co+cl) sorts strictly after the one at [po, po+pl) (Go sorts map keys by bytes)
AFC_HD bool vc_key_after(const uint8_t* d, uint32_t po, uint32_t pl, uint32_t co, uint32_t cl) {
    const uint32_t m = pl < cl ? pl : cl;
    for (uint32_t j = 0; j < m; j++) {
        const uint32_t a = d[po + j], b = d[co + j];
        if (a != b) return b > a;
    }
    return cl > pl;
}

// map[string]interface{} after json.Unmarshal: null, or an object whose values are strings, true / false / null, integers that
// float64 holds exactly and strconv writes back unchanged (-?(0|[1-9][0-9]{0,14}), and -0), arrays and objects (keys sorted by
// bytes, no escapes in keys) nested at most VC_MAX_DEPTH deep.  `len` = document length (positions are len - w.rem).
AFC_HD bool vc_any(ByteWindow& w, const uint8_t* d, uint64_t len) {
    w.fill();
    if (w.have && w.peek(0) == 'n') return vc_word(w, 0x6c6c756eu, 4);
    if (!vc_byte(w, '{')) return false;
    uint32_t is_obj = 1, depth = 1;                // bit k of is_obj: container k is an object
    uint32_t pko[VC_MAX_DEPTH], pkl[VC_MAX_DEPTH];  // previous key of each open object (pkl = 0xffffffff: none yet)
    pkl[0] = 0xffffffffu; pko[0] = 0;
    bool first = true;                              // just after an opening bracket
    for (;;) {
        const uint32_t top = depth - 1;
        const bool obj = (is_obj >> top) & 1;
        w.fill();
        if (w.have == 0) return false;
        uint32_t c = w.peek(0);
        if (first && c == (obj ? '}' : ']')) {
            w.skip(1);
            goto closed;
        }
        if (!first) {                               // after a value: separator or close
            w.skip(1);
            if (c == (obj ? '}' : ']')) goto closed;
            if (c != ',') return false;
        }
        first = false;
        if (obj) {                                  // key
            const uint32_t ko = (uint32_t)(len - w.rem) + 1;
            uint32_t kl;
            if (!vc_quoted(w, false, &kl)) return false;
            if (pkl[top] != 0xffffffffu && !vc_key_after(d, pko[top], pkl[top], ko, kl)) return false;
            pko[top] = ko; pkl[top] = kl;
            if (!vc_byte(w, ':')) return false;
        }
        w.fill();                                   // value
        if (w.have == 0) return false;
        c = w.peek(0);
        if (c == '"') { uint32_t n; if (!vc_quoted(w, true, &n)) return false; }
        else if (c == 't') { if (!vc_word(w, 0x65757274u, 4)) return false; }                 // true
        else if (c == 'f') { if (!vc_word(w, 0x736c6166u, 4) || !vc_byte(w, 'e')) return false; }   // false
        else if (c == 'n') { if (!vc_word(w, 0x6c6c756eu, 4)) return false; }                 // null
        else if (c == '-' || (c >= '0' && c <= '9')) { if (!vc_int(w, 15, true)) return false; }
        else if (c == '{' || c == '[') {
            if (depth == VC_MAX_DEPTH) return false;
            w.skip(1);
            is_obj = (is_obj & ~(1u << depth)) | ((c == '{' ? 1u : 0u) << depth);
            pkl[depth] = 0xffffffffu; pko[depth] = 0;
            ++depth; first = true;
        } else return false;
        continue;
    closed:
        if (--depth == 0) return true;
        first = false;
    }
}

// ---- capture for the audit (afc_vc_audit_stored_batch): the string spans the record's columns are compared with, and what the
// structure and compliance rules ask of @context and type.  Spans are string bodies as stored (escaped), offsets from the document
// start.  The first ten slots are in the order of the record's columns (AFC_AUDIT_COLUMNS).
enum VcCapSlot { CAP_ISSUER, CAP_EXECUTION_ID, CAP_WORKFLOW_ID, CAP_SESSION_ID, CAP_CALLER_DID, CAP_TARGET_DID, CAP_STATUS, CAP_INPUT_HASH,
                 CAP_OUTPUT_HASH, CAP_PROOF_VALUE, CAP_ID, CAP_ISSUANCE, VC_CAP_SPANS };
constexpr int VC_AUDIT_COLUMNS = 10;
constexpr int VC_CAP_FLAGS = 2 * VC_CAP_SPANS, VC_CAP_WORDS = 28;          // word 2k / 2k+1: offset / length of slot k; then flags; padding
enum : uint32_t {
    CAPF_CONTEXT_EMPTY = 1, CAPF_TYPE_EMPTY = 2,                             // the list is null or []
    CAPF_W3C = 4,                                                            // @context holds https://www.w3.org/2018/credentials/v1
    CAPF_VC = 8, CAPF_AF_EXECUTION = 16, CAPF_AF_WORKFLOW = 32               // type holds VerifiableCredential / AgentField{Execution,Workflow}Credential
};

// audit issue bits (include/afcrypto.h AFC_AUDIT_*): bit k < 10 = column k differs from the document
enum : uint32_t {
    AUD_INVALID_TIMESTAMP = 1u << 10, AUD_MISSING_CONTEXT = 1u << 11, AUD_MISSING_TYPE = 1u << 12, AUD_MISSING_ID = 1u << 13,
    AUD_MISSING_ISSUER = 1u << 14, AUD_MISSING_ISSUANCE_DATE = 1u << 15, AUD_NOT_W3C = 1u << 16, AUD_NOT_AGENTFIELD = 1u << 17,
    AUD_STATUS_UNDECIDED = 1u << 18, AUD_TIMESTAMP_UNDECIDED = 1u << 19
};

AFC_HD bool vc_bytes_are(const uint8_t* s, uint32_t n, const char* lit, uint32_t m) {
    if (n != m) return false;
    for (uint32_t j = 0; j < m; j++) if (s[j] != (uint8_t)lit[j]) return false;
    return true;
}
// The required literals need no escaping, so in a canonical document an element equals one iff its body is the literal's bytes.
AFC_HD uint32_t vc_list_literal(const uint8_t* s, uint32_t n, uint32_t which) {
    if (which == 0) return vc_bytes_are(s, n, "https://www.w3.org/2018/credentials/v1", 38) ? CAPF_W3C : 0;
    if (vc_bytes_are(s, n, "VerifiableCredential", 20)) return CAPF_VC;
    if (vc_bytes_are(s, n, "AgentFieldExecutionCredential", 29)) return CAPF_AF_EXECUTION;
    return vc_bytes_are(s, n, "AgentFieldWorkflowCredential", 28) ? CAPF_AF_WORKFLOW : 0;
}
// vc_strlist for @context (which = 0) and type (1), recording emptiness and the required literals in *flags
AFC_HD bool vc_strlist_capture(ByteWindow& w, const uint8_t* d, uint64_t len, uint32_t which, uint32_t* flags) {
    const uint32_t empty = which == 0 ? CAPF_CONTEXT_EMPTY : CAPF_TYPE_EMPTY;
    w.fill();
    if (w.have && w.peek(0) == 'n') { *flags |= empty; return vc_word(w, 0x6c6c756eu, 4); }
    if (!vc_byte(w, '[')) return false;
    w.fill();
    if (w.have && w.peek(0) == ']') { w.skip(1); *flags |= empty; return true; }
    for (;;) {
        uint32_t n;
        if (!vc_byte(w, '"')) return false;
        const uint32_t pos = (uint32_t)(len - w.rem);
        if (!vc_str(w, true, &n) || !vc_byte(w, '"')) return false;
        *flags |= vc_list_literal(d + pos, n, which);
        w.fill();
        if (w.have == 0) return false;
        const uint32_t c = w.peek(0);
        w.skip(1);
        if (c == ']') return true;
        if (c != ',') return false;
    }
}

// Walks one document through the schema.  The string spans are offsets from the document start.  With CAPTURE the walk also fills
// the VC_CAP_WORDS words at `cap` (a VOP_STR op whose len is k + 1 records its span in slot k), completely when the document is
// canonical (r.ok) and partly otherwise; without it `cap` is never touched.
template <bool CAPTURE>
AFC_HD void vc_parse_doc_t(const VcSchema& S, const uint8_t* d, uint64_t len, VcParse& r, uint32_t* cap) {
    r.ok = r.proof_at = r.iss_off = r.iss_len = r.date_off = r.date_len = r.pv_off = r.pv_len = 0;
    uint32_t lists = 0, flags = 0;
    if (len >= 0x7fffffffu) return;
    ByteWindow w; w.init(d, len);
    for (uint32_t i = 0; i < S.n_ops; i++) {
        const VcOp op = S.ops[i];
        const uint32_t pos = (uint32_t)(len - w.rem);
        uint32_t n;
        switch (op.code) {
        case VOP_LIT: if (!vc_lit(w, S.pool, op.off, op.len)) return; break;
        case VOP_STR:
            if (!vc_str(w, true, &n)) return;
            if (CAPTURE && op.len) { cap[2 * (op.len - 1)] = pos; cap[2 * (op.len - 1) + 1] = n; }
            break;
        case VOP_ISSUER: if (!vc_str(w, false, &n)) return; r.iss_off = pos; r.iss_len = n; break;
        case VOP_ISSUANCE: if (!vc_str(w, true, &n)) return; r.date_off = pos; r.date_len = n; break;
        case VOP_PROOFVALUE: if (!vc_str(w, false, &n)) return; r.pv_off = pos; r.pv_len = n; break;
        case VOP_STRLIST:
            if (CAPTURE && lists < 2) { if (!vc_strlist_capture(w, d, len, lists++, &flags)) return; }
            else if (!vc_strlist(w)) return;
            break;
        case VOP_INT: if (!vc_int(w, 18, false)) return; break;
        case VOP_ANY: if (!vc_any(w, d, len)) return; break;
        case VOP_PROOF: r.proof_at = pos; break;
        case VOP_OPT_STR:
        case VOP_OPT_STR_NE: {
            // present iff the first three bytes of the member text are there: enough to tell it from what may follow instead
            // (,"errorMessage" vs },"audit"; ,"endTime" vs ,"snapshotTime")
            w.fill();
            if (w.have < 3 || (((uint32_t)w.win ^ S.pool[op.off >> 2]) & 0xffffffu)) break;
            if (!vc_lit(w, S.pool, op.off, op.len) || !vc_str(w, true, &n) || !vc_byte(w, '"')) return;
            if (op.code == VOP_OPT_STR_NE && n == 0) return;                       // "" is omitted by omitempty
            break;
        }
        case VOP_END: if (w.rem) return; break;
        default: return;
        }
    }
    r.ok = 1;
    if (CAPTURE) {
        cap[2 * CAP_ISSUER] = r.iss_off; cap[2 * CAP_ISSUER + 1] = r.iss_len;
        cap[2 * CAP_ISSUANCE] = r.date_off; cap[2 * CAP_ISSUANCE + 1] = r.date_len;
        cap[2 * CAP_PROOF_VALUE] = r.pv_off; cap[2 * CAP_PROOF_VALUE + 1] = r.pv_len;
        for (int k = VC_CAP_FLAGS; k < VC_CAP_WORDS; k++) cap[k] = k == VC_CAP_FLAGS ? flags : 0;
    }
}
AFC_HD void vc_parse_doc(const VcSchema& S, const uint8_t* d, uint64_t len, VcParse& r) { vc_parse_doc_t<false>(S, d, len, r, nullptr); }

// ---- the cross-check of a captured document against its record (k_vc_crosscheck)

// Byte sink that compares what it is given with a span, a word at a time where it can
struct SpanMatch {
    ByteWindow w;
    bool ok;
    AFC_HDM void put(uint32_t b) {
        if (!ok) return;
        w.fill();
        if (w.have == 0 || w.peek(0) != b) { ok = false; return; }
        w.skip(1);
    }
    AFC_HDM void put4(uint32_t x) {
        if (!ok) return;
        w.fill();
        if (w.have < 4 || (uint32_t)w.win != x) { ok = false; return; }
        w.skip(4);
    }
};
// Unmarshal(span) == col, decided as go_json_escape(col) == span.  This is exact for every byte string col, invalid UTF-8 included:
// the parser accepted the span only in the encoder's own form (one spelling per string) and never with the escape of U+FFFD, so the
// span is the escape of exactly one valid UTF-8 string.  A valid col matches iff it is that string.  An invalid col escapes to text
// that holds the U+FFFD escape and so never matches, which is right: the unmarshalled span is valid UTF-8 and cannot equal it.
AFC_HD bool vc_column_equals(const uint8_t* span, uint32_t span_len, const uint8_t* col, uint64_t col_len) {
    if (col_len > span_len) return false;                       // escaping never shortens
    SpanMatch m; m.w.init(span, span_len); m.ok = true;
    go_json_escape(m, col, col_len);
    return m.ok && m.w.rem == 0;
}

// NormalizeExecutionStatus (pkg/types/status.go:51-63; services.normalize_execution_status) of a lower-cased, trimmed name in three
// little-endian words: 0 unknown, 1 pending, 2 queued, 3 running, 4 succeeded, 5 failed, 6 cancelled, 7 timeout
AFC_HD bool vc_name_is(uint32_t n, const uint32_t* b, const char* s, uint32_t m) {
    if (n != m) return false;
    uint32_t x[3] = {0, 0, 0};
    for (uint32_t j = 0; j < m; j++) x[j >> 2] |= (uint32_t)(uint8_t)s[j] << (8 * (j & 3));
    return x[0] == b[0] && x[1] == b[1] && x[2] == b[2];
}
AFC_HD uint32_t vc_status_id(uint32_t n, const uint32_t* b) {
    if (vc_name_is(n, b, "unknown", 7)) return 0;
    if (vc_name_is(n, b, "pending", 7)) return 1;
    if (vc_name_is(n, b, "queued", 6) || vc_name_is(n, b, "wait", 4) || vc_name_is(n, b, "waiting", 7)) return 2;
    if (vc_name_is(n, b, "running", 7) || vc_name_is(n, b, "in_progress", 11) || vc_name_is(n, b, "processing", 10)) return 3;
    if (vc_name_is(n, b, "succeeded", 9) || vc_name_is(n, b, "success", 7) || vc_name_is(n, b, "successful", 10) ||
        vc_name_is(n, b, "completed", 9) || vc_name_is(n, b, "complete", 8) || vc_name_is(n, b, "done", 4) || vc_name_is(n, b, "ok", 2)) return 4;
    if (vc_name_is(n, b, "failed", 6) || vc_name_is(n, b, "error", 5) || vc_name_is(n, b, "failure", 7) || vc_name_is(n, b, "errored", 7)) return 5;
    if (vc_name_is(n, b, "cancelled", 9) || vc_name_is(n, b, "canceled", 8) || vc_name_is(n, b, "cancel", 6)) return 6;
    if (vc_name_is(n, b, "timeout", 7) || vc_name_is(n, b, "timed_out", 9)) return 7;
    return 0;
}
constexpr uint32_t VC_UNDECIDED = 0xffu;
// The status class of a document span (is_span) or a column, or VC_UNDECIDED.  Decided only for printable ASCII (and, in a column,
// \t \n \v \f \r), without backslashes in the span: there Go's TrimSpace / ToLower and Python's strip / lower agree.  Python also strips
// U+001C-U+001F and both lower-case some non-ASCII letters (the Kelvin sign), so those inputs are left to the host mirror.
AFC_HD uint32_t vc_status_class(const uint8_t* s, uint64_t n, bool is_span) {
    uint64_t lo = 0, hi = n;
    for (uint64_t j = 0; j < n; j++) {
        const uint32_t c = s[j];
        const bool ws = c == ' ' || (c >= 0x09 && c <= 0x0d);
        if (!((c >= 0x20 && c <= 0x7e) || (!is_span && ws)) || (is_span && c == '\\')) return VC_UNDECIDED;
    }
    while (lo < hi && (s[lo] == ' ' || (s[lo] >= 0x09 && s[lo] <= 0x0d))) ++lo;
    while (hi > lo && (s[hi - 1] == ' ' || (s[hi - 1] >= 0x09 && s[hi - 1] <= 0x0d))) --hi;
    if (hi - lo > 11) return 0;                                  // longer than every name: unknown
    uint32_t b[3] = {0, 0, 0};
    for (uint64_t j = lo; j < hi; j++) {
        uint32_t c = s[j];
        if (c >= 'A' && c <= 'Z') c += 32;
        b[(j - lo) >> 2] |= c << (8 * ((j - lo) & 3));
    }
    return vc_status_id((uint32_t)(hi - lo), b);
}

// services._is_rfc3339 on an issuanceDate span: 0 valid, 1 invalid, VC_UNDECIDED for a byte >= 0x80 (Python's \d also matches
// non-ASCII digits).  A backslash in an ASCII span means invalid: no escaped character belongs to the grammar.
// Grammar: DDDD-DD-DDTDD:DD:DD(.D+)?(Z|[+-]DD:DD), month 1-12, day 1-(days of the month, Gregorian leap years), hour <= 23,
// minute and second <= 59, offset hour <= 23 and minute <= 59.
AFC_HD uint32_t vc_d2(const uint8_t* s, uint32_t j) {
    const uint32_t a = s[j] - '0', b = s[j + 1] - '0';
    return a <= 9 && b <= 9 ? 10 * a + b : 100;
}
AFC_HD uint32_t vc_rfc3339(const uint8_t* s, uint32_t n) {
    bool esc = false;
    for (uint32_t j = 0; j < n; j++) {
        if (s[j] >= 0x80) return VC_UNDECIDED;
        esc |= s[j] == '\\';
    }
    if (esc || n < 20) return 1;
    const uint32_t y0 = vc_d2(s, 0), y1 = vc_d2(s, 2), mo = vc_d2(s, 5), d = vc_d2(s, 8), h = vc_d2(s, 11), mi = vc_d2(s, 14), sec = vc_d2(s, 17);
    if (y0 > 99 || y1 > 99 || s[4] != '-' || s[7] != '-' || s[10] != 'T' || s[13] != ':' || s[16] != ':') return 1;
    if (mo < 1 || mo > 12 || d < 1 || h > 23 || mi > 59 || sec > 59) return 1;
    uint32_t j = 19;
    if (s[j] == '.') {
        const uint32_t f = ++j;
        while (j < n && s[j] >= '0' && s[j] <= '9') ++j;
        if (j == f) return 1;
    }
    if (j >= n) return 1;
    if (s[j] == 'Z') { if (j + 1 != n) return 1; }
    else if (s[j] == '+' || s[j] == '-') {
        if (j + 6 != n || s[j + 3] != ':') return 1;
        const uint32_t oh = vc_d2(s, j + 1), om = vc_d2(s, j + 4);
        if (oh > 23 || om > 59) return 1;
    } else return 1;
    const uint32_t year = 100 * y0 + y1;
    const bool leap = year % 4 == 0 && (year % 100 != 0 || year % 400 == 0);
    const uint32_t mdays = mo == 2 ? (leap ? 29u : 28u) : (mo == 4 || mo == 6 || mo == 9 || mo == 11) ? 30u : 31u;
    return d <= mdays ? 0 : 1;
}

// The issue mask of one canonical document (its capture) against its record.  col_off: this record's AFC_AUDIT_COLUMNS + 1 absolute
// offsets into cols (execution documents only).  For workflow documents only the AgentField type rule (checkWorkflowVCCompliance,
// vc_service.go:1628-1644) is defined.
AFC_HD uint32_t vc_audit_mask(int kind, const uint8_t* d, const uint32_t* cap, const uint8_t* cols, const uint64_t* col_off) {
    const uint32_t f = cap[VC_CAP_FLAGS];
    if (kind == VC_DOC_WORKFLOW) return (f & CAPF_VC) && (f & CAPF_AF_WORKFLOW) ? 0 : AUD_NOT_AGENTFIELD;
    uint32_t m = 0;
#pragma unroll 1
    for (uint32_t k = 0; k < VC_AUDIT_COLUMNS; k++) {
        const uint64_t c0 = col_off[k], cl = col_off[k + 1] - c0;
        const uint8_t* s = d + cap[2 * k];
        const uint32_t sl = cap[2 * k + 1];
        if (k == CAP_STATUS) {
            const uint32_t a = vc_status_class(s, sl, true), b = vc_status_class(cols + c0, cl, false);
            if (a == VC_UNDECIDED || b == VC_UNDECIDED) m |= AUD_STATUS_UNDECIDED;
            else if (a != b) m |= 1u << k;
        } else if (!vc_column_equals(s, sl, cols + c0, cl)) {
            m |= 1u << k;
        }
    }
    const uint32_t t = vc_rfc3339(d + cap[2 * CAP_ISSUANCE], cap[2 * CAP_ISSUANCE + 1]);
    if (t == VC_UNDECIDED) m |= AUD_TIMESTAMP_UNDECIDED;
    else if (t) m |= AUD_INVALID_TIMESTAMP;
    if (f & CAPF_CONTEXT_EMPTY) m |= AUD_MISSING_CONTEXT;
    if (f & CAPF_TYPE_EMPTY) m |= AUD_MISSING_TYPE;
    if (cap[2 * CAP_ID + 1] == 0) m |= AUD_MISSING_ID;
    if (cap[2 * CAP_ISSUER + 1] == 0) m |= AUD_MISSING_ISSUER;
    if (cap[2 * CAP_ISSUANCE + 1] == 0) m |= AUD_MISSING_ISSUANCE_DATE;
    if (!(f & CAPF_W3C)) m |= AUD_NOT_W3C;
    if (!((f & CAPF_VC) && (f & CAPF_AF_EXECUTION))) m |= AUD_NOT_AGENTFIELD;
    return m;
}

// base64.RawURLEncoding.DecodeString of the proofValue span (lenient trailing bits, as Go's default decoder): VC_BAD_ENCODING for
// a character outside A-Za-z0-9-_ or a length = 1 (mod 4), VC_INVALID for a decoded length other than 64, else VC_VALID with the
// 64 bytes written as 16 little-endian words to sig (a candidate for verification).
AFC_HD uint32_t vc_b64_signature(const uint8_t* s, uint32_t len, uint32_t* sig) {
    ByteWindow w; w.init(s, len);
    const bool store = len == 86;
    uint32_t acc = 0, bits = 0, o = 0, word = 0;
    while (w.rem) {
        w.fill();
        const uint32_t c = w.peek(0);
        w.skip(1);
        uint32_t v;
        if (c >= 'A' && c <= 'Z') v = c - 'A';
        else if (c >= 'a' && c <= 'z') v = c - 'a' + 26;
        else if (c >= '0' && c <= '9') v = c - '0' + 52;
        else if (c == '-') v = 62;
        else if (c == '_') v = 63;
        else return VC_BAD_ENCODING;
        acc = (acc << 6) | v; bits += 6;
        if (bits >= 8) {
            bits -= 8;
            if (store && o < 64) {
                word |= ((acc >> bits) & 0xffu) << (8 * (o & 3));
                if ((o & 3) == 3) { sig[o >> 2] = word; word = 0; }
            }
            ++o;
        }
    }
    if ((len & 3) == 1) return VC_BAD_ENCODING;
    return store ? VC_VALID : VC_INVALID;
}

// FNV-1a over the DID bytes: the key set's table and the lookup agree on it
AFC_HD uint32_t vc_did_hash_byte(uint32_t h, uint32_t b) { return (h ^ b) * 16777619u; }

#if !AFC_DEVICE_CODE
// ---- the two schemas (host side: built once, copied to the device by afcrypto.cu, used directly by tests/hostsim) ----------
// VCDocument and WorkflowVCDocument, pkg/types/did_types.go:135-220, as json.Marshal writes them; the literal text is that of
// canonical.vc_document_template_parts(True) / workflow_vc_document_template_parts(True).
struct VcStep { uint8_t code; const char* lit; uint8_t cap; };   // cap: audit capture slot + 1 of a VOP_STR (0: none)
static const VcStep kVcExecutionSteps[] = {
    {VOP_LIT, "{\"@context\":"}, {VOP_STRLIST, nullptr}, {VOP_LIT, ",\"type\":"}, {VOP_STRLIST, nullptr},
    {VOP_LIT, ",\"id\":\""}, {VOP_STR, nullptr, CAP_ID + 1}, {VOP_LIT, "\",\"issuer\":\""}, {VOP_ISSUER, nullptr},
    {VOP_LIT, "\",\"issuanceDate\":\""}, {VOP_ISSUANCE, nullptr},
    {VOP_LIT, "\",\"credentialSubject\":{\"executionId\":\""}, {VOP_STR, nullptr, CAP_EXECUTION_ID + 1}, {VOP_LIT, "\",\"workflowId\":\""}, {VOP_STR, nullptr, CAP_WORKFLOW_ID + 1},
    {VOP_LIT, "\",\"sessionId\":\""}, {VOP_STR, nullptr, CAP_SESSION_ID + 1}, {VOP_LIT, "\",\"caller\":{\"did\":\""}, {VOP_STR, nullptr, CAP_CALLER_DID + 1},
    {VOP_LIT, "\",\"type\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"agentNodeDid\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\"},\"target\":{\"did\":\""}, {VOP_STR, nullptr, CAP_TARGET_DID + 1}, {VOP_LIT, "\",\"agentNodeDid\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"functionName\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\"},\"execution\":{\"inputHash\":\""}, {VOP_STR, nullptr, CAP_INPUT_HASH + 1},
    {VOP_LIT, "\",\"outputHash\":\""}, {VOP_STR, nullptr, CAP_OUTPUT_HASH + 1}, {VOP_LIT, "\",\"timestamp\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"durationMs\":"}, {VOP_INT, nullptr}, {VOP_LIT, ",\"status\":\""}, {VOP_STR, nullptr, CAP_STATUS + 1}, {VOP_LIT, "\""},
    {VOP_OPT_STR_NE, ",\"errorMessage\":\""},
    {VOP_LIT, "},\"audit\":{\"inputDataHash\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"outputDataHash\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"metadata\":"}, {VOP_ANY, nullptr},
    {VOP_LIT, "}},\"proof\":"}, {VOP_PROOF, nullptr}, {VOP_LIT, "{\"type\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"created\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"verificationMethod\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"proofPurpose\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"proofValue\":\""}, {VOP_PROOFVALUE, nullptr},
    {VOP_LIT, "\"}}"}, {VOP_END, nullptr}};
static const VcStep kVcWorkflowSteps[] = {
    {VOP_LIT, "{\"@context\":"}, {VOP_STRLIST, nullptr}, {VOP_LIT, ",\"type\":"}, {VOP_STRLIST, nullptr},
    {VOP_LIT, ",\"id\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"issuer\":\""}, {VOP_ISSUER, nullptr},
    {VOP_LIT, "\",\"issuanceDate\":\""}, {VOP_ISSUANCE, nullptr},
    {VOP_LIT, "\",\"credentialSubject\":{\"workflowId\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"sessionId\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"componentVcIds\":"}, {VOP_STRLIST, nullptr}, {VOP_LIT, ",\"totalSteps\":"}, {VOP_INT, nullptr},
    {VOP_LIT, ",\"completedSteps\":"}, {VOP_INT, nullptr}, {VOP_LIT, ",\"status\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"startTime\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\""}, {VOP_OPT_STR, ",\"endTime\":\""},
    {VOP_LIT, ",\"snapshotTime\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"orchestrator\":{\"did\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"type\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"agentNodeDid\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\"},\"audit\":{\"inputDataHash\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"outputDataHash\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"metadata\":"}, {VOP_ANY, nullptr},
    {VOP_LIT, "}},\"proof\":"}, {VOP_PROOF, nullptr}, {VOP_LIT, "{\"type\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"created\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"verificationMethod\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"proofPurpose\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"proofValue\":\""}, {VOP_PROOFVALUE, nullptr},
    {VOP_LIT, "\"}}"}, {VOP_END, nullptr}};
// what follows "proof": in the message the reference verifies: json.Marshal(VCProof{}) and the document's closing brace
static const char kVcZeroProofTail[] = "{\"type\":\"\",\"created\":\"\",\"verificationMethod\":\"\",\"proofPurpose\":\"\",\"proofValue\":\"\"}}";

static inline uint32_t vc_pool_add(VcSchema& s, uint32_t& used, const char* t) {
    const uint32_t off = used, n = (uint32_t)strlen(t);
    uint8_t* p = (uint8_t*)s.pool;
    if (off + n <= sizeof(s.pool)) memcpy(p + off, t, n);
    used = (off + n + 3) & ~3u;
    return off;
}
// 0 on success, -1 for an unknown kind
static inline int vc_schema_build(int kind, VcSchema* s) {
    const VcStep* st; uint32_t n;
    if (kind == VC_DOC_EXECUTION) { st = kVcExecutionSteps; n = sizeof(kVcExecutionSteps) / sizeof(VcStep); }
    else if (kind == VC_DOC_WORKFLOW) { st = kVcWorkflowSteps; n = sizeof(kVcWorkflowSteps) / sizeof(VcStep); }
    else return -1;
    if (n > (uint32_t)VC_MAX_OPS) return -1;
    memset(s, 0, sizeof(*s));
    uint32_t used = 0;
    for (uint32_t i = 0; i < n; i++) {
        VcOp& op = s->ops[i];
        op.code = st[i].code;
        if (st[i].lit) { op.len = (uint8_t)strlen(st[i].lit); op.off = (uint16_t)vc_pool_add(*s, used, st[i].lit); }
        if (st[i].code == VOP_STR && st[i].cap) op.len = st[i].cap;          // read only by the capturing walk
    }
    s->n_ops = n;
    s->tail_len = (uint32_t)strlen(kVcZeroProofTail);
    s->tail_off = vc_pool_add(*s, used, kVcZeroProofTail);
    return n <= (uint32_t)VC_MAX_OPS && used <= sizeof(s->pool) ? 0 : -1;
}
#endif

}  // namespace afc
