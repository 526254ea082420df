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

// Walks one document through the schema.  The string spans are offsets from the document start.
AFC_HD void vc_parse_doc(const VcSchema& S, const uint8_t* d, uint64_t len, VcParse& r) {
    r.ok = r.proof_at = r.iss_off = r.iss_len = r.date_off = r.date_len = r.pv_off = r.pv_len = 0;
    if (len >= 0x7fffffffu) return;
    ByteWindow w; w.init(d, len);
    for (uint32_t i = 0; i < S.n_ops; i++) {
        const VcOp op = S.ops[i];
        const uint32_t pos = (uint32_t)(len - w.rem);
        uint32_t n;
        switch (op.code) {
        case VOP_LIT: if (!vc_lit(w, S.pool, op.off, op.len)) return; break;
        case VOP_STR: if (!vc_str(w, true, &n)) return; break;
        case VOP_ISSUER: if (!vc_str(w, false, &n)) return; r.iss_off = pos; r.iss_len = n; break;
        case VOP_ISSUANCE: if (!vc_str(w, true, &n)) return; r.date_off = pos; r.date_len = n; break;
        case VOP_PROOFVALUE: if (!vc_str(w, false, &n)) return; r.pv_off = pos; r.pv_len = n; break;
        case VOP_STRLIST: if (!vc_strlist(w)) return; break;
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
struct VcStep { uint8_t code; const char* lit; };
static const VcStep kVcExecutionSteps[] = {
    {VOP_LIT, "{\"@context\":"}, {VOP_STRLIST, nullptr}, {VOP_LIT, ",\"type\":"}, {VOP_STRLIST, nullptr},
    {VOP_LIT, ",\"id\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"issuer\":\""}, {VOP_ISSUER, nullptr},
    {VOP_LIT, "\",\"issuanceDate\":\""}, {VOP_ISSUANCE, nullptr},
    {VOP_LIT, "\",\"credentialSubject\":{\"executionId\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"workflowId\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"sessionId\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"caller\":{\"did\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"type\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"agentNodeDid\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\"},\"target\":{\"did\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"agentNodeDid\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"functionName\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\"},\"execution\":{\"inputHash\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"outputHash\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\",\"timestamp\":\""}, {VOP_STR, nullptr},
    {VOP_LIT, "\",\"durationMs\":"}, {VOP_INT, nullptr}, {VOP_LIT, ",\"status\":\""}, {VOP_STR, nullptr}, {VOP_LIT, "\""},
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
    }
    s->n_ops = n;
    s->tail_len = (uint32_t)strlen(kVcZeroProofTail);
    s->tail_off = vc_pool_add(*s, used, kVcZeroProofTail);
    return n <= (uint32_t)VC_MAX_OPS && used <= sizeof(s->pool) ? 0 : -1;
}
#endif

}  // namespace afc
