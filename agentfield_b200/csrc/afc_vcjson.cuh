// Credential documents in any JSON spelling, re-marshalled on the device (afc_vc_verify_json_batch, include/afcrypto.h).
//
// VCService.VerifyVC (internal/services/vc_service.go:242-289, 469-505) verifies json.Marshal(json.Unmarshal(D)) with a zero proof, so
// its verdict does not depend on how D is spelled.  afc_vcdoc.cuh proves that D is already what json.Marshal writes; this header
// is the tolerant walk of the same schema programs (kVcExecutionSteps / kVcWorkflowSteps) for the spellings clients produce —
// Python's json.dumps, JavaScript's JSON.stringify, pretty-printed files — and writes Go's canonical text of the document into a
// sink while it reads it:
//   literals       matched token by token; JSON whitespace (0x20 0x09 0x0A 0x0D) may precede every byte outside a quoted name
//                  (VcjSchema::ws, precomputed on the host); member names are exact bytes; the literal's canonical text is written
//   strings        escapes decoded on the fly (every JSON escape, \uXXXX in either case, surrogate pairs), each code point written back
//                  with Go's rules (vcj_put_cp); plain runs copied four bytes at a time
//   int members    -?(0|[1-9][0-9]*), at most 18 digits, written as Go does (-0 -> 0)
//   metadata       strings, true / false / null, integers float64 writes back unchanged (-?(0|[1-9][0-9]{0,14}), -0 kept), arrays and
//                  objects up to VC_MAX_DEPTH; keys without backslashes, strictly increasing by bytes, written through Go's escaper
//   omitempty      "errorMessage":"" is dropped, "endTime":null is dropped, "endTime":"" is written
// Everything else is VC_HOST (never a guess): other member orders, missing / unknown / duplicate / re-cased / escaped names, null for
// a string, anything that is not JSON (BOM, NaN, trailing commas, raw control bytes, leading zeros), fractions and exponents, depth
// beyond VC_MAX_DEPTH, an escape in issuer or proofValue, raw invalid UTF-8, lone surrogate escapes, and a canonical message longer
// than the document.  The last bound keeps the message buffer of afc_vc_verify_stored_batch: the proof object the message drops
// leaves a few hundred bytes of slack.
//
// One walk, two sinks: ByteCounter in the sizes pass (k_vcj_parse), ByteWriter in the emit pass (k_vcj_emit), so the length the
// first reports and the bytes the second writes come from the same code.  Shared by k_vcjson.cu and the CPU build in tests/hostsim.
#pragma once
#include "afc_vcdoc.cuh"

namespace afc {

// A VcSchema plus, per op, where whitespace may stand in its literal: bit j of ws[i] = JSON whitespace may precede byte j
struct VcjSchema {
    VcSchema s;
    uint64_t ws[VC_MAX_OPS];
};
constexpr uint32_t VCJ_MAX_LIT = 64;

struct VcjParse {
    uint32_t ok;                          // 1 = the document was read and re-marshalled
    uint32_t prefix;                      // length of the canonical text up to "proof": (sizes pass only)
    uint32_t iss_off, iss_len, date_off, date_len, pv_off, pv_len;   // string bodies in the input document
};

AFC_HD bool vcj_is_ws(uint32_t c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }
// skips JSON whitespace; leaves the window filled
AFC_HD void vcj_skip_ws(ByteWindow& w) {
    for (;;) {
        w.fill();
        if (w.have >= 4 && (uint32_t)w.win == 0x20202020u) { w.skip(4); continue; }
        if (w.have == 0 || !vcj_is_ws(w.peek(0))) return;
        w.skip(1);
    }
}

AFC_HD uint32_t vcj_ctz64(uint64_t x) {          // x != 0
#if AFC_DEVICE_CODE
    return (uint32_t)__ffsll((long long)x) - 1u;
#else
    return (uint32_t)__builtin_ctzll(x);
#endif
}
// four pool bytes starting at byte b (any alignment)
AFC_HD uint32_t vcj_pool_word(const uint32_t* pool, uint32_t b) {
    const uint32_t k = b >> 2, s = (b & 3) * 8;
    return s ? (pool[k] >> s) | (pool[k + 1] << (32 - s)) : pool[k];
}
// the pool literal at byte `off`, `len` bytes, with whitespace allowed before byte j where bit j of ws is set
AFC_HD bool vcj_lit(ByteWindow& w, const uint32_t* pool, uint32_t off, uint32_t len, uint64_t ws) {
    uint32_t j = 0;
    while (j < len) {
        if ((ws >> j) & 1) vcj_skip_ws(w);
        // the run up to the next byte whitespace may precede is compared a word at a time
        const uint64_t later = j + 1 < 64 ? ws >> (j + 1) : 0;
        uint32_t end = later ? j + 1 + vcj_ctz64(later) : len;
        if (end > len) end = len;
        while (j < end) {
            const uint32_t m = end - j < 4 ? end - j : 4;
            w.fill();
            if (w.have < m || (((uint32_t)w.win ^ vcj_pool_word(pool, off + j)) & vc_mask(m))) return false;
            w.skip(m); j += m;
        }
    }
    return true;
}
template <class Sink>
AFC_HD void vcj_put_lit(Sink& out, const uint32_t* pool, uint32_t off, uint32_t len) {
    uint32_t k = 0;
    for (; k + 4 <= len; k += 4) out.put4(pool[(off + k) >> 2]);
    for (; k < len; k++) out.put((pool[(off + k) >> 2] >> (8 * ((off + k) & 3))) & 0xffu);
}

// One code point (a Unicode scalar value) as Go's encoder writes it (encode.go appendString with escapeHTML): short escapes for
// " \ and \b \f \n \r \t, backslash-u 00xx for the other control characters and for < > &, backslash-u 2028 / 2029 for U+2028 /
// U+2029, everything else as UTF-8.  The rules of go_json_escape (afc_json.cuh), which works on bytes; the CPU build checks the two
// against each other.
template <class Sink>
AFC_HD void vcj_put_cp(Sink& out, uint32_t cp) {
    if (cp < 0x80) {
        if (cp >= 0x20 && cp != '"' && cp != '\\' && cp != '<' && cp != '>' && cp != '&') { out.put(cp); return; }
        out.put('\\');
        uint32_t c = 0;
        switch (cp) {
        case '"': case '\\': c = cp; break;
        case '\b': c = 'b'; break;
        case '\f': c = 'f'; break;
        case '\n': c = 'n'; break;
        case '\r': c = 'r'; break;
        case '\t': c = 't'; break;
        default: break;
        }
        if (c) out.put(c);
        else { out.put('u'); out.put('0'); out.put('0'); out.put(json_hex_digit(cp >> 4)); out.put(json_hex_digit(cp & 15)); }
        return;
    }
    if (cp < 0x800) { out.put(0xC0 | (cp >> 6)); out.put(0x80 | (cp & 63)); return; }
    if (cp == 0x2028 || cp == 0x2029) { out.put('\\'); out.put('u'); out.put('2'); out.put('0'); out.put('2'); out.put(json_hex_digit(cp & 15)); return; }
    if (cp < 0x10000) { out.put(0xE0 | (cp >> 12)); out.put(0x80 | ((cp >> 6) & 63)); out.put(0x80 | (cp & 63)); return; }
    out.put(0xF0 | (cp >> 18)); out.put(0x80 | ((cp >> 12) & 63)); out.put(0x80 | ((cp >> 6) & 63)); out.put(0x80 | (cp & 63));
}

AFC_HD uint32_t vcj_hex(uint32_t c) {             // the digit's value, or 16
    if (c >= '0' && c <= '9') return c - '0';
    c |= 0x20;
    return c >= 'a' && c <= 'f' ? c - 'a' + 10 : 16;
}
// the four hex digits after \u (either case) -> their value (consumed), or 0xffffffff
AFC_HD uint32_t vcj_u4(ByteWindow& w) {
    w.fill();
    if (w.have < 4) return 0xffffffffu;
    const uint32_t a = vcj_hex(w.peek(0)), b = vcj_hex(w.peek(1)), c = vcj_hex(w.peek(2)), d = vcj_hex(w.peek(3));
    if ((a | b | c | d) & 16) return 0xffffffffu;
    w.skip(4);
    return (a << 12) | (b << 8) | (c << 4) | d;
}

// A string body up to (not including) its closing quote, decoded and written back in Go's form.  allow_escape = false: a backslash
// declines (issuer, proofValue and metadata keys, whose input bytes are used as the value).
template <class Sink>
AFC_HD bool vcj_str(ByteWindow& w, Sink& out, bool allow_escape) {
    for (;;) {
        w.fill();
        if (w.have >= 4 && json_word_is_plain((uint32_t)w.win)) { out.put4((uint32_t)w.win); w.skip(4); continue; }
        if (w.have == 0) return false;
        const uint32_t b = w.peek(0);
        if (b == '"') return true;
        if (b < 0x20) return false;                                           // raw control byte: not JSON
        if (b == '\\') {
            if (!allow_escape || w.have < 2) return false;
            const uint32_t e = w.peek(1);
            w.skip(2);
            uint32_t cp;
            switch (e) {
            case '"': case '\\': case '/': cp = e; break;
            case 'b': cp = '\b'; break;
            case 'f': cp = '\f'; break;
            case 'n': cp = '\n'; break;
            case 'r': cp = '\r'; break;
            case 't': cp = '\t'; break;
            case 'u':
                cp = vcj_u4(w);
                if (cp == 0xffffffffu || (cp >= 0xDC00 && cp < 0xE000)) return false;     // lone low surrogate
                if (cp >= 0xD800 && cp < 0xDC00) {                                      // a high surrogate needs its low half
                    w.fill();
                    if (w.have < 2 || w.peek(0) != '\\' || w.peek(1) != 'u') return false;
                    w.skip(2);
                    const uint32_t lo = vcj_u4(w);
                    if (lo < 0xDC00 || lo >= 0xE000) return false;
                    cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
                }
                break;
            default: return false;
            }
            vcj_put_cp(out, cp);
            continue;
        }
        if (b < 0x80) { vcj_put_cp(out, b); w.skip(1); continue; }
        const uint32_t k = utf8_valid_len(w, w.rem);
        if (k == 0) return false;                                             // raw invalid UTF-8: left to the host
        if (k == 3 && b == 0xE2 && w.peek(1) == 0x80 && (w.peek(2) == 0xA8 || w.peek(2) == 0xA9)) {
            vcj_put_cp(out, 0x2028u | (w.peek(2) & 1));
            w.skip(3);
            continue;
        }
        for (uint32_t j = 0; j < k; j++) out.put(w.peek(j));
        w.skip(k);
    }
}
// "..." after optional whitespace, written back with its quotes
template <class Sink>
AFC_HD bool vcj_quoted(ByteWindow& w, Sink& out, bool allow_escape) {
    vcj_skip_ws(w);
    if (!vc_byte(w, '"')) return false;
    out.put('"');
    if (!vcj_str(w, out, allow_escape)) return false;
    w.skip(1);
    out.put('"');
    return true;
}

// -?(0|[1-9][0-9]*) with at most max_digits digits after optional whitespace; -0 is written as -0 (keep_neg_zero, a float64) or 0
// (a Go int).  What follows is checked by the caller.
template <class Sink>
AFC_HD bool vcj_int(ByteWindow& w, Sink& out, uint32_t max_digits, bool keep_neg_zero) {
    vcj_skip_ws(w);
    if (w.have == 0) return false;
    const bool neg = w.peek(0) == '-';
    if (neg) { w.skip(1); w.fill(); if (w.have == 0) return false; }
    uint32_t d = w.peek(0);
    if (d < '0' || d > '9') return false;
    if (d == '0') {
        w.skip(1);
        if (neg && keep_neg_zero) out.put('-');
        out.put('0');
        return true;
    }
    if (neg) out.put('-');
    uint32_t count = 0;
    while (w.have && (d = w.peek(0)) >= '0' && d <= '9') {
        if (++count > max_digits) return false;
        out.put(d);
        w.skip(1); w.fill();
    }
    return true;
}

// the 4-byte word x (null / true / fals) after optional whitespace, written back
template <class Sink>
AFC_HD bool vcj_word(ByteWindow& w, Sink& out, uint32_t x) {
    vcj_skip_ws(w);
    if (!vc_word(w, x, 4)) return false;
    out.put4(x);
    return true;
}
constexpr uint32_t VCJ_NULL = 0x6c6c756eu, VCJ_TRUE = 0x65757274u, VCJ_FALS = 0x736c6166u;

// []string: null or [ "..." , ... ]
template <class Sink>
AFC_HD bool vcj_strlist(ByteWindow& w, Sink& out) {
    vcj_skip_ws(w);
    if (w.have && w.peek(0) == 'n') return vcj_word(w, out, VCJ_NULL);
    if (!vc_byte(w, '[')) return false;
    out.put('[');
    vcj_skip_ws(w);
    if (w.have && w.peek(0) == ']') { w.skip(1); out.put(']'); return true; }
    for (;;) {
        if (!vcj_quoted(w, out, true)) return false;
        vcj_skip_ws(w);
        if (w.have == 0) return false;
        const uint32_t c = w.peek(0);
        if (c != ']' && c != ',') return false;
        w.skip(1);
        out.put(c);
        if (c == ']') return true;
    }
}

// map[string]interface{} (metadata): the rules of vc_any, with whitespace between tokens and escapes in values
template <class Sink>
AFC_HD bool vcj_any(ByteWindow& w, Sink& out, const uint8_t* d, uint64_t len) {
    vcj_skip_ws(w);
    if (w.have && w.peek(0) == 'n') return vcj_word(w, out, VCJ_NULL);
    if (!vc_byte(w, '{')) return false;
    out.put('{');
    uint32_t is_obj = 1, depth = 1;                // bit k of is_obj: container k is an object
    uint32_t pko[VC_MAX_DEPTH], pkl[VC_MAX_DEPTH];  // previous key of each open object (pkl = 0xffffffff: none yet)
    pkl[0] = 0xffffffffu; pko[0] = 0;
    bool first = true;                              // just after an opening bracket
    for (;;) {
        const uint32_t top = depth - 1;
        const bool obj = (is_obj >> top) & 1;
        const uint32_t close = obj ? '}' : ']';
        vcj_skip_ws(w);
        if (w.have == 0) return false;
        uint32_t c = w.peek(0);
        if (c == close && first) { w.skip(1); out.put(c); goto closed; }
        if (!first) {                               // after a value: separator or close
            w.skip(1);
            if (c == close) { out.put(c); goto closed; }
            if (c != ',') return false;
            out.put(',');
        }
        first = false;
        if (obj) {                                  // key: no escapes, so its input bytes are the key Go sorts by
            vcj_skip_ws(w);
            const uint32_t ko = (uint32_t)(len - w.rem) + 1;
            if (!vcj_quoted(w, out, false)) return false;
            const uint32_t kl = (uint32_t)(len - w.rem) - 1 - ko;
            if (pkl[top] != 0xffffffffu && !vc_key_after(d, pko[top], pkl[top], ko, kl)) return false;
            pko[top] = ko; pkl[top] = kl;
            vcj_skip_ws(w);
            if (!vc_byte(w, ':')) return false;
            out.put(':');
        }
        vcj_skip_ws(w);                             // value
        if (w.have == 0) return false;
        c = w.peek(0);
        if (c == '"') { if (!vcj_quoted(w, out, true)) return false; }
        else if (c == 't') { if (!vcj_word(w, out, VCJ_TRUE)) return false; }
        else if (c == 'f') { if (!vcj_word(w, out, VCJ_FALS) || !vc_byte(w, 'e')) return false; out.put('e'); }
        else if (c == 'n') { if (!vcj_word(w, out, VCJ_NULL)) return false; }
        else if (c == '-' || (c >= '0' && c <= '9')) { if (!vcj_int(w, out, 15, true)) return false; }
        else if (c == '{' || c == '[') {
            if (depth == VC_MAX_DEPTH) return false;
            w.skip(1);
            out.put(c);
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

// Walks one document through the schema and writes its canonical text to `out`.  SIZES (the sizes pass): the whole document is
// checked, r.prefix is the length of the text up to "proof": and r.ok says whether the document is accepted; the sink also sees
// what the proof members write, which r.prefix leaves out.  Otherwise (the emit pass, over a document the sizes pass accepted) the
// walk stops at "proof":.
template <bool SIZES, class Sink>
AFC_HD void vcj_walk(const VcjSchema& S, const uint8_t* d, uint64_t len, Sink& out, VcjParse& r) {
    r.ok = r.prefix = r.iss_off = r.iss_len = r.date_off = r.date_len = r.pv_off = r.pv_len = 0;
    if (len >= 0x7fffffffu) return;
    const uint32_t* pool = S.s.pool;
    ByteWindow w; w.init(d, len);
    for (uint32_t i = 0; i < S.s.n_ops; i++) {
        const VcOp op = S.s.ops[i];
        const uint32_t pos = (uint32_t)(len - w.rem);
        switch (op.code) {
        case VOP_LIT:
            if (!vcj_lit(w, pool, op.off, op.len, S.ws[i])) return;
            vcj_put_lit(out, pool, op.off, op.len);
            break;
        case VOP_STR: if (!vcj_str(w, out, true)) return; break;
        case VOP_ISSUER: if (!vcj_str(w, out, false)) return; r.iss_off = pos; r.iss_len = (uint32_t)(len - w.rem) - pos; break;
        case VOP_ISSUANCE: if (!vcj_str(w, out, true)) return; r.date_off = pos; r.date_len = (uint32_t)(len - w.rem) - pos; break;
        case VOP_PROOFVALUE: if (!vcj_str(w, out, false)) return; r.pv_off = pos; r.pv_len = (uint32_t)(len - w.rem) - pos; break;
        case VOP_STRLIST: if (!vcj_strlist(w, out)) return; break;
        case VOP_INT: if (!vcj_int(w, out, 18, false)) return; break;
        case VOP_ANY: if (!vcj_any(w, out, d, len)) return; break;
        case VOP_PROOF:
            if (!SIZES) { r.ok = 1; return; }
            // the message (prefix + zero-proof tail) must fit in the document's own bytes; decided on the 64-bit count, which
            // re-escaping can push past 2^32 for a document of under 2 GB (a raw '<' becomes six bytes)
            if (out.n + S.s.tail_len > len) return;
            r.prefix = (uint32_t)out.n;
            break;
        case VOP_OPT_STR:
        case VOP_OPT_STR_NE: {
            // present iff the member's text up to its colon is there (the literal minus its opening quote); otherwise read again from pos
            if (!vcj_lit(w, pool, op.off, op.len - 1u, S.ws[i])) { w.init(d + pos, len - pos); break; }
            vcj_skip_ws(w);
            if (op.code == VOP_OPT_STR && w.have && w.peek(0) == 'n') { if (!vc_word(w, VCJ_NULL, 4)) return; break; }   // nil: omitted
            if (!vc_byte(w, '"')) return;
            w.fill();
            if (op.code == VOP_OPT_STR_NE && w.have && w.peek(0) == '"') { w.skip(1); break; }                              // "": omitted
            vcj_put_lit(out, pool, op.off, op.len);
            if (!vcj_str(w, out, true)) return;
            w.skip(1);
            out.put('"');
            break;
        }
        case VOP_END: vcj_skip_ws(w); if (w.rem) return; break;
        default: return;
        }
    }
    r.ok = 1;                                       // the length bound was checked at "proof":
}

// The issuer's key index: FNV-1a of its bytes, probe, confirm byte for byte; 0xffffffff if the key set has no such DID
// (the probe k_vc_parse does inline in vc_parse_one, k_vcdoc.cu; a deliberate copy, so that the existing kernels' machine code stays
// exactly as it was: moving their probe into a shared helper would recompile them)
AFC_HD uint32_t vcj_resolve(const uint8_t* iss, uint32_t iss_len, const uint8_t* dids, const uint32_t* did_off, const uint32_t* slots,
                            uint32_t slot_mask) {
    ByteWindow w; w.init(iss, iss_len);
    uint32_t h = 2166136261u;
    while (w.rem) { w.fill(); h = vc_did_hash_byte(h, w.peek(0)); w.skip(1); }
    for (uint32_t s = h & slot_mask;; s = (s + 1) & slot_mask) {
        const uint32_t k = slots[s];
        if (k == 0xffffffffu) return k;
        const uint32_t k0 = did_off[k], kl = did_off[k + 1] - k0;
        if (kl != iss_len) continue;
        uint32_t j = 0;
        while (j < kl && dids[k0 + j] == iss[j]) ++j;
        if (j == kl) return k;
    }
}

#if !AFC_DEVICE_CODE
// 0 on success, -1 for an unknown kind.  The whitespace masks follow from the literals alone: whitespace may precede a byte that is
// not inside a quoted name or value (an opening quote included, a closing one not).  A literal after a string op starts inside that
// string; an optional member's op ends outside the string it reads.
static inline int vcj_schema_build(int kind, VcjSchema* s) {
    memset(s, 0, sizeof(*s));
    if (vc_schema_build(kind, &s->s) != 0) return -1;
    bool in = false;
    const uint8_t* pool = (const uint8_t*)s->s.pool;
    for (uint32_t i = 0; i < s->s.n_ops; i++) {
        const VcOp& op = s->s.ops[i];
        if (op.code != VOP_LIT && op.code != VOP_OPT_STR && op.code != VOP_OPT_STR_NE) continue;
        if (op.len > VCJ_MAX_LIT) return -1;
        uint64_t m = 0;
        for (uint32_t j = 0; j < op.len; j++) {
            if (!in) m |= 1ull << j;
            if (pool[op.off + j] == '"') in = !in;
        }
        s->ws[i] = m;
        if (op.code != VOP_LIT) in = false;
    }
    return 0;
}
#endif

}  // namespace afc
