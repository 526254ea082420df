// json.Marshal(json.Unmarshal(raw)) for an interface{} value, on the device (afc_webhook_sign_batch, include/afcrypto.h).
//
// ExecutionWebhookPayload.Result is decodeExecutionPayload(raw) (internal/services/webhook_dispatcher.go:459-468): Unmarshal turns
// every object into a map[string]interface{} and every number into a float64, so Marshal writes the value back with map keys
// sorted by bytes (strings.Compare), numbers in strconv's shortest float64 form (afc_float.cuh) and strings re-escaped with Go's
// HTML-safe rules (vcj_str / vcj_put_cp, afc_vcjson.cuh).
//
//   jv_validate  Go's scanner (checkValid): RFC 8259 with whitespace only 0x20 0x09 0x0A 0x0D around tokens, exactly one value,
//                top-level scalars allowed, no BOM.  JV_SYNTAX: Unmarshal rejects the text, so the payload carries string(raw).
//   jv_emit      the canonical text of a value jv_validate accepted, one template over the sink: ByteCounter in the sizes pass,
//                ByteWriter in the emit pass, so the length the first reports is what the second writes.
//
// Declines (JV_HOST, left to the host; never a guess), all of them values Unmarshal accepts that the device does not re-marshal:
//   - duplicate keys in an object (Go keeps the last value)
//   - a backslash in a key (the sort compares the key's input bytes)
//   - raw invalid UTF-8 and lone surrogate escapes in a string or key (Go writes U+FFFD)
//   - nesting deeper than JV_MAX_DEPTH
//   - a number fl_parse declines: overflow (Unmarshal's range error), underflow to zero, subnormals, Eisel-Lemire give-ups
//   - a text of 2^31 bytes or more
//
// Objects are written in key order with a per-value tape of uint32 entries: at each container the walk records where its direct
// children start (an object: each key's first byte; an array: each element), heap-sorts an object's keys, checks neighbours for
// duplicates and then writes the children in that order, descending through an explicit stack.  A child costs at least two
// bytes of text (its first byte and the ',' or closing bracket after it), so a text of L bytes needs at most L / 2 entries however
// it nests: the tape is sized from the byte count alone.  Both passes sort (the sizes pass must see duplicates); sorting does
// not change the length.
#pragma once
#include "afc_float.cuh"
#include "afc_vcjson.cuh"

namespace afc {

enum : uint32_t { JV_OK = 0, JV_SYNTAX = 1, JV_HOST = 2 };
constexpr uint32_t JV_MAX_DEPTH = 32;
constexpr uint32_t JV_MAX_LEN = 0x7fffffffu;

AFC_HD uint32_t jv_skip_ws(const uint8_t* d, uint32_t p, uint32_t len) {
    while (p < len && vcj_is_ws(d[p])) ++p;
    return p;
}
AFC_HD bool jv_digit(uint32_t c) { return c >= '0' && c <= '9'; }

// end of the string token whose opening quote is at p, or 0 for a syntax error (p + 1 > 0 for any real end)
AFC_HD uint32_t jv_check_string(const uint8_t* d, uint32_t p, uint32_t len) {
    for (++p; p < len; ++p) {
        const uint32_t c = d[p];
        if (c == '"') return p + 1;
        if (c < 0x20) return 0;
        if (c == '\\') {
            if (++p >= len) return 0;
            const uint32_t e = d[p];
            if (e == 'u') {
                if (p + 4 >= len) return 0;
                for (uint32_t k = 1; k <= 4; k++) if (vcj_hex(d[p + k]) == 16) return 0;
                p += 4;
            } else if (!(e == '"' || e == '\\' || e == '/' || e == 'b' || e == 'f' || e == 'n' || e == 'r' || e == 't')) return 0;
        }
    }
    return 0;
}
// end of the number token at p, or 0 for a syntax error
AFC_HD uint32_t jv_check_number(const uint8_t* d, uint32_t p, uint32_t len) {
    if (d[p] == '-') ++p;
    if (p >= len || !jv_digit(d[p])) return 0;
    if (d[p] == '0') ++p;
    else while (p < len && jv_digit(d[p])) ++p;
    if (p < len && d[p] == '.') {
        ++p;
        if (p >= len || !jv_digit(d[p])) return 0;
        while (p < len && jv_digit(d[p])) ++p;
    }
    if (p < len && (d[p] == 'e' || d[p] == 'E')) {
        ++p;
        if (p < len && (d[p] == '+' || d[p] == '-')) ++p;
        if (p >= len || !jv_digit(d[p])) return 0;
        while (p < len && jv_digit(d[p])) ++p;
    }
    return p;
}
AFC_HD bool jv_is_lit(const uint8_t* d, uint32_t p, uint32_t len, const char* s, uint32_t n) {
    if (len - p < n) return false;
    for (uint32_t k = 0; k < n; k++) if (d[p + k] != (uint8_t)s[k]) return false;
    return true;
}

// Go's checkValid: JV_OK, JV_SYNTAX, or JV_HOST for nesting deeper than JV_MAX_DEPTH (or a text too long for 32-bit positions)
AFC_HD uint32_t jv_validate(const uint8_t* d, uint64_t len64) {
    if (len64 > JV_MAX_LEN) return JV_HOST;
    const uint32_t len = (uint32_t)len64;
    uint32_t p = jv_skip_ws(d, 0, len), depth = 0, is_obj = 0;     // bit k of is_obj: container k is an object
    bool want_key = false;
    for (;;) {
        // a value (or, after '{' / ',' in an object, a key and its colon first)
        if (p >= len) return JV_SYNTAX;
        if (want_key) {
            if (d[p] != '"') return JV_SYNTAX;
            p = jv_check_string(d, p, len);
            if (!p) return JV_SYNTAX;
            p = jv_skip_ws(d, p, len);
            if (p >= len || d[p] != ':') return JV_SYNTAX;
            p = jv_skip_ws(d, p + 1, len);
            if (p >= len) return JV_SYNTAX;
            want_key = false;
        }
        const uint32_t c = d[p];
        if (c == '{' || c == '[') {
            if (depth == JV_MAX_DEPTH) return JV_HOST;
            is_obj = (is_obj & ~(1u << depth)) | ((c == '{' ? 1u : 0u) << depth);
            ++depth;
            p = jv_skip_ws(d, p + 1, len);
            if (p < len && d[p] == (c == '{' ? '}' : ']')) { --depth; ++p; }
            else { want_key = c == '{'; continue; }
        } else if (c == '"') {
            p = jv_check_string(d, p, len);
        } else if (c == '-' || jv_digit(c)) {
            p = jv_check_number(d, p, len);
        } else if (c == 't') {
            p = jv_is_lit(d, p, len, "true", 4) ? p + 4 : 0;
        } else if (c == 'f') {
            p = jv_is_lit(d, p, len, "false", 5) ? p + 5 : 0;
        } else if (c == 'n') {
            p = jv_is_lit(d, p, len, "null", 4) ? p + 4 : 0;
        } else return JV_SYNTAX;
        if (!p) return JV_SYNTAX;
        // after a value: ',' or the closing bracket of the container, or the end of the text at depth 0
        for (;;) {
            p = jv_skip_ws(d, p, len);
            if (depth == 0) return p == len ? JV_OK : JV_SYNTAX;
            if (p >= len) return JV_SYNTAX;
            const bool obj = (is_obj >> (depth - 1)) & 1;
            if (d[p] == ',') { p = jv_skip_ws(d, p + 1, len); want_key = obj; break; }
            if (d[p] != (obj ? '}' : ']')) return JV_SYNTAX;
            --depth; ++p;
        }
    }
}

// ---- the re-marshalling walk (valid JSON only)

// the end of the value starting at p
AFC_HD uint32_t jv_skip_value(const uint8_t* d, uint32_t p, uint32_t len) {
    uint32_t depth = 0;
    do {
        const uint32_t c = d[p];
        if (c == '"') {
            for (++p; d[p] != '"'; ++p) if (d[p] == '\\') ++p;
            ++p;
        } else if (c == '{' || c == '[') { ++depth; ++p; }
        else if (c == '}' || c == ']') { --depth; ++p; }
        else if (depth) ++p;
        else while (p < len && !(d[p] == ',' || d[p] == '}' || d[p] == ']' || vcj_is_ws(d[p]))) ++p;     // a scalar
    } while (depth);
    return p;
}

// strings.Compare of two keys without backslashes, each given by its first byte (the closing quote ends it)
AFC_HD int jv_key_cmp(const uint8_t* d, uint32_t a, uint32_t b) {
    for (;; ++a, ++b) {
        const uint32_t x = d[a], y = d[b];
        if (x == '"') return y == '"' ? 0 : -1;
        if (y == '"') return 1;
        if (x != y) return x < y ? -1 : 1;
    }
}
AFC_HD void jv_sift(const uint8_t* d, uint32_t* t, uint32_t i, uint32_t n) {
    const uint32_t v = t[i];
    for (;;) {
        uint32_t c = 2 * i + 1;
        if (c >= n) break;
        if (c + 1 < n && jv_key_cmp(d, t[c], t[c + 1]) < 0) ++c;
        if (jv_key_cmp(d, v, t[c]) >= 0) break;
        t[i] = t[c];
        i = c;
    }
    t[i] = v;
}
AFC_HD void jv_heapsort(const uint8_t* d, uint32_t* t, uint32_t n) {
    if (n < 2) return;
    for (uint32_t i = n / 2; i-- > 0;) jv_sift(d, t, i, n);
    for (uint32_t end = n - 1; end > 0; --end) {
        const uint32_t x = t[0]; t[0] = t[end]; t[end] = x;
        jv_sift(d, t, 0, end);
    }
}

// a string body starting at p (after its quote), decoded and written back as Go does; false = declined
template <class Sink>
AFC_HD bool jv_string(Sink& out, const uint8_t* d, uint32_t p, uint32_t len) {
    ByteWindow w; w.init(d + p, len - p);
    out.put('"');
    if (!vcj_str(w, out, true)) return false;
    out.put('"');
    return true;
}

// a scalar at p: string, number or literal; false = declined
template <class Sink>
AFC_HD bool jv_scalar(Sink& out, const uint8_t* d, uint32_t p, uint32_t len) {
    const uint32_t c = d[p];
    if (c == '"') return jv_string(out, d, p + 1, len);
    if (c == 't') { out.put4(VCJ_TRUE); return true; }
    if (c == 'n') { out.put4(VCJ_NULL); return true; }
    if (c == 'f') { out.put4(VCJ_FALS); out.put('e'); return true; }
    uint32_t e = p;
    while (e < len && !(d[e] == ',' || d[e] == '}' || d[e] == ']' || vcj_is_ws(d[e]))) ++e;
    uint64_t bits;
    if (!fl_parse(d + p, e - p, &bits)) return false;
    fl_put(out, bits);
    return true;
}

// The canonical text of the value d[0..len) (jv_validate == JV_OK).  tape: at least len / 2 + 1 entries.  false = declined.
template <class Sink>
AFC_HD bool jv_emit(Sink& out, const uint8_t* d, uint32_t len, uint32_t* tape) {
    uint32_t f_base[JV_MAX_DEPTH], f_n[JV_MAX_DEPTH], f_j[JV_MAX_DEPTH];
    uint32_t is_obj = 0, top = 0, tp = 0;          // top: open containers; tp: tape entries in use
    uint32_t p = jv_skip_ws(d, 0, len);
    for (;;) {
        const uint32_t c = d[p];
        if (c == '{' || c == '[') {
            if (top == JV_MAX_DEPTH) return false;
            const bool obj = c == '{';
            const uint32_t close = obj ? '}' : ']';
            uint32_t k = 0, q = jv_skip_ws(d, p + 1, len);
            if (d[q] != close) {
                for (;;) {                         // record the children's starts
                    if (obj) {
                        const uint32_t k0 = q + 1;
                        for (q = k0; d[q] != '"'; ++q) if (d[q] == '\\') return false;      // escaped key: declined
                        tape[tp + k] = k0;
                        q = jv_skip_ws(d, q + 1, len);       // ':'
                        q = jv_skip_ws(d, q + 1, len);
                    } else tape[tp + k] = q;
                    ++k;
                    q = jv_skip_ws(d, jv_skip_value(d, q, len), len);
                    if (d[q] != ',') break;
                    q = jv_skip_ws(d, q + 1, len);
                }
            }
            if (obj) {
                jv_heapsort(d, tape + tp, k);
                for (uint32_t j = 1; j < k; j++) if (jv_key_cmp(d, tape[tp + j - 1], tape[tp + j]) == 0) return false;   // duplicate key
            }
            out.put(c);
            is_obj = (is_obj & ~(1u << top)) | ((obj ? 1u : 0u) << top);
            f_base[top] = tp; f_n[top] = k; f_j[top] = 0;
            ++top; tp += k;
        } else if (!jv_scalar(out, d, p, len)) return false;
        // the next child of the innermost open container, closing those that are done
        for (;;) {
            if (top == 0) return true;
            const uint32_t t = top - 1;
            const bool obj = (is_obj >> t) & 1;
            if (f_j[t] == f_n[t]) { out.put(obj ? '}' : ']'); tp = f_base[t]; --top; continue; }
            if (f_j[t]) out.put(',');
            const uint32_t e = tape[f_base[t] + f_j[t]++];
            if (obj) {
                if (!jv_string(out, d, e, len)) return false;
                out.put(':');
                uint32_t q = e;
                while (d[q] != '"') ++q;
                q = jv_skip_ws(d, q + 1, len);
                p = jv_skip_ws(d, q + 1, len);
            } else p = e;
            break;
        }
    }
}

}  // namespace afc
