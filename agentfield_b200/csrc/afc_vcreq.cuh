// VC verification requests answered on the device (afc_vc_verify_request_batch, include/afcrypto.h): the status and bytes the handlers of
// POST /api/v1/did/verify (internal/handlers/did_handlers.go:97-111) and POST /api/ui/v1/vc/verify (internal/handlers/ui/did.go:442-469)
// write for a request body, through VCService.VerifyVC (internal/services/vc_service.go:242-289).
//
//   vrq_bind    what c.ShouldBindJSON(&types.VCVerificationRequest) does with the body (gin's default build: json.NewDecoder(body).Decode,
//               the validator has nothing to check): Go's scanner over the first JSON value only (bytes after it are never read), its
//               top-level type, and the span of the last member whose name is vc_document or an ASCII-case-insensitive spelling of it
//               (json.RawMessage keeps the value's bytes as they stand)
//   vrq_body    the response: {"error":"Invalid request body"} for a bind error, else json.Marshal(types.VCVerificationResponse)
//               (pkg/types/did_types.go:273-279) for the verdict of the json-verify path on the value's bytes
//
// Declined (VRB_HOST): a top-level member name with an escape or a byte >= 0x80 (Go unquotes and folds those; no client sends them), and
// nesting deeper than VRQ_MAX_DEPTH (Go allows 10 000).  Shared by k_vcreq.cu and the CPU build in tests/hostsim.
#pragma once
#include "afc_vcissue.cuh"
#include "afc_vcjson.cuh"

namespace afc {

enum : uint32_t { VRQ_OK = 0, VRQ_BAD_REQUEST = 1, VRQ_HOST = 2 };                                   // AFC_VREQ_*
// what the bind found: a 400; no vc_document (or a top-level null); vc_document null; a value the device leaves to the host; an object
enum : uint32_t { VRB_BAD = 0, VRB_NO_DOC = 1, VRB_NULL_DOC = 2, VRB_HOST = 3, VRB_OBJECT = 4 };
constexpr uint32_t VRQ_MAX_DEPTH = 64;
constexpr uint64_t VRQ_REQ_MAX = 0x7fffffffull;           // a request of 2^31 bytes or more is AFC_EINVAL

#define VRQ_BAD_BODY "{\"error\":\"Invalid request body\"}"
#define VRQ_NO_DOC_BODY "{\"valid\":false,\"error\":\"failed to parse VC document: unexpected end of JSON input\"}"
#define VRQ_INVALID_BODY "{\"valid\":false,\"message\":\"Invalid signature\"}"
#define VRQ_UNRESOLVED_HEAD "{\"valid\":false,\"error\":\"failed to resolve issuer DID: DID not found: "
#define VRQ_BAD_B64_HEAD "{\"valid\":false,\"error\":\"failed to verify signature: failed to decode signature: illegal base64 data at input byte "
#define VRQ_ERROR_TAIL "\"}"
#define VRQ_VALID_HEAD "{\"valid\":true"
#define VRQ_VALID_ISSUER ",\"issuer_did\":\""
#define VRQ_VALID_DATE ",\"issued_at\":\""
#define VRQ_VALID_TAIL ",\"message\":\"VC verified successfully\"}"

constexpr uint64_t vrq_len(const char* s) { return *s ? 1 + vrq_len(s + 1) : 0; }
constexpr uint64_t vrq_max(uint64_t a, uint64_t b) { return a > b ? a : b; }
// the longest constant text of one body (10 digits for the base64 index); every other byte is one of I or D written with at most 6 bytes
// per byte of the request they stand in
constexpr uint64_t VRQ_FIXED =
    vrq_max(vrq_max(vrq_len(VRQ_BAD_BODY), vrq_len(VRQ_NO_DOC_BODY)),
            vrq_max(vrq_max(vrq_len(VRQ_INVALID_BODY), vrq_len(VRQ_UNRESOLVED_HEAD VRQ_ERROR_TAIL)),
                    vrq_max(vrq_len(VRQ_BAD_B64_HEAD VRQ_ERROR_TAIL) + 10,
                            vrq_len(VRQ_VALID_HEAD VRQ_VALID_ISSUER "\"" VRQ_VALID_DATE "\"" VRQ_VALID_TAIL))));

struct VrqBind {
    uint32_t kind;           // VRB_*
    uint32_t off, len;       // VRB_OBJECT: the value's bytes in the request
};

AFC_HD bool vrq_ws(uint32_t c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }
AFC_HD uint64_t vrq_skip_ws(const uint8_t* p, uint64_t i, uint64_t len) {
    while (i < len && vrq_ws(p[i])) ++i;
    return i;
}
AFC_HD bool vrq_digit(const uint8_t* p, uint64_t i, uint64_t len) { return i < len && p[i] >= '0' && p[i] <= '9'; }

// A string body from i (after its opening quote) as Go's scanner reads it: no byte below 0x20, escapes \" \\ \/ \b \f \n \r \t and \u
// with four hex digits (surrogates are not the scanner's business).  The index after the closing quote, or 0.  plain: no escape and no
// byte >= 0x80, so the bytes are the name Go compares.
AFC_HD uint64_t vrq_string(const uint8_t* p, uint64_t i, uint64_t len, bool& plain) {
    plain = true;
    while (i < len) {
        const uint32_t c = p[i];
        if (c == '"') return i + 1;
        if (c < 0x20) return 0;
        if (c >= 0x80) plain = false;
        if (c != '\\') { ++i; continue; }
        plain = false;
        if (i + 1 >= len) return 0;
        const uint32_t e = p[i + 1];
        if (e == 'u') {
            if (len - i < 6) return 0;
            for (uint32_t k = 2; k < 6; k++) if (vcj_hex(p[i + k]) == 16) return 0;
            i += 6;
            continue;
        }
        if (e != '"' && e != '\\' && e != '/' && e != 'b' && e != 'f' && e != 'n' && e != 'r' && e != 't') return 0;
        i += 2;
    }
    return 0;
}
// -?(0|[1-9][0-9]*)(\.[0-9]+)?([eE][+-]?[0-9]+)? from i; the index after it, or 0.  What follows is the caller's to check (a digit after
// a leading 0 is then an error, as in Go's stateEndValue).
AFC_HD uint64_t vrq_number(const uint8_t* p, uint64_t i, uint64_t len) {
    if (p[i] == '-') ++i;
    if (!vrq_digit(p, i, len)) return 0;
    if (p[i] == '0') ++i;
    else while (vrq_digit(p, i, len)) ++i;
    if (i < len && p[i] == '.') {
        if (!vrq_digit(p, ++i, len)) return 0;
        while (vrq_digit(p, i, len)) ++i;
    }
    if (i < len && (p[i] == 'e' || p[i] == 'E')) {
        ++i;
        if (i < len && (p[i] == '+' || p[i] == '-')) ++i;
        if (!vrq_digit(p, i, len)) return 0;
        while (vrq_digit(p, i, len)) ++i;
    }
    return i;
}
// the literal word at i; the index after it, or 0
AFC_HD uint64_t vrq_word(const uint8_t* p, uint64_t i, uint64_t len, const char* w) {
    for (; *w; ++w, ++i) if (i >= len || p[i] != (uint8_t)*w) return 0;
    return i;
}
// Go's field match for a name without escapes or bytes >= 0x80: the exact name, or equal after upper-casing ASCII letters (foldName)
AFC_HD bool vrq_is_vc_document(const uint8_t* p, uint64_t len) {
    const char* want = "VC_DOCUMENT";
    if (len != 11) return false;
    for (uint32_t k = 0; k < 11; k++) {
        uint32_t c = p[k];
        if (c >= 'a' && c <= 'z') c -= 32;
        if (c != (uint8_t)want[k]) return false;
    }
    return true;
}

// json.NewDecoder(body).Decode(&req): the first value is scanned whole before it is decoded, so a syntax error anywhere inside it is a
// 400; a value that is neither an object nor null does not decode into the struct (a 400 too); unknown members are skipped; the last
// vc_document wins.
AFC_HD VrqBind vrq_bind(const uint8_t* p, uint64_t len) {
    VrqBind r; r.kind = VRB_BAD; r.off = r.len = 0;
    uint64_t i = vrq_skip_ws(p, 0, len);
    if (i == len) return r;                                        // io.EOF
    if (p[i] == 'n') { if (vrq_word(p, i, len, "null")) r.kind = VRB_NO_DOC; return r; }
    if (p[i] != '{') return r;
    uint64_t arr = 0;                   // bit d: the container at depth d + 1 is an array
    uint32_t depth = 1;
    bool first = true, host = false, open_match = false;
    uint32_t found = VRB_NO_DOC;
    uint64_t v0 = 0, v1 = 0;
    ++i;
    for (;;) {
        const bool in_arr = (arr >> (depth - 1)) & 1;
        const uint32_t close = in_arr ? ']' : '}';
        i = vrq_skip_ws(p, i, len);
        if (i == len) return r;
        uint32_t c = p[i];
        if (c == close) { ++i; goto closed; }
        if (!first) {
            if (c != ',') return r;
            i = vrq_skip_ws(p, i + 1, len);
            if (i == len) return r;
            c = p[i];
        }
        first = false;
        {
            bool match = false;
            if (!in_arr) {
                if (c != '"') return r;
                bool plain;
                const uint64_t k0 = i + 1;
                i = vrq_string(p, k0, len, plain);
                if (!i) return r;
                if (depth == 1) {
                    if (!plain) host = true;
                    else match = vrq_is_vc_document(p + k0, i - 1 - k0);
                }
                i = vrq_skip_ws(p, i, len);
                if (i == len || p[i] != ':') return r;
                i = vrq_skip_ws(p, i + 1, len);
                if (i == len) return r;
                c = p[i];
            }
            const uint64_t at = i;
            if (c == '{' || c == '[') {
                if (depth == VRQ_MAX_DEPTH) { r.kind = VRB_HOST; return r; }
                if (match) { open_match = true; v0 = at; found = c == '{' ? VRB_OBJECT : VRB_HOST; }
                arr = c == '[' ? arr | (1ull << depth) : arr & ~(1ull << depth);
                ++depth; first = true; ++i;
                continue;
            }
            bool plain;
            if (c == '"') i = vrq_string(p, i + 1, len, plain);
            else if (c == 't') i = vrq_word(p, i, len, "true");
            else if (c == 'f') i = vrq_word(p, i, len, "false");
            else if (c == 'n') i = vrq_word(p, i, len, "null");
            else if (c == '-' || (c >= '0' && c <= '9')) i = vrq_number(p, i, len);
            else return r;
            if (!i) return r;
            if (match) { found = c == 'n' ? VRB_NULL_DOC : VRB_HOST; v0 = at; v1 = i; }
            continue;
        }
    closed:
        if (--depth == 0) break;
        if (depth == 1 && open_match) { v1 = i; open_match = false; }
        first = false;
    }
    r.kind = host ? VRB_HOST : found;
    if (r.kind == VRB_OBJECT) { r.off = (uint32_t)v0; r.len = (uint32_t)(v1 - v0); }
    return r;
}

// The response to a request: bind = vrq_bind's kind; for VRB_OBJECT, status / f (4 words) are the json-verify verdict and fields of the value's
// bytes doc, and b64_at the base64 error index of a VC_BAD_ENCODING one.  Returns the state; a VRQ_HOST request writes nothing.  I
// (issuer, never escaped in a document the walk accepts) is written through go_json_escape; D (issuanceDate, which may hold escapes) is
// decoded and written back by vcj_str, whose code-point writer follows go_json_escape's rules.
template <class Sink>
AFC_HD uint32_t vrq_body(Sink& out, uint32_t bind, uint32_t status, const uint8_t* doc, const uint32_t* f, uint32_t b64_at) {
    switch (bind) {
    case VRB_BAD: vci_put_text(out, VRQ_BAD_BODY); return VRQ_BAD_REQUEST;
    case VRB_NO_DOC: vci_put_text(out, VRQ_NO_DOC_BODY); return VRQ_OK;
    case VRB_NULL_DOC: vci_put_text(out, VRQ_UNRESOLVED_HEAD VRQ_ERROR_TAIL); return VRQ_OK;
    case VRB_OBJECT: break;
    default: return VRQ_HOST;
    }
    switch (status) {
    case VC_VALID:
        vci_put_text(out, VRQ_VALID_HEAD);
        if (f[1]) { vci_put_text(out, VRQ_VALID_ISSUER); go_json_escape(out, doc + f[0], f[1]); out.put('"'); }
        if (f[3]) {
            vci_put_text(out, VRQ_VALID_DATE);
            ByteWindow w; w.init(doc + f[2], (uint64_t)f[3] + 1);        // the body and its closing quote
            vcj_str(w, out, true);
            out.put('"');
        }
        vci_put_text(out, VRQ_VALID_TAIL);
        return VRQ_OK;
    case VC_INVALID: vci_put_text(out, VRQ_INVALID_BODY); return VRQ_OK;
    case VC_UNRESOLVED:
        vci_put_text(out, VRQ_UNRESOLVED_HEAD);
        go_json_escape(out, doc + f[0], f[1]);
        vci_put_text(out, VRQ_ERROR_TAIL);
        return VRQ_OK;
    case VC_BAD_ENCODING:
        vci_put_text(out, VRQ_BAD_B64_HEAD);
        vci_put_int(out, b64_at);
        vci_put_text(out, VRQ_ERROR_TAIL);
        return VRQ_OK;
    default: return VRQ_HOST;
    }
}

// base64.RawURLEncoding.DecodeString's CorruptInputError offset for a proofValue vc_b64_signature rejects: the first byte outside the
// URL alphabet, else (length 1 mod 4) the last byte.  Go skips \r and \n; a proofValue the walk accepts holds neither.
AFC_HD uint32_t vrq_b64_error_at(const uint8_t* s, uint32_t len) {
    for (uint32_t k = 0; k < len; k++) {
        const uint32_t c = s[k];
        if (!((c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || (c >= '0' && c <= '9') || c == '-' || c == '_')) return k;
    }
    return len ? len - 1 : 0;
}

}  // namespace afc
