// DIDs resolved and W3C DID documents served on the device (afc_did_resolve_batch, include/afcrypto.h): the bodies gin's c.JSON writes
// for GET /api/v1/did/resolve/:did and GET /api/v1/did/document/:did (internal/handlers/did_handlers.go:73-94, 368-429) after
// DIDService.ResolveDID (internal/services/did_service.go:368-473).
//
//   dres_resolve     the resolve handler's gin.H, keys sorted: component_type, derivation_path, did, function_name, public_key_jwk (the
//                    stored JWK text as a JSON string)
//   dres_document    the document handler's map, keys sorted at every level, publicKeyJwk the stored JWK re-marshalled through
//                    map[string]interface{} (jv_emit, afc_jsonval.cuh), copied from the text dres_entry chose
//   dres_not_found   the two 404 bodies; the document's details is err.Error() = "DID not found: " + the request
//   dres_entry       one directory entry at attach time: both body lengths (0 = HOST), and whether the stored JWK is already the text
//                    jv_emit writes (then the document copies it; otherwise k_dres_canon writes the canonical text once, beside it)
//
// Shared by the kernels of k_didresolve.cu and the CPU build of the same logic in tests/hostsim.
#pragma once
#include "afc_jsonval.cuh"
#include "afc_vcissue.cuh"

namespace afc {

enum : uint32_t { DRES_SERVER = 0, DRES_AGENT = 1, DRES_REASONER = 2, DRES_SKILL = 3, DRES_KINDS = 4 };     // AFC_DID_KIND_*
enum : uint32_t { DRES_RESOLVE = 0, DRES_DOCUMENT = 1 };                                                    // AFC_DIDRES_RESOLVE / _DOCUMENT
enum : uint32_t { DRES_FOUND = 0, DRES_NOT_FOUND = 1, DRES_BAD_REQUEST = 2, DRES_HOST = 3 };                // AFC_DIDRES_* states
enum : uint32_t { DRES_COL_PATH = 0, DRES_COL_FUNCTION = 1, DRES_COL_JWK = 2, DRES_COLUMNS = 3 };
constexpr uint32_t DRES_CAP = 4096;          // a longer body is left to the host: keeps afc_did_resolve_bound small
constexpr uint32_t DRES_REQ_MAX = 0x7fffffffu;

#define DRES_NOT_FOUND_BODY "{\"error\":\"DID not found\"}"
#define DRES_BAD_REQUEST_BODY "{\"error\":\"DID parameter is required\"}"
#define DRES_DOC404_HEAD "{\"details\":\"DID not found: "
#define DRES_DOC404_TAIL "\",\"error\":\"DID not found\"}"
constexpr uint32_t DRES_NOT_FOUND_LEN = sizeof(DRES_NOT_FOUND_BODY) - 1;
constexpr uint32_t DRES_BAD_REQUEST_LEN = sizeof(DRES_BAD_REQUEST_BODY) - 1;
constexpr uint32_t DRES_DOC404_FIXED = sizeof(DRES_DOC404_HEAD) - 1 + sizeof(DRES_DOC404_TAIL) - 1;

struct DresStr { const uint8_t* p; uint64_t len; };

AFC_HD const char* dres_component_type(uint32_t kind) {
    return kind == DRES_SERVER ? "agentfield_server" : kind == DRES_AGENT ? "agent" : kind == DRES_REASONER ? "reasoner" : "skill";
}

template <class Sink>
AFC_HD void dres_str(Sink& out, DresStr s) {
    out.put('"');
    go_json_escape(out, s.p, s.len);
    out.put('"');
}

template <class Sink>
AFC_HD void dres_resolve(Sink& out, uint32_t kind, DresStr did, DresStr path, DresStr fn, DresStr jwk) {
    vci_put_text(out, "{\"component_type\":\"");
    vci_put_text(out, dres_component_type(kind));
    vci_put_text(out, "\",\"derivation_path\":");
    dres_str(out, path);
    vci_put_text(out, ",\"did\":");
    dres_str(out, did);
    vci_put_text(out, ",\"function_name\":");
    dres_str(out, fn);
    vci_put_text(out, ",\"public_key_jwk\":");
    dres_str(out, jwk);
    out.put('}');
}

// jwk: the canonical text (copied as it is; jwk.p == nullptr writes nothing there, for the length of the rest)
template <class Sink>
AFC_HD void dres_document(Sink& out, DresStr did, DresStr jwk) {
    vci_put_text(out, "{\"@context\":[\"https://www.w3.org/ns/did/v1\",\"https://w3id.org/security/suites/ed25519-2020/v1\"],"
                      "\"assertionMethod\":[\"");
    go_json_escape(out, did.p, did.len);
    vci_put_text(out, "#key-1\"],\"authentication\":[\"");
    go_json_escape(out, did.p, did.len);
    vci_put_text(out, "#key-1\"],\"id\":");
    dres_str(out, did);
    vci_put_text(out, ",\"service\":[{\"description\":\"AgentField Agent Platform Service\",\"id\":\"");
    go_json_escape(out, did.p, did.len);
    vci_put_text(out, "#agentfield-service\",\"serviceEndpoint\":\"https://agentfield.example.com/api/v1\",\"type\":\"AgentFieldAgentService\"}],"
                      "\"verificationMethod\":[{\"controller\":");
    dres_str(out, did);
    vci_put_text(out, ",\"id\":\"");
    go_json_escape(out, did.p, did.len);
    vci_put_text(out, "#key-1\",\"publicKeyJwk\":");
    if (jwk.p) json_copy_raw(out, jwk.p, jwk.len);
    vci_put_text(out, ",\"type\":\"Ed25519VerificationKey2020\"}]}");
}

// the 404 body of a request of either kind
template <class Sink>
AFC_HD void dres_not_found(Sink& out, uint32_t kind, DresStr req) {
    if (kind == DRES_RESOLVE) { vci_put_text(out, DRES_NOT_FOUND_BODY); return; }
    vci_put_text(out, DRES_DOC404_HEAD);
    go_json_escape(out, req.p, req.len);
    vci_put_text(out, DRES_DOC404_TAIL);
}

// A sink that counts what it is given and checks it against a text: whether jv_emit would write the text back unchanged
struct ByteMatcher {
    const uint8_t* ref;
    uint64_t len, n;
    bool same;
    AFC_HDM void init(const uint8_t* r, uint64_t l) { ref = r; len = l; n = 0; same = true; }
    AFC_HDM void put(uint32_t b) { same = same && n < len && ref[n] == (uint8_t)b; ++n; }
    AFC_HDM void put4(uint32_t x) { put(x & 0xff); put((x >> 8) & 0xff); put((x >> 16) & 0xff); put(x >> 24); }
};

struct DresEntry {
    uint32_t rlen, dlen;     // the resolve and document body lengths, 0 = HOST
    uint32_t side;           // bytes of canonical JWK text to write beside the stored one (0: the stored text is canonical, or HOST)
};

// Entry k at attach time.  tape: jv_emit's, at least jwk.len / 2 + 1 entries.
AFC_HD DresEntry dres_entry(uint32_t kind, DresStr did, DresStr path, DresStr fn, DresStr jwk, uint32_t* tape) {
    DresEntry e; e.rlen = 0; e.dlen = 0; e.side = 0;
    {
        ByteCounter c; c.init();
        dres_resolve(c, kind, did, path, fn, jwk);
        if (c.n <= DRES_CAP) e.rlen = (uint32_t)c.n;
    }
    // json.Unmarshal into map[string]interface{}: an object, or null (a nil map, written as null); anything else is an error (a 500)
    if (jv_validate(jwk.p, jwk.len) != JV_OK) return e;
    const uint32_t len = (uint32_t)jwk.len, p = jv_skip_ws(jwk.p, 0, len);
    if (jwk.p[p] != '{' && jwk.p[p] != 'n') return e;
    ByteMatcher m; m.init(jwk.p, jwk.len);
    if (!jv_emit(m, jwk.p, len, tape)) return e;
    ByteCounter c; c.init();
    DresStr none; none.p = nullptr; none.len = 0;
    dres_document(c, did, none);
    if (c.n + m.n > DRES_CAP) return e;
    e.dlen = (uint32_t)(c.n + m.n);
    e.side = m.same && m.n == jwk.len ? 0 : (uint32_t)m.n;
    return e;
}

}  // namespace afc
