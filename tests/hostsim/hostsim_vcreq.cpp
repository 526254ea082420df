// TEST-ONLY CPU build of the request bind and the response writer (agentfield_b200/csrc/afc_vcreq.cuh): what one thread of k_vrq_bind,
// of k_vcj_parse / k_vcj_emit on the bound value, and of k_vrq_sizes / k_vrq_emit do for one request, with the issuer lookup and the
// signature check left to the caller.  Compiled on its own by tests/test_vcreq_hostsim.py.
#define AFC_HOSTSIM 1
#include "../../agentfield_b200/csrc/afc_vcreq.cuh"

using namespace afc;

extern "C" {

// vrq_bind: returns the VRB_* kind; span[0], span[1] = the object value's offset and length
uint32_t hs_vrq_bind(const uint8_t* req, uint64_t len, uint32_t span[2]) {
    const VrqBind b = vrq_bind(req, len);
    span[0] = b.off; span[1] = b.len;
    return b.kind;
}
// The json-verify walk of an execution document (msg must hold len + 64 bytes): VC_HOST, or the base64 status of proofValue (VC_VALID:
// a 64-byte signature in sig64, to be checked over msg[0 .. *msg_len)); fields: issuer / issuanceDate offsets and lengths; *b64_at: the
// base64 error index k_vrq_sizes computes for a VC_BAD_ENCODING document
int hs_vrq_doc(const uint8_t* doc, uint64_t len, uint8_t* msg, uint64_t* msg_len, uint8_t sig64[64], uint32_t fields[4], uint32_t* b64_at) {
    static VcjSchema S;
    static bool built = false;
    if (!built) { if (vcj_schema_build(VC_DOC_EXECUTION, &S)) return -1; built = true; }
    VcjParse r;
    ByteCounter c; c.init();
    vcj_walk<true>(S, doc, len, c, r);
    *msg_len = 0;
    if (!r.ok) return VC_HOST;
    fields[0] = r.iss_off; fields[1] = r.iss_len; fields[2] = r.date_off; fields[3] = r.date_len;
    ByteWriter w; w.init(msg);
    VcjParse r2;
    vcj_walk<false>(S, doc, len, w, r2);
    vcj_put_lit(w, S.s.pool, S.s.tail_off, S.s.tail_len);
    w.finish();
    *msg_len = (uint64_t)r.prefix + S.s.tail_len;
    uint32_t sig[16] = {0};
    const uint32_t st = vc_b64_signature(doc + r.pv_off, r.pv_len, sig);
    for (int k = 0; k < 16; k++) store_le32(sig64 + 4 * k, sig[k]);
    *b64_at = st == VC_BAD_ENCODING ? vrq_b64_error_at(doc + r.pv_off, r.pv_len) : 0;
    return (int)st;
}
// vrq_body through both sinks: returns the state; out (at least VRQ_FIXED + 6 len bytes) holds the body, *out_len its length, and the
// counted length must equal the written one (else -1)
int hs_vrq_body(uint32_t bind, uint32_t status, const uint8_t* doc, const uint32_t fields[4], uint32_t b64_at, uint8_t* out, uint64_t* out_len) {
    ByteCounter c; c.init();
    const uint32_t s = vrq_body(c, bind, status, doc, fields, b64_at);
    ByteWriter w; w.init(out);
    const uint32_t s2 = vrq_body(w, bind, status, doc, fields, b64_at);
    w.finish();
    *out_len = c.n;
    return s == s2 ? (int)s : -1;
}
uint64_t hs_vrq_fixed() { return VRQ_FIXED; }

}  // extern "C"
