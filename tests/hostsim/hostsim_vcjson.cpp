// TEST-ONLY CPU build of the tolerant document walk (agentfield_b200/csrc/afc_vcjson.cuh): what one thread of k_vcj_parse and then
// k_vcj_emit does for one document, with the issuer lookup left out (the span is returned instead).  Compiled on its own by
// tests/test_vcjson_hostsim.py.
#define AFC_HOSTSIM 1
#include "../../agentfield_b200/csrc/afc_vcjson.cuh"

using namespace afc;

namespace {
struct BufSink {                 // plain byte sink for the escaper checks
    uint8_t* p; uint64_t n;
    void put(uint32_t b) { p[n++] = (uint8_t)b; }
    void put4(uint32_t x) { put(x & 0xff); put((x >> 8) & 0xff); put((x >> 16) & 0xff); put(x >> 24); }
};
}  // namespace

extern "C" {

// Returns VC_HOST, or — the document being accepted and its issuer assumed known — VC_BAD_ENCODING, VC_INVALID (decoded length
// other than 64) or VC_VALID (sig64 holds the decoded signature).  For every accepted document msg / *msg_len hold the signing
// message (sizes pass and emit pass, as the kernels run them); *msg_len is the length the sizes pass reported.
// spans: issuer offset, length, issuanceDate offset, length, prefix length.  msg must hold len + 32 bytes.
int hs_vcj_parse(int kind, const uint8_t* doc, uint64_t len, uint8_t* msg, uint64_t* msg_len, uint8_t sig64[64], uint32_t spans[5]) {
    static VcjSchema S[2];
    static bool built = false;
    if (!built) { if (vcj_schema_build(VC_DOC_EXECUTION, &S[0]) || vcj_schema_build(VC_DOC_WORKFLOW, &S[1])) return -1; built = true; }
    if (kind != VC_DOC_EXECUTION && kind != VC_DOC_WORKFLOW) return -1;
    const VcjSchema& s = S[kind];
    VcjParse r;
    ByteCounter c; c.init();
    vcj_walk<true>(s, doc, len, c, r);
    *msg_len = 0;
    if (!r.ok) return VC_HOST;
    spans[0] = r.iss_off; spans[1] = r.iss_len; spans[2] = r.date_off; spans[3] = r.date_len; spans[4] = r.prefix;
    ByteWriter w; w.init(msg);
    VcjParse r2;
    vcj_walk<false>(s, doc, len, w, r2);
    vcj_put_lit(w, s.s.pool, s.s.tail_off, s.s.tail_len);
    w.finish();
    *msg_len = (uint64_t)r.prefix + s.s.tail_len;
    if (!r2.ok) return -2;                                     // the emit pass must accept what the sizes pass accepted
    uint32_t sig[16] = {0};
    const uint32_t st = vc_b64_signature(doc + r.pv_off, r.pv_len, sig);
    for (int k = 0; k < 16; k++) store_le32(sig64 + 4 * k, sig[k]);
    return (int)st;
}
// The sizes pass alone (what k_vcj_parse runs): 1 if the document is accepted, with *count the canonical bytes the walk counted
// up to where it stopped (the whole prefix, 64-bit, when it reached "proof":).
int hs_vcj_sizes(int kind, const uint8_t* doc, uint64_t len, uint64_t* count) {
    VcjSchema s;
    if (vcj_schema_build(kind, &s)) return -1;
    VcjParse r;
    ByteCounter c; c.init();
    vcj_walk<true>(s, doc, len, c, r);
    *count = c.n;
    return (int)r.ok;
}
// one code point through vcj_put_cp; returns the number of bytes written to out (at most 6)
uint32_t hs_vcj_put_cp(uint32_t cp, uint8_t* out) { BufSink s{out, 0}; vcj_put_cp(s, cp); return (uint32_t)s.n; }
// a byte string through go_json_escape; returns the number of bytes written to out (at most 6 len)
uint64_t hs_go_json_escape(const uint8_t* p, uint64_t len, uint8_t* out) { BufSink s{out, 0}; go_json_escape(s, p, len); return s.n; }

}  // extern "C"
