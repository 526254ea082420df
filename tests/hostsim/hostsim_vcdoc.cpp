// TEST-ONLY CPU build of the stored-document parser (agentfield_b200/csrc/afc_vcdoc.cuh): what one thread of
// k_vc_parse and then k_vc_emit does for one document, with the issuer lookup left out (the span is returned instead).  Compiled
// on its own by tests/test_vcdoc_hostsim.py.
#define AFC_HOSTSIM 1
#include "../../agentfield_b200/csrc/afc_vcdoc.cuh"

using namespace afc;

extern "C" {

// Returns VC_HOST, or — the document being canonical and its issuer assumed known — VC_BAD_ENCODING, VC_INVALID (decoded length
// other than 64) or VC_VALID (a candidate: msg / *msg_len hold the signing message, sig64 the decoded signature).
// spans: issuer offset, length, issuanceDate offset, length, proof_at.  msg must hold len + 32 bytes.
int hs_vc_parse(int kind, const uint8_t* doc, uint64_t len, uint8_t* msg, uint64_t* msg_len, uint8_t sig64[64], uint32_t spans[5]) {
    static VcSchema S[2];
    static bool built = false;
    if (!built) { if (vc_schema_build(VC_DOC_EXECUTION, &S[0]) || vc_schema_build(VC_DOC_WORKFLOW, &S[1])) return -1; built = true; }
    if (kind != VC_DOC_EXECUTION && kind != VC_DOC_WORKFLOW) return -1;
    const VcSchema& s = S[kind];
    VcParse r;
    vc_parse_doc(s, doc, len, r);
    *msg_len = 0;
    if (!r.ok) return VC_HOST;
    spans[0] = r.iss_off; spans[1] = r.iss_len; spans[2] = r.date_off; spans[3] = r.date_len; spans[4] = r.proof_at;
    uint32_t sig[16] = {0};
    const uint32_t st = vc_b64_signature(doc + r.pv_off, r.pv_len, sig);
    if (st != VC_VALID) return (int)st;
    for (int k = 0; k < 16; k++) store_le32(sig64 + 4 * k, sig[k]);
    ByteWriter w; w.init(msg);
    json_copy_raw(w, doc, r.proof_at);
    const uint32_t* t = s.pool + (s.tail_off >> 2);
    uint32_t k = 0;
    for (; k + 4 <= s.tail_len; k += 4) w.put4(t[k >> 2]);
    for (; k < s.tail_len; k++) w.put((t[k >> 2] >> (8 * (k & 3))) & 0xffu);
    w.finish();
    *msg_len = (uint64_t)r.proof_at + s.tail_len;
    return VC_VALID;
}
// FNV-1a of a DID as the key set's table and k_vc_parse compute it
uint32_t hs_vc_did_hash(const uint8_t* p, uint64_t n) { uint32_t h = 2166136261u; for (uint64_t j = 0; j < n; j++) h = vc_did_hash_byte(h, p[j]); return h; }

}  // extern "C"
