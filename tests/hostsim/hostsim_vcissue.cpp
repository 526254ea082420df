// TEST-ONLY CPU build of the issuing routines (agentfield_b200/csrc/afc_vcissue.cuh): what one thread of k_vci_hashdata,
// k_vci_sizes, k_vci_fill and k_vci_proof does.  Compiled on its own by tests/test_vcissue_hostsim.py.
#define AFC_HOSTSIM 1
#include "../../agentfield_b200/csrc/afc_vcissue.cuh"

using namespace afc;

extern "C" {

// hashData of one payload: 43 characters at out
void hs_vci_hashdata(const uint8_t* p, uint64_t len, int nil, uint8_t* out) { vci_hashdata_one(p, len, nil != 0, out); }

// One credential: cols with 15 absolute offsets, hashes = 86 characters or NULL.  Writes the signing message and the stored document
// (proofValue placeholder) as the fill pass does and their lengths as the sizes pass reports them; returns -2 if the two passes
// disagree.  msg and doc must hold the sizes plus 32 bytes.
int hs_vci_doc(const uint8_t* cols, const uint64_t* coff, int64_t duration, const uint8_t* hashes, uint8_t* msg, uint64_t* msg_len,
               uint8_t* doc, uint64_t* doc_len) {
    static VciProgram P;
    static bool built = false;
    if (!built) { if (!vci_program_build(&P)) return -1; built = true; }
    VciItem it{cols, coff, hashes, duration};
    vci_doc_sizes(P, it, msg_len, doc_len);
    if (!msg || !doc) return 0;
    vci_doc_fill(P, it, msg, doc);
    ByteCounter a; a.init();
    vci_pieces(a, P, 0, VCI_COMMON + 1, it);
    return a.n == *msg_len ? 0 : -2;
}

// the two lengths only (the bound checks run on long inputs)
int hs_vci_sizes(const uint8_t* cols, const uint64_t* coff, int64_t duration, const uint8_t* hashes, uint64_t* msg_len, uint64_t* doc_len) {
    return hs_vci_doc(cols, coff, duration, hashes, nullptr, msg_len, nullptr, doc_len);
}

// 86 proofValue characters, into both outputs
void hs_vci_proof(const uint8_t* sig64, uint8_t* out_a, uint8_t* out_b) {
    uint32_t w[16];
    for (int k = 0; k < 16; k++) w[k] = load_le32(sig64 + 4 * k);
    vci_proof_one(w, out_a, out_b);
}

}  // extern "C"
