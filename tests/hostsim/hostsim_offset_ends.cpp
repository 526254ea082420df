// TEST-ONLY CPU build of offset_ends (agentfield_b200/csrc/afc_common.cuh): what the one thread of k_offset_ends and every afc_*_bound
// compute from a call's offset arrays.  Compiled on its own by tests/test_offset_ends_hostsim.py.
#define AFC_HOSTSIM 1
#include "../../agentfield_b200/csrc/afc_common.cuh"

using namespace afc;

extern "C" {

// k spans: array j is offs[j], with strides[j] and vias[j]; out: 2 k words
void hs_offset_ends(const uint64_t* const* offs, const uint32_t* strides, const int32_t* vias, int k, uint32_t n, uint64_t* out) {
    OffsetSpan s[8];
    for (int j = 0; j < k; j++) s[j] = OffsetSpan{offs[j], strides[j], vias[j]};
    offset_ends(s, k, n, out);
}

}  // extern "C"
