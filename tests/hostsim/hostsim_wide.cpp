// TEST-ONLY CPU build of the recoding that the table-driven verify's radix-2^w fixed-base table is read with (sc_recode_wide /
// sc_digit_wide in agentfield_b200/csrc/afc_sc.cuh, base_table_* in afc_ge.cuh).  Compiled on its own by
// tests/test_wide_base_hostsim.py.
#define AFC_HOSTSIM 1
#include "../../agentfield_b200/csrc/afc_ge.cuh"

using namespace afc;

extern "C" {

// the signed digits of s (32 bytes, little endian) into out[0..rows), as ed25519_keyed_point walks them; returns rows.
// *top_max / *entries: the table geometry base_table_entries allocates for w
int hs_wide_digits(int w, const uint8_t s32[32], int32_t* out, int* top_max, uint64_t* entries) {
    uint32_t s[8], t[8];
    for (int i = 0; i < 8; i++) s[i] = load_le32(s32 + 4 * i);
    const base_table b = base_table_make(nullptr, w);
    sc_recode_wide(t, s, b.offset);
    for (int i = 0; i < b.rows; i++) out[i] = sc_digit_wide(t, i, w, b.rows);
    *top_max = base_table_top_max(w);
    *entries = base_table_entries(w);
    return b.rows;
}

}  // extern "C"
