// tests/devsim — TEST-ONLY CPU build of ge_ops.cuh: the portable twins, compiled by g++ with -DAFC_HOSTSIM.
// tests/test_ge_boundaries_hostsim.py and tests/test_ge_boundaries_gpu.py compile this file into a temporary directory.
#define AFC_HOSTSIM 1
#include <vector>

#include "ge_ops.cuh"

using namespace gesim;

template <int OP>
static int run_batch(const uint32_t* in, uint32_t* out, uint64_t n) {
    constexpr int IN = ge_in_words(OP), OUT = ge_out_words(OP), SCR = ge_scratch_words(OP);
    std::vector<uint32_t> scratch(SCR ? SCR : 1);
    for (uint64_t i = 0; i < n; i++)
        if (run_op<OP, false>(in + i * IN, out + i * OUT, scratch.data())) return 1;
    return 0;
}

extern "C" {

// out[n][ge_out_words(op)] = OP(in[n][ge_in_words(op)]); 1 for an unknown operation or an item outside its domain
int ge_run(int op, const uint32_t* in, uint32_t* out, uint64_t n) {
    switch (op) {
#define GE_CASE(OPC) case OPC: return run_batch<OPC>(in, out, n);
        GE_CASE(GE_DECODE) GE_CASE(GE_ENCODE) GE_CASE(GE_ENCODE_CALL) GE_CASE(GE_GROUP_KC) GE_CASE(GE_GROUP_SIGN)
        GE_CASE(GE_GROUP_SIGN2) GE_CASE(GE_DBL) GE_CASE(GE_DBL_CALL) GE_CASE(GE_ADDSUB) GE_CASE(GE_ADDSUB_CALL)
        GE_CASE(GE_TO_PRECOMP) GE_CASE(GE_MADD) GE_CASE(GE_CT_SELECT) GE_CASE(GE_SMALL_MULT) GE_CASE(GE_SMALL_MULT_CALL)
        GE_CASE(GE_AFFINE_RUN) GE_CASE(GE_AFFINE_RUN_CALL) GE_CASE(GE_AFFINE_FWDBWD) GE_CASE(GE_KEY_ROWS) GE_CASE(GE_RECODE)
        GE_CASE(GE_WELLFORMED)
#undef GE_CASE
    default: return 1;
    }
}
static_assert(GE_OP_COUNT == 21, "ge_run lists every operation");

int ge_op_count(void) { return GE_OP_COUNT; }
int ge_words(int op, int which) { return which == 0 ? ge_in_words(op) : which == 1 ? ge_out_words(op) : ge_scratch_words(op); }

}  // extern "C"
