// tests/devsim — TEST-ONLY CPU build of devsim_ops.cuh: the portable twins, compiled by g++ with -DAFC_HOSTSIM.
// tests/test_fe_boundaries_hostsim.py compiles this file into a temporary directory.
#define AFC_HOSTSIM 1
#include "devsim_ops.cuh"

using namespace devsim;

template <int OP>
static int run_batch(const uint32_t* in, uint32_t* out, uint64_t n) {
    for (uint64_t i = 0; i < n; i++)
        if (run_op<OP, false>(in + i * 32, out + i * 16)) return 1;
    return 0;
}

extern "C" {

// out[n][16] = OP(in[n][32]); 1 for an operation the CPU build lacks (the Karatsuba product, the out-of-line multiplies)
int devsim_run(int op, const uint32_t* in, uint32_t* out, uint64_t n) {
    switch (op) {
#define DEVSIM_CASE(OPC) case OPC: return run_batch<OPC>(in, out, n);
        DEVSIM_CASE(OP_MUL_WIDE) DEVSIM_CASE(OP_SQ_WIDE) DEVSIM_CASE(OP_MUL_WIDE_KARA) DEVSIM_CASE(OP_FOLD16)
        DEVSIM_CASE(OP_MUL) DEVSIM_CASE(OP_SQ) DEVSIM_CASE(OP_MUL_CALL) DEVSIM_CASE(OP_SQ_CALL) DEVSIM_CASE(OP_ADD)
        DEVSIM_CASE(OP_SUB) DEVSIM_CASE(OP_ADDSUB) DEVSIM_CASE(OP_TOWORDS) DEVSIM_CASE(OP_INVERT) DEVSIM_CASE(OP_POW22523)
        DEVSIM_CASE(OP_SC_REDUCE512) DEVSIM_CASE(OP_SC_REDUCE256) DEVSIM_CASE(OP_SC_MULADD)
#undef DEVSIM_CASE
    default: return 1;
    }
}

int devsim_op_count(void) { return OP_COUNT; }

}  // extern "C"
