// tests/devsim — TEST-ONLY harness over the field and scalar routines, one operation per item on raw 32-bit limbs.
//
// The product headers are included unchanged.  devsim.cu compiles this for sm_90a, where afc_fe.cuh takes its inline-PTX
// carry chains (and, under -DAFC_FOLD_SHIFT=1 / -DAFC_FE_KARATSUBA=1, the alternative fold and multiply); devsim_host.cpp
// compiles it with g++ -DAFC_HOSTSIM, where the portable twins run.  tests/test_fe_boundaries_*.py feed both the
// constructed boundary operands of tests/fe_cases.py and compare bit for bit with Python integers.
//
// Item layout: 32 input words (a = in[0..7], b = in[8..15], c = in[16..23]; a 16-word input is in[0..15]; fe_addsub_m
// takes keep = in[16] & 1, sgn = in[17] & 1 as all-ones masks), 16 output words.  Weakly reduced results come back as the
// raw limbs the routine left, not as canonical words.
#pragma once
#include "../../agentfield_b200/csrc/afc_fe.cuh"
#include "../../agentfield_b200/csrc/afc_sc.cuh"

namespace devsim {
using namespace afc;

enum Op {
    OP_MUL_WIDE = 0, OP_SQ_WIDE, OP_MUL_WIDE_KARA, OP_FOLD16, OP_MUL, OP_SQ, OP_MUL_CALL, OP_SQ_CALL, OP_ADD, OP_SUB, OP_ADDSUB,
    OP_TOWORDS, OP_INVERT, OP_POW22523, OP_SC_REDUCE512, OP_SC_REDUCE256, OP_SC_MULADD, OP_COUNT
};

// the portable twins as a multiplication policy, so the exponentiation chains can run on them too
struct FePortable {
    static AFC_HDM void mul(fe& h, const fe& f, const fe& g) { fe_mul_c(h, f, g); }
    static AFC_HDM void sq(fe& h, const fe& f) { fe_sq_c(h, f); }
};

AFC_HD void put8(uint32_t* out, const fe& h) {
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = h.v[i];
#pragma unroll
    for (int i = 8; i < 16; i++) out[i] = 0;
}
AFC_HD void zero_hi(uint32_t* out) {
#pragma unroll
    for (int i = 8; i < 16; i++) out[i] = 0;
}

// Runs OP on one item.  PORTABLE selects the _c twins where afc_fe.cuh has them (the device's own reference for the bulk
// runs); operations with one form only run that form either way.  Returns 0, or 1 for an operation this build lacks.
template <int OP, bool PORTABLE>
AFC_HD int run_op(const uint32_t* in, uint32_t* out) {
    fe a, b, h;
    fe_from_words(a, in);
    fe_from_words(b, in + 8);
    if constexpr (OP == OP_MUL_WIDE) {
        if constexpr (PORTABLE) fe_mul_wide_c(out, a.v, b.v); else fe_mul_wide(out, a.v, b.v);
    } else if constexpr (OP == OP_SQ_WIDE) {
        if constexpr (PORTABLE) fe_sq_wide_c(out, a.v); else fe_sq_wide(out, a.v);
    } else if constexpr (OP == OP_MUL_WIDE_KARA) {
#if AFC_DEVICE_CODE && AFC_FE_PTX
        if constexpr (PORTABLE) fe_mul_wide_c(out, a.v, b.v); else fe_mul_wide_kara(out, a.v, b.v);
#else
        return 1;
#endif
    } else if constexpr (OP == OP_FOLD16) {
        uint32_t t[16];
#pragma unroll
        for (int i = 0; i < 16; i++) t[i] = in[i];
        if constexpr (PORTABLE) fe_fold16_c(h, t); else fe_fold16(h, t);
        put8(out, h);
    } else if constexpr (OP == OP_MUL) {
        if constexpr (PORTABLE) fe_mul_c(h, a, b); else FeInline::mul(h, a, b);
        put8(out, h);
    } else if constexpr (OP == OP_SQ) {
        if constexpr (PORTABLE) fe_sq_c(h, a); else FeInline::sq(h, a);
        put8(out, h);
    } else if constexpr (OP == OP_MUL_CALL || OP == OP_SQ_CALL) {
#if !defined(AFC_HOSTSIM)
        if constexpr (PORTABLE) { if constexpr (OP == OP_MUL_CALL) fe_mul_c(h, a, b); else fe_sq_c(h, a); }
        else { if constexpr (OP == OP_MUL_CALL) FeCall::mul(h, a, b); else FeCall::sq(h, a); }
        put8(out, h);
#else
        return 1;
#endif
    } else if constexpr (OP == OP_ADD) {
        if constexpr (PORTABLE) fe_add_c(h, a, b); else fe_add(h, a, b);
        put8(out, h);
    } else if constexpr (OP == OP_SUB) {
        if constexpr (PORTABLE) fe_sub_c(h, a, b); else fe_sub(h, a, b);
        put8(out, h);
    } else if constexpr (OP == OP_ADDSUB) {
        const uint32_t keep = 0u - (in[16] & 1u), sgn = 0u - (in[17] & 1u);
        if constexpr (PORTABLE) fe_addsub_m_c(h, a, b, keep, sgn); else fe_addsub_m(h, a, b, keep, sgn);
        put8(out, h);
    } else if constexpr (OP == OP_TOWORDS) {
        fe_towords(out, a);
        zero_hi(out);
    } else if constexpr (OP == OP_INVERT) {
        if constexpr (PORTABLE) fe_invert<FePortable>(h, a); else fe_invert<FeInline>(h, a);
        put8(out, h);
    } else if constexpr (OP == OP_POW22523) {
        if constexpr (PORTABLE) fe_pow22523<FePortable>(h, a); else fe_pow22523<FeInline>(h, a);
        put8(out, h);
    } else if constexpr (OP == OP_SC_REDUCE512) {
        sc_reduce512(out, in);
        zero_hi(out);
    } else if constexpr (OP == OP_SC_REDUCE256) {
        sc_reduce256(out, in);
        zero_hi(out);
    } else if constexpr (OP == OP_SC_MULADD) {
        sc_muladd(out, in, in + 8, in + 16);
        zero_hi(out);
    } else {
        return 1;
    }
    return 0;
}

}  // namespace devsim
