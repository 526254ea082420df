// tests/devsim — TEST-ONLY harness over the group routines of afc_ge.cuh (and the scalar recodings of afc_sc.cuh), one
// operation per item on raw 32-bit limbs.
//
// The product headers are included unchanged.  ge.cu compiles this for sm_90a (the PTX field paths, under the same three
// builds as devsim.cu); ge_host.cpp compiles it with g++ -DAFC_HOSTSIM, where the portable twins run.
// tests/test_ge_boundaries_*.py feed both the constructed cases of tests/ge_cases.py and compare with big-integer Edwards
// arithmetic.  Each routine runs with the field policy its kernels give it (k_ed25519.cu): FeInline in verify and in the key
// chain, FeCall in signing (AFC_SIGN_FE), the base-table build and the start and inversion of a key-row slice.  FeCall has
// no CPU form; the CPU build runs those operations with FeInline, which computes the same limbs through the portable twins.
//
// Item layout: every operation has its own input and output width (ge_in_words / ge_out_words below), a multiple of 8 words
// so that table entries inside an item keep the 32-byte alignment the product's 128-bit loads need.  Points are raw limbs:
// a P3 point is X, Y, Z, T (32 words), a precomputed entry y+x, y-x, 2dxy (24 words).
#pragma once
#include <type_traits>

#include "devsim_ops.cuh"
#include "../../agentfield_b200/csrc/afc_ge.cuh"

namespace gesim {
using namespace afc;
using devsim::FePortable;

// The kernels' parameters (k_ed25519.cu; tests/test_ge_boundaries_hostsim.py checks that they still match it).
constexpr int KC_GMAX = 32, SIGN_GMAX = 8;       // group sizes of the table-driven verify and of the signing kernels
constexpr int KR_PARTS = 4, KR_SLICE = COMB_COLS / KR_PARTS;
#if defined(AFC_HOSTSIM)
using GeCall = FeInline;
#else
using GeCall = FeCall;
#endif

enum GeOp {
    GE_DECODE = 0,        // ge_frombytes<FeInline>: in enc[8]; out X, Y, Z, T, ok (word 32)
    GE_ENCODE,            // ge_encode<FeInline>: in X, Y, Z; out 8 words
    GE_ENCODE_CALL,       // ge_encode<FeCall>
    GE_GROUP_KC,          // ge_encode_group<FeInline, KC_GMAX>: in G (word 0), member g at 8 + 24 g (X, Y, Z); out 8 words per member
    GE_GROUP_SIGN,        // ge_encode_group<FeCall, SIGN_GMAX>
    GE_GROUP_SIGN2,       // ge_encode_group<FeCall, 2 SIGN_GMAX>
    GE_DBL,               // ge_dbl<FeInline> + ge_p1p1_to_p3: in P3 (T unused); out P3
    GE_DBL_CALL,          // the same with FeCall
    GE_ADDSUB,            // ge_p3_to_cached(Q) + ge_addsub<FeInline> + ge_p1p1_to_p3: in P (0), Q (32), neg (64); out P3
    GE_ADDSUB_CALL,       // the same with FeCall
    GE_TO_PRECOMP,        // ge_p3_to_precomp<FeInline>: in P3; out entry
    GE_MADD,              // in P (0), entry (32), neg (56), mode (57); mode 0: ge_maddsub<FeInline>, 1: ge_load_precomp_arranged +
                          // ge_madd_arranged<FeInline>; + ge_p1p1_to_p3; out P3
    GE_CT_SELECT,         // ge_ct_select: in 8 entries (0), d (192, signed); out entry
    GE_SMALL_MULT,        // ge_p3_to_cached(P) + ge_small_multiple<FeInline>: in P (0), m (32); out P3
    GE_SMALL_MULT_CALL,   // the same with FeCall
    GE_AFFINE_RUN,        // ge_p3_to_cached(P) + ge_affine_run<FeInline, 64>: in M (0), P (32); out 64 entries, then M (1536)
    GE_AFFINE_RUN_CALL,   // ge_affine_run<FeCall, 64> (the base-table build)
    GE_AFFINE_FWDBWD,     // ge_p3_to_cached<FeCall>(P) + ge_affine_run_fwd<FeInline, 32> + fe_invert<FeCall> + _bwd<FeInline, 32>:
                          // in M, P; out 32 entries, then M (768)
    GE_KEY_ROWS,          // in pk (0), row (8), stages (9: 1, 2 or 4); out ok of the staged build (0), ok of ge_build_key_row (1),
                          // the row from ge_key_chain_stage + ge_key_slice_start + fwd / fe_invert / bwd (8), then the row from
                          // ge_build_key_row (8 + 3072)
    GE_RECODE,            // in s (0), kind (8: 0 sc_recode16, 1 sc_recode256, 2 sc_recode65536, 16..22 sc_recode_wide at w = kind);
                          // out t (0), the digits as int32 (8..), and for the wide form base_table_top_max (72) and
                          // base_table_entries (73, 74: low and high words)
    GE_WELLFORMED,        // ed25519_sig_wellformed: in sig[16]; out the result (word 0)
    GE_OP_COUNT
};

AFC_HHD constexpr int ge_in_words(int op) {
    return op == GE_DECODE ? 8
         : op == GE_GROUP_KC ? 8 + 24 * KC_GMAX
         : op == GE_GROUP_SIGN ? 8 + 24 * SIGN_GMAX
         : op == GE_GROUP_SIGN2 ? 8 + 48 * SIGN_GMAX
         : op == GE_ADDSUB || op == GE_ADDSUB_CALL ? 72
         : op == GE_MADD || op == GE_AFFINE_RUN || op == GE_AFFINE_RUN_CALL || op == GE_AFFINE_FWDBWD ? 64
         : op == GE_CT_SELECT ? 200
         : op == GE_SMALL_MULT || op == GE_SMALL_MULT_CALL ? 40
         : op == GE_KEY_ROWS || op == GE_RECODE || op == GE_WELLFORMED ? 16
         : 32;
}
AFC_HHD constexpr int ge_out_words(int op) {
    return op == GE_DECODE ? 40
         : op == GE_ENCODE || op == GE_ENCODE_CALL || op == GE_WELLFORMED ? 8
         : op == GE_GROUP_KC ? 8 * KC_GMAX
         : op == GE_GROUP_SIGN ? 8 * SIGN_GMAX
         : op == GE_GROUP_SIGN2 ? 16 * SIGN_GMAX
         : op == GE_TO_PRECOMP || op == GE_CT_SELECT ? 24
         : op == GE_AFFINE_RUN || op == GE_AFFINE_RUN_CALL ? 64 * 24 + 32
         : op == GE_AFFINE_FWDBWD ? KR_SLICE * 24 + 32
         : op == GE_KEY_ROWS ? 8 + 2 * COMB_COLS * 24
         : op == GE_RECODE ? 80
         : 32;
}
// per-item scratch in global memory: the key chain's COMB_ROWS x KB_PTS points
AFC_HHD constexpr int ge_scratch_words(int op) { return op == GE_KEY_ROWS ? COMB_ROWS * KB_PTS * 32 : 0; }

AFC_HD void load_p3(ge_p3& p, const uint32_t* w) {
    fe_from_words(p.X, w); fe_from_words(p.Y, w + 8); fe_from_words(p.Z, w + 16); fe_from_words(p.T, w + 24);
}
AFC_HD void store_fe(uint32_t* w, const fe& f) {
#pragma unroll
    for (int i = 0; i < 8; i++) w[i] = f.v[i];
}
AFC_HD void store_p3(uint32_t* w, const ge_p3& p) { store_fe(w, p.X); store_fe(w + 8, p.Y); store_fe(w + 16, p.Z); store_fe(w + 24, p.T); }
AFC_HD void store_pre(uint32_t* w, const ge_precomp& e) { store_fe(w, e.ypx); store_fe(w + 8, e.ymx); store_fe(w + 16, e.xy2d); }
AFC_HD void zero_words(uint32_t* w, int n) {
    for (int i = 0; i < n; i++) w[i] = 0;
}

template <class F, int GMAX>
AFC_HD int run_group(const uint32_t* in, uint32_t* out) {
    const int G = (int)in[0];
    if (G < 1 || G > GMAX) return 1;
    fe X[GMAX], Y[GMAX], Z[GMAX];
    for (int g = 0; g < GMAX; g++) {                 // members past G are loaded too (and must not matter)
        fe_from_words(X[g], in + 8 + 24 * g); fe_from_words(Y[g], in + 16 + 24 * g); fe_from_words(Z[g], in + 24 + 24 * g);
    }
    uint32_t enc[GMAX][8];
    ge_encode_group<F, GMAX>(enc, X, Y, Z, G);
    zero_words(out, 8 * GMAX);
    for (int g = 0; g < G; g++)
        for (int w = 0; w < 8; w++) out[8 * g + w] = enc[g][w];
    return 0;
}

// ge_affine_run_fwd, one inversion, ge_affine_run_bwd: a k_kc_rows slice with the CTA's shared inversion replaced by the
// single-thread one
template <class FR, class FC, int CH>
AFC_HD void run_slice(ge_precomp* out, ge_p3& M, const ge_cached& c) {
    fe X[CH], Y[CH], Z[CH], Pz[CH];
    ge_affine_run_fwd<FR, CH>(X, Y, Z, Pz, M, c);
    fe inv;
    fe_invert<FC>(inv, Pz[CH - 1]);
    ge_affine_run_bwd<FR, CH>(out, X, Y, Z, Pz, inv);
}

// Runs OP on one item.  PORTABLE runs every field multiplication through the portable twins (FePortable): the device's own
// reference for the bulk runs.  Operations without field multiplications run the same code either way.  Returns 0, or 1 for
// an item outside the operation's domain (a group size, row, stage count or recoding kind that does not exist).
template <int OP, bool PORTABLE>
AFC_HD int run_op(const uint32_t* in, uint32_t* out, uint32_t* scratch) {
    using FI = std::conditional_t<PORTABLE, FePortable, FeInline>;
    using FC = std::conditional_t<PORTABLE, FePortable, GeCall>;
    using F = std::conditional_t<OP == GE_ENCODE_CALL || OP == GE_DBL_CALL || OP == GE_ADDSUB_CALL || OP == GE_SMALL_MULT_CALL ||
                                 OP == GE_AFFINE_RUN_CALL, FC, FI>;
    ge_p3 P, Q;
    ge_p1p1 t;
    if constexpr (OP == GE_DECODE) {
        const int ok = ge_frombytes<F>(P, in);
        store_p3(out, P);
        out[32] = (uint32_t)ok;
        zero_words(out + 33, 7);
    } else if constexpr (OP == GE_ENCODE || OP == GE_ENCODE_CALL) {
        load_p3(P, in);
        ge_encode<F>(out, P.X, P.Y, P.Z);
    } else if constexpr (OP == GE_GROUP_KC) {
        return run_group<FI, KC_GMAX>(in, out);
    } else if constexpr (OP == GE_GROUP_SIGN) {
        return run_group<FC, SIGN_GMAX>(in, out);
    } else if constexpr (OP == GE_GROUP_SIGN2) {
        return run_group<FC, 2 * SIGN_GMAX>(in, out);
    } else if constexpr (OP == GE_DBL || OP == GE_DBL_CALL) {
        load_p3(P, in);
        ge_dbl<F>(t, P.X, P.Y, P.Z);
        ge_p1p1_to_p3<F>(Q, t);
        store_p3(out, Q);
    } else if constexpr (OP == GE_ADDSUB || OP == GE_ADDSUB_CALL) {
        load_p3(P, in);
        load_p3(Q, in + 32);
        ge_cached c;
        ge_p3_to_cached<F>(c, Q);
        ge_addsub<F>(t, P, c, (int)(in[64] & 1u));
        ge_p1p1_to_p3<F>(Q, t);
        store_p3(out, Q);
    } else if constexpr (OP == GE_TO_PRECOMP) {
        load_p3(P, in);
        ge_precomp e;
        ge_p3_to_precomp<F>(e, P);
        store_pre(out, e);
    } else if constexpr (OP == GE_MADD) {
        load_p3(P, in);
        const ge_precomp* src = (const ge_precomp*)(in + 32);
        const int neg = (int)(in[56] & 1u);
        if (in[57] & 1u) {
            ge_precomp e;
            ge_load_precomp_arranged(e, src, neg);
            ge_madd_arranged<F>(t, P, e, neg);
        } else {
            ge_maddsub<F>(t, P, *src, neg);
        }
        ge_p1p1_to_p3<F>(Q, t);
        store_p3(out, Q);
    } else if constexpr (OP == GE_CT_SELECT) {
        ge_precomp e;
        ge_ct_select(e, (const ge_precomp*)in, (int)in[192]);
        store_pre(out, e);
    } else if constexpr (OP == GE_SMALL_MULT || OP == GE_SMALL_MULT_CALL) {
        load_p3(P, in);
        ge_cached c;
        ge_p3_to_cached<F>(c, P);
        ge_small_multiple<F>(Q, P, c, in[32]);
        store_p3(out, Q);
    } else if constexpr (OP == GE_AFFINE_RUN || OP == GE_AFFINE_RUN_CALL) {
        load_p3(P, in);
        load_p3(Q, in + 32);
        ge_cached c;
        ge_p3_to_cached<F>(c, Q);
        ge_affine_run<F, 64>((ge_precomp*)out, P, c);
        store_p3(out + 64 * 24, P);
    } else if constexpr (OP == GE_AFFINE_FWDBWD) {
        load_p3(P, in);
        load_p3(Q, in + 32);
        ge_cached c;
        ge_p3_to_cached<FC>(c, Q);
        run_slice<FI, FC, KR_SLICE>((ge_precomp*)out, P, c);
        store_p3(out + KR_SLICE * 24, P);
    } else if constexpr (OP == GE_KEY_ROWS) {
        const int row = (int)in[8], stages = (int)in[9];
        if (row < 0 || row >= COMB_ROWS || (stages != 1 && stages != 2 && stages != 4)) return 1;
        ge_p3* bases3 = (ge_p3*)scratch;
        const int nr = COMB_ROWS / stages;
        int ok1 = 0;
        for (int s = 0; s * nr <= row; s++) {        // k_kc_chain, stage by stage, up to the stage holding `row`
            const int ok = ge_key_chain_stage<FI>(bases3, in, s * nr, nr);
            if (s == 0) ok1 = ok;
        }
        ge_precomp* tab = (ge_precomp*)(out + 8);
        for (int part = 0; part < KR_PARTS; part++) {  // k_kc_rows: one slice per thread
            ge_cached c;
            ge_key_slice_start<FC, KR_PARTS>(P, c, bases3 + row * KB_PTS, part);
            run_slice<FI, FC, KR_SLICE>(tab + part * KR_SLICE, P, c);
        }
        const int ok2 = ge_build_key_row<FI>(tab + COMB_COLS, in, row);
        out[0] = (uint32_t)ok1;
        out[1] = (uint32_t)ok2;
        zero_words(out + 2, 6);
    } else if constexpr (OP == GE_RECODE) {
        const int kind = (int)in[8];
        uint32_t t8[8];
        zero_words(out, 80);
        if (kind == 0) {
            sc_recode16(t8, in);
            for (int i = 0; i < 64; i++) out[8 + i] = (uint32_t)sc_digit16(t8, i);
        } else if (kind == 1) {
            sc_recode256(t8, in);
            for (int i = 0; i < 32; i++) out[8 + i] = (uint32_t)sc_digit256(t8, i);
        } else if (kind == 2) {
            sc_recode65536(t8, in);
            for (int i = 0; i < 16; i++) out[8 + i] = (uint32_t)sc_digit65536(t8, i);
        } else if (kind >= 16 && kind <= 22) {
            uint32_t c[8];
            sc_wide_offset(c, kind);
            sc_recode_wide(t8, in, c);
            const int rows = sc_wide_rows(kind);
            for (int i = 0; i < rows; i++) out[8 + i] = (uint32_t)sc_digit_wide(t8, i, kind, rows);
            out[72] = (uint32_t)base_table_top_max(kind);
            const uint64_t e = (uint64_t)base_table_entries(kind);
            out[73] = (uint32_t)e;
            out[74] = (uint32_t)(e >> 32);
        } else {
            return 1;
        }
        for (int i = 0; i < 8; i++) out[i] = t8[i];
    } else if constexpr (OP == GE_WELLFORMED) {
        zero_words(out, 8);
        out[0] = (uint32_t)ed25519_sig_wellformed(in);
    } else {
        return 1;
    }
    return 0;
}

}  // namespace gesim
