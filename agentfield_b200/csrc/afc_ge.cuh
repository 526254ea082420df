// Edwards25519 group arithmetic and the per-credential Ed25519 routines (RFC 8032 §5.1, with the exact
// accept/reject behaviour of Go 1.24 crypto/ed25519 — SURVEY.md §8a rows E1/E2).
//
// Replaces, per credential, the body of ed25519.Verify / ed25519.Sign / ed25519.NewKeyFromSeed that the
// reference calls at vc_service.go:460,463,504,712,715,1624, did_service.go:523 and
// cli/vc_verification_enhanced.go:453.
//
// GPU shape (differs from Go's variable-time NAF on purpose): every lane of a warp must run the same
// instruction stream, so the double-scalar multiplication R' = [S]B + [k](-A) uses FIXED signed radix-16
// windows over one shared doubling chain (Straus): 252 doublings, 64 additions from a per-credential table of
// 8 cached multiples of -A (4-bit digits, thread-local), and 32 mixed additions from a 128-entry affine table of
// B (8-bit digits, 12 KB staged in shared memory).  Results are bit-identical to Go's because
// both compute the same group element and compare canonical encodings.
#pragma once
#include "afc_fe.cuh"
#include "afc_sc.cuh"

namespace afc {

struct ge_p3 { fe X, Y, Z, T; };
struct ge_p2 { fe X, Y, Z; };
struct ge_p1p1 { fe X, Y, Z, T; };
struct ge_cached { fe YpX, YmX, Z, T2d; };
struct ge_precomp { fe ypx, ymx, xy2d; };

AFC_HD void fe_const(fe& h, const uint32_t* c) {
#pragma unroll
    for (int i = 0; i < 8; i++) h.v[i] = c[i];
}


AFC_HD void ge_p3_0(ge_p3& h) { fe_0(h.X); fe_1(h.Y); fe_1(h.Z); fe_0(h.T); }
template <class F = FeInline>
AFC_HD void ge_p1p1_to_p2(ge_p2& r, const ge_p1p1& p) { F::mul(r.X, p.X, p.T); F::mul(r.Y, p.Y, p.Z); F::mul(r.Z, p.Z, p.T); }
template <class F = FeInline>
AFC_HD void ge_p1p1_to_p3(ge_p3& r, const ge_p1p1& p) {
    F::mul(r.X, p.X, p.T); F::mul(r.Y, p.Y, p.Z); F::mul(r.Z, p.Z, p.T); F::mul(r.T, p.X, p.Y);
}
template <class F = FeInline>
AFC_HD void ge_p3_to_cached(ge_cached& r, const ge_p3& p) {
    fe d2; fe_const(d2, AFC_D2_32);
    fe_add(r.YpX, p.Y, p.X); fe_sub(r.YmX, p.Y, p.X); fe_copy(r.Z, p.Z); F::mul(r.T2d, p.T, d2);
}
// r = 2 * (X:Y:Z)
template <class F = FeInline>
AFC_HD void ge_dbl(ge_p1p1& r, const fe& X, const fe& Y, const fe& Z) {
    fe xx, yy, b, a;
    F::sq(xx, X); F::sq(yy, Y); F::sq(b, Z); fe_dbl(b, b);
    fe_add(a, X, Y); F::sq(a, a);
    fe_add(r.Y, yy, xx); fe_sub(r.Z, yy, xx); fe_sub(r.X, a, r.Y); fe_sub(r.T, b, r.Z);
}
AFC_HD void fe_select(fe& h, const fe& a, const fe& b, int pick_b) {
    uint32_t m = 0u - (uint32_t)(pick_b != 0);
#pragma unroll
    for (int i = 0; i < 8; i++) h.v[i] = (a.v[i] & ~m) | (b.v[i] & m);
}
// r = p + q (neg = 0) or p - q (neg = 1)
template <class F = FeInline>
AFC_HD void ge_addsub(ge_p1p1& r, const ge_p3& p, const ge_cached& q, int neg) {
    fe a, b, c, d, qa, qb;
    fe_select(qa, q.YpX, q.YmX, neg);
    fe_select(qb, q.YmX, q.YpX, neg);
    fe_add(a, p.Y, p.X); fe_sub(b, p.Y, p.X);
    F::mul(a, a, qa); F::mul(b, b, qb); F::mul(c, q.T2d, p.T); F::mul(d, p.Z, q.Z); fe_dbl(d, d);
    fe_sub(r.X, a, b); fe_add(r.Y, a, b);
    fe dpc, dmc;
    fe_add(dpc, d, c); fe_sub(dmc, d, c);
    fe_select(r.Z, dpc, dmc, neg); fe_select(r.T, dmc, dpc, neg);
}
// One 96-byte table entry from global memory as six 128-bit loads (entries are 32-byte aligned: the tables come from cudaMalloc
// and sizeof(ge_precomp) = 96).  Each lane gathers its own entry, so what a load costs is its line accesses, not its width: left
// to the compiler a `const ge_precomp&` becomes 24 LDG.32 — 768 L1 accesses per warp and mixed addition, more L1 time than the
// addition has IMAD.WIDE time.
#ifndef AFC_TABLE_LOAD256
#define AFC_TABLE_LOAD256 1
#endif
AFC_HD void ge_load_precomp(ge_precomp& e, const ge_precomp* src) {
#if AFC_DEVICE_CODE && AFC_TABLE_LOAD256
    const uint32_t* p = (const uint32_t*)src;
    ldg_nc_32B(e.ypx.v, p);
    ldg_nc_32B(e.ymx.v, p + 8);
    ldg_nc_32B(e.xy2d.v, p + 16);
#else
    e = *src;
#endif
}
// The same entry already arranged for subtraction when neg != 0 — ypx and ymx change places at LOAD time (an address, not 16
// selects per addition); what is left of the sign is the exchange of the two outputs in ge_madd_arranged.
AFC_HD void ge_load_precomp_arranged(ge_precomp& e, const ge_precomp* src, int neg) {
#if AFC_DEVICE_CODE && AFC_TABLE_LOAD256
    const uint32_t* p = (const uint32_t*)src;
    const uint32_t* pa = p + (neg ? 8 : 0);
    const uint32_t* pb = p + (neg ? 0 : 8);
    ldg_nc_32B(e.ypx.v, pa);
    ldg_nc_32B(e.ymx.v, pb);
    ldg_nc_32B(e.xy2d.v, p + 16);
#else
    e = *src;
    if (neg) { fe t = e.ypx; e.ypx = e.ymx; e.ymx = t; }
#endif
}
template <class F = FeInline>
AFC_HD void ge_madd_arranged(ge_p1p1& r, const ge_p3& p, const ge_precomp& q, int neg) {
    fe a, b, c, d;
    fe_add(a, p.Y, p.X); fe_sub(b, p.Y, p.X);
    F::mul(a, a, q.ypx); F::mul(b, b, q.ymx); F::mul(c, q.xy2d, p.T); fe_dbl(d, p.Z);
    fe_sub(r.X, a, b); fe_add(r.Y, a, b);
    fe dpc, dmc;
    fe_add(dpc, d, c); fe_sub(dmc, d, c);
    fe_select(r.Z, dpc, dmc, neg); fe_select(r.T, dmc, dpc, neg);
}
// mixed addition with an affine precomputed point
template <class F = FeInline>
AFC_HD void ge_maddsub(ge_p1p1& r, const ge_p3& p, const ge_precomp& q, int neg) {
    fe a, b, c, d, qa, qb;
    fe_select(qa, q.ypx, q.ymx, neg);
    fe_select(qb, q.ymx, q.ypx, neg);
    fe_add(a, p.Y, p.X); fe_sub(b, p.Y, p.X);
    F::mul(a, a, qa); F::mul(b, b, qb); F::mul(c, q.xy2d, p.T); fe_dbl(d, p.Z);
    fe_sub(r.X, a, b); fe_add(r.Y, a, b);
    fe dpc, dmc;
    fe_add(dpc, d, c); fe_sub(dmc, d, c);
    fe_select(r.Z, dpc, dmc, neg); fe_select(r.T, dmc, dpc, neg);
}
// ---- the same mixed addition on FOUR lanes (k_ed_verify_quad) -------------------------------------------------------------
// Lane `role` of a quad owns one coordinate of the running point (0 X, 1 Y, 2 Z, 3 T) and does 2 of the 7 (+1 idle)
// multiplications; everything else it needs arrives by shuffle from lane q0 + src.  One step is
//   stage 1   u = own ± (shfl(own, src1) & keep1)        X - Y | Y + X | Z + Z | T + 0
//   round 1   m = u * v, v = the lane's 32 bytes of the table entry (or 1)         -A' | B' | D | C      (A', B', C, D of ge_maddsub)
//   stage 2   w = shfl(m, srcA2) ± shfl(m, srcB2)        F = D∓C | H = B'+A' | G = D±C | E = B'-A'      (signs follow `neg`)
//   round 2   own = w * shfl(w, src3)                    X3 = F E | Y3 = H G | Z3 = G F | T3 = E H
// so the layout is the same after every step.  Signs are masks for fe_addsub_m (0: add, ~0: subtract).  The plan is plain data
// so that tests/hostsim can replay the four lanes on the CPU against ge_maddsub + ge_p1p1_to_p3.
struct quad_plan { int src1, srcA2, srcB2, src3; uint32_t keep1, sgn1, sgn2, v_off; int v_load; };
AFC_HD quad_plan ge_quad_plan(int role, int neg) {
    quad_plan p;
    const uint32_t nm = 0u - (uint32_t)(neg != 0);
    p.src1 = role == 0 ? 1 : role == 1 ? 0 : role;
    p.keep1 = role == 3 ? 0u : 0xffffffffu;
    p.sgn1 = role == 0 ? 0xffffffffu : 0u;
    p.srcA2 = (role & 1) ? 1 : 2;
    p.srcB2 = (role & 1) ? 0 : 3;
    p.sgn2 = role == 0 ? ~nm : role == 1 ? 0xffffffffu : role == 2 ? nm : 0u;
    p.src3 = role == 0 ? 3 : role == 1 ? 2 : role == 2 ? 0 : 1;
    // bytes into the 96-byte entry {ypx, ymx, xy2d}: the X lane multiplies by ymx (ypx when subtracting), the Y lane the other way round
    p.v_off = role == 3 ? 64u : (((uint32_t)(role == 0) ^ (uint32_t)(neg != 0)) ? 32u : 0u);
    p.v_load = role != 2;
    return p;
}
// what a lane multiplies by when it has nothing to load: 1 (Z lane; digit 0 on the X and Y lanes) or 0 (digit 0 on the T lane)
AFC_HD void ge_quad_neutral(fe& v, int role) { fe_0(v); v.v[0] = role == 3 ? 0u : 1u; }

template <class F = FeInline>
AFC_HD void ge_p3_to_precomp(ge_precomp& r, const ge_p3& p) {
    fe zi, x, y, xy, d2;
    fe_const(d2, AFC_D2_32);
    fe_invert<F>(zi, p.Z); F::mul(x, p.X, zi); F::mul(y, p.Y, zi);
    fe_add(r.ypx, y, x); fe_sub(r.ymx, y, x); F::mul(xy, x, y); F::mul(r.xy2d, xy, d2);
}
// canonical 32-byte encoding as little-endian words (Point.Bytes)
template <class F = FeInline>
AFC_HD void ge_encode(uint32_t* out, const fe& X, const fe& Y, const fe& Z) {
    fe zi, x, y;
    fe_invert<F>(zi, Z); F::mul(x, X, zi); F::mul(y, Y, zi);
    fe_towords(out, y);
    out[7] |= (uint32_t)fe_isnegative(x) << 31;
}
// Point.SetBytes: 1 on success, 0 if the encoding is not on the curve.  Non-canonical y and
// "x = 0 with sign bit" are accepted exactly as Go does.
template <class F = FeInline>
AFC_HD int ge_frombytes(ge_p3& h, const uint32_t* enc) {
    fe u, v, v3, vxx, one, dd, sm1;
    fe_1(one); fe_const(dd, AFC_D_32); fe_const(sm1, AFC_SQRTM1_32);
    fe_frombytes_words(h.Y, enc);
    fe_1(h.Z);
    F::sq(u, h.Y); F::mul(v, u, dd);
    fe_sub(u, u, one);                      // u = y^2 - 1
    fe_add(v, v, one);                      // v = d y^2 + 1
    F::sq(v3, v); F::mul(v3, v3, v);        // v^3
    F::sq(h.X, v3); F::mul(h.X, h.X, v); F::mul(h.X, h.X, u);   // u v^7
    fe_pow22523<F>(h.X, h.X);
    F::mul(h.X, h.X, v3); F::mul(h.X, h.X, u);                   // r = u v^3 (u v^7)^((p-5)/8)
    F::sq(vxx, h.X); F::mul(vxx, vxx, v);                        // v r^2
    int ok_pos = fe_equal(vxx, u);
    fe nu; fe_neg(nu, u);
    int ok_neg = fe_equal(vxx, nu);
    fe xi; F::mul(xi, h.X, sm1);
    fe_select(h.X, h.X, xi, ok_neg & !ok_pos);
    int flip = fe_isnegative(h.X) != (int)(enc[7] >> 31);
    fe nx; fe_neg(nx, h.X);
    fe_select(h.X, h.X, nx, flip);
    F::mul(h.T, h.X, h.Y);
    return ok_pos | ok_neg;
}

// Table of multiples of the base point, built on the device at afc_init (k_ed_build_tables), radix 2^W (W = AFC_BASE_WINDOW):
//   base[i][j] = (j+1) * 2^(W i) * B     i = 0..256/W-1, j = 0..2^(W-1)-1     affine precomputed form, 96 B per entry
//   W = 16 (default): 16 x 32768 entries = 48 MB.  A fixed-base multiplication is 16 mixed additions with signed 16-bit
//                     digits; every lane reads its own 96-byte entry (L2 / HBM gathers, like the per-issuer tables).
//   W = 8:            32 x 128 entries = 384 KB, 32 mixed additions (the first build of this library; kept for A/B runs).
// Row 0 starts with the 128 small multiples of B (12 KB) that the generic Straus kernel stages in shared memory.
// The per-issuer tables of -A stay radix 256 (COMB_ROWS x COMB_COLS): their build cost is paid per key, not per process.
#ifndef AFC_BASE_WINDOW
#define AFC_BASE_WINDOW 16
#endif
static constexpr int COMB_ROWS = 32, COMB_COLS = 128;
static constexpr int BASE_W = AFC_BASE_WINDOW, BASE_ROWS = 256 / BASE_W, BASE_COLS = 1 << (BASE_W - 1);
static constexpr int BASE_CHUNK = 64;            // entries per thread at build time (one field inversion per chunk)
static_assert(BASE_W == 8 || BASE_W == 16, "base-point window must be 8 or 16 bits");
static_assert(BASE_COLS % BASE_CHUNK == 0 && BASE_COLS >= COMB_COLS, "chunking");

AFC_HD void sc_recode_base(uint32_t* t, const uint32_t* s) { if (BASE_W == 16) sc_recode65536(t, s); else sc_recode256(t, s); }
AFC_HD int sc_digit_base(const uint32_t* t, int i) { return BASE_W == 16 ? sc_digit65536(t, i) : sc_digit256(t, i); }

// The fixed-base table the table-driven verify reads (ed25519_keyed_point), radix 2^w for w in 16..22 (sc_recode_wide):
//   tab[i][j] = (j+1) * 2^(w i) * B     rows i = 0..rows-1 of 2^(w-1) entries each; the top row holds only as many entries as its
//   digit can reach (base_table_entries rounds them up to whole build chunks).
// At w = 16 this is the radix-65536 table above, shared with signing; wider tables are verify-only, allocated per context at its
// first table-driven verify.  Passed to the kernels by value: the recoding offset is a kernel parameter, not a register.
struct base_table { const ge_precomp* tab; uint32_t offset[8]; int w, rows; };
AFC_HHD base_table base_table_make(const ge_precomp* tab, int w) {
    base_table b;
    b.tab = tab; b.w = w; b.rows = sc_wide_rows(w);
    sc_wide_offset(b.offset, w);
    return b;
}
// largest top-row digit of any S < 2^253 (every canonical S < L): what the top row must hold
AFC_HHD int base_table_top_max(int w) {
    uint32_t c[8], s[8], t[8];
    sc_wide_offset(c, w);
    for (int i = 0; i < 8; i++) s[i] = i < 7 ? 0xffffffffu : 0x1fffffffu;
    sc_recode_wide(t, s, c);
    return sc_digit_wide(t, sc_wide_rows(w) - 1, w, sc_wide_rows(w));
}
AFC_HHD size_t base_table_entries(int w) {
    const size_t top = ((size_t)base_table_top_max(w) + BASE_CHUNK - 1) / BASE_CHUNK * BASE_CHUNK;
    return (size_t)(sc_wide_rows(w) - 1) * ((size_t)1 << (w - 1)) + top;
}

// out[j] = affine precomputed form of M + j P for j = 0..CH-1, with ONE field inversion (Montgomery's trick); on return
// M has advanced to M + CH P.  c = P in cached form.  Scratch: 4 CH field elements of thread-local memory.
template <class F, int CH>
AFC_HD void ge_affine_run(ge_precomp* out, ge_p3& M, const ge_cached& c) {
    fe X[CH], Y[CH], Z[CH], Pz[CH];
    ge_p1p1 t;
    fe d2; fe_const(d2, AFC_D2_32);
#pragma unroll 1
    for (int j = 0; j < CH; j++) {
        fe_copy(X[j], M.X); fe_copy(Y[j], M.Y); fe_copy(Z[j], M.Z);
        if (j == 0) fe_copy(Pz[0], M.Z); else F::mul(Pz[j], Pz[j - 1], M.Z);
        ge_addsub<F>(t, M, c, 0); ge_p1p1_to_p3<F>(M, t);
    }
    fe inv; fe_invert<F>(inv, Pz[CH - 1]);               // 1 / (Z_0 ... Z_{CH-1})
#pragma unroll 1
    for (int j = CH - 1; j >= 0; j--) {
        fe zi;
        if (j > 0) { F::mul(zi, inv, Pz[j - 1]); F::mul(inv, inv, Z[j]); } else fe_copy(zi, inv);
        fe x, y, xy;
        F::mul(x, X[j], zi); F::mul(y, Y[j], zi);
        ge_precomp& r = out[j];
        fe_add(r.ypx, y, x); fe_sub(r.ymx, y, x); F::mul(xy, x, y); F::mul(r.xy2d, xy, d2);
    }
}

// M = m P for 1 <= m < 2^22, left-to-right double-and-add.  c = P in cached form.
template <class F = FeInline>
AFC_HD void ge_small_multiple(ge_p3& M, const ge_p3& P, const ge_cached& c, uint32_t m) {
    ge_p1p1 t;
    int started = 0;
    M = P;
#pragma unroll 1
    for (int bit = 21; bit >= 0; bit--) {
        if (started) { ge_dbl<F>(t, M.X, M.Y, M.Z); ge_p1p1_to_p3<F>(M, t); }
        if ((m >> bit) & 1) {
            if (started) { ge_addsub<F>(t, M, c, 0); ge_p1p1_to_p3<F>(M, t); }
            else { M = P; started = 1; }
        }
    }
}

// One chunk of a base-point table of radix 2^w per thread: out[0..BASE_CHUNK) = (j0+1 .. j0+BASE_CHUNK) * 2^(w i) * B.
template <class F = FeInline>
AFC_HD void ge_build_base_chunk(ge_precomp* out, int i, int j0, int w = BASE_W) {
    ge_p3 P, M;
    fe_const(P.X, AFC_BX_32); fe_const(P.Y, AFC_BY_32); fe_1(P.Z); F::mul(P.T, P.X, P.Y);
    ge_p1p1 t;
#pragma unroll 1
    for (int k = 0; k < w * i; k++) { ge_dbl<F>(t, P.X, P.Y, P.Z); ge_p1p1_to_p3<F>(P, t); }
    ge_cached c;
    ge_p3_to_cached<F>(c, P);
    ge_small_multiple<F>(M, P, c, (uint32_t)j0 + 1);
    ge_affine_run<F, BASE_CHUNK>(out, M, c);
}

// h = a * B for a reduced scalar a (< 2^253): one mixed addition per signed radix-2^W digit, no doublings.
template <class F = FeInline>
AFC_HD void ge_scalarmult_base(ge_p3& h, const uint32_t* a, const ge_precomp* base) {
    uint32_t t[8];
    sc_recode_base(t, a);
    ge_p3_0(h);
#pragma unroll 1
    for (int i = 0; i < BASE_ROWS; i++) {
        int d = sc_digit_base(t, i);
#if AFC_DEVICE_CODE
        if (BASE_W == 16 && i + 1 < BASE_ROWS) {       // the next entry is a random 96-byte read: start it now
            int nd = sc_digit_base(t, i + 1), nm = nd < 0 ? -nd : nd;
            if (nm) { const char* p = (const char*)&base[(size_t)(i + 1) * BASE_COLS + (nm - 1)]; asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); asm volatile("prefetch.global.L1 [%0];" ::"l"(p + 95)); }
        }
#endif
        if (d != 0) {
            int neg = d < 0;
            int m = neg ? -d : d;
            ge_p1p1 r;
            ge_precomp e;
            ge_load_precomp(e, &base[(size_t)i * BASE_COLS + (m - 1)]);
            ge_maddsub<F>(r, h, e, neg);
            ge_p1p1_to_p3<F>(h, r);
        }
    }
}

// ---- constant-time fixed-base multiplication, for SECRET scalars (signing nonces r and private scalars s) --------------------
// ge_scalarmult_base above gathers table entries at addresses made of the scalar's digits and skips zero digits: fine for
// public scalars (verification), a cache/timing side channel for secret ones — Go's crypto/ed25519, which signing replaces
// (vc_service.go:460-463), selects table entries in constant time.  The constant-time path: signed radix 16, 64 rows of 8
// multiples (48 KB, staged in shared memory by the kernels), EVERY entry of a row read for every digit and one kept by mask,
// no branch and no address that depends on the scalar; a zero digit adds the neutral element.
//   ct16[i][j] = (j+1) 16^i B — all 512 entries already exist in the radix-65536 table: base[i/4][16^(i%4) (j+1) - 1].
static constexpr int CT_ROWS = 64, CT_COLS = 8;
AFC_HD size_t ge_ct16_source(int i, int j) { return (size_t)(i >> 2) * BASE_COLS + (((size_t)(j + 1)) << (4 * (i & 3))) - 1; }
AFC_HD void ge_ct_select(ge_precomp& e, const ge_precomp* row, int d) {
    const uint32_t neg = (uint32_t)(d >> 31);                              // all ones iff d < 0
    const uint32_t m = ((uint32_t)d ^ neg) - neg;                          // |d| in 0..8
    fe_1(e.ypx); fe_1(e.ymx); fe_0(e.xy2d);                                // d = 0: the neutral element in precomputed form
#pragma unroll
    for (int j = 0; j < CT_COLS; j++) {
        const uint32_t mask = 0u - (uint32_t)(m == (uint32_t)(j + 1));
#pragma unroll
        for (int w = 0; w < 8; w++) {
            e.ypx.v[w] ^= (e.ypx.v[w] ^ row[j].ypx.v[w]) & mask;
            e.ymx.v[w] ^= (e.ymx.v[w] ^ row[j].ymx.v[w]) & mask;
            e.xy2d.v[w] ^= (e.xy2d.v[w] ^ row[j].xy2d.v[w]) & mask;
        }
    }
    fe nx; fe_neg(nx, e.xy2d);
#pragma unroll
    for (int w = 0; w < 8; w++) {                                          // -P: swap y+x and y-x, negate 2dxy
        const uint32_t t = (e.ypx.v[w] ^ e.ymx.v[w]) & neg;
        e.ypx.v[w] ^= t; e.ymx.v[w] ^= t;
        e.xy2d.v[w] ^= (e.xy2d.v[w] ^ nx.v[w]) & neg;
    }
}
template <class F = FeInline>
AFC_HD void ge_scalarmult_base_ct(ge_p3& h, const uint32_t* a, const ge_precomp* ct16) {
    uint32_t t[8];
    sc_recode16(t, a);                                                     // 64 signed digits in [-8, 7]
    ge_p3_0(h);
#pragma unroll 1
    for (int i = 0; i < CT_ROWS; i++) {
        ge_precomp e;
        ge_ct_select(e, ct16 + i * CT_COLS, sc_digit16(t, i));
        ge_p1p1 r;
        ge_maddsub<F>(r, h, e, 0);
        ge_p1p1_to_p3<F>(h, r);
    }
}

// Canonical encodings of G projective points with ONE field inversion (Montgomery's trick).  Every Z must be non-zero
// (true for any point on the curve: the a = -1 twisted Edwards addition law is complete).
template <class F, int G>
AFC_HD void ge_encode_many(uint32_t (*enc)[8], const fe* X, const fe* Y, const fe* Z) {
    fe pz[G];
    fe_copy(pz[0], Z[0]);
#pragma unroll
    for (int g = 1; g < G; g++) F::mul(pz[g], pz[g - 1], Z[g]);
    fe inv; fe_invert<F>(inv, pz[G - 1]);
#pragma unroll
    for (int g = G - 1; g >= 0; g--) {
        fe zi;
        if (g > 0) { F::mul(zi, inv, pz[g - 1]); F::mul(inv, inv, Z[g]); } else fe_copy(zi, inv);
        fe x, y;
        F::mul(x, X[g], zi); F::mul(y, Y[g], zi);
        fe_towords(enc[g], y);
        enc[g][7] |= (uint32_t)fe_isnegative(x) << 31;
    }
}

// The same with a run-time count G <= GMAX (the table-driven kernels choose G per launch).
template <class F, int GMAX>
AFC_HD void ge_encode_group(uint32_t (*enc)[8], const fe* X, const fe* Y, const fe* Z, int G) {
    fe pz[GMAX];
    fe_copy(pz[0], Z[0]);
#pragma unroll 1
    for (int g = 1; g < G; g++) F::mul(pz[g], pz[g - 1], Z[g]);
    fe inv; fe_invert<F>(inv, pz[G - 1]);
#pragma unroll 1
    for (int g = G - 1; g >= 0; g--) {
        fe zi;
        if (g > 0) { F::mul(zi, inv, pz[g - 1]); F::mul(inv, inv, Z[g]); } else fe_copy(zi, inv);
        fe x, y;
        F::mul(x, X[g], zi); F::mul(y, Y[g], zi);
        fe_towords(enc[g], y);
        enc[g][7] |= (uint32_t)fe_isnegative(x) << 31;
    }
}

// Go's checks that do not involve the curve: sig[63] & 224 == 0 and S canonical
AFC_HD int ed25519_sig_wellformed(const uint32_t* sig) { return !(sig[15] & 0xE0000000u) && sc_is_canonical(sig + 8); }

// ---------------------------------------------------------------------------------- verify core
// pk, sig: little-endian words of the given byte strings; k = SHA-512(R || A || M) mod L.
// Returns 1 iff Go's ed25519.Verify would return true.
// Returns 1 iff Go's ed25519.Verify would return true.  (A split into point + shared-inversion finish, as the table-driven
// kernels use, was tried on this kernel and dropped: ptxas allocates far fewer registers to it and the Straus loop runs
// slower.)
template <class F = FeInline>
AFC_HD int ed25519_verify_core(const uint32_t* pk, const uint32_t* sig, const uint32_t* k, const ge_precomp* b128) {
    int ok = 1;
    if (sig[15] & 0xE0000000u) ok = 0;                 // sig[63] & 224 != 0
    if (!sc_is_canonical(sig + 8)) ok = 0;             // S >= L
    ge_p3 A;
    if (!ge_frombytes<F>(A, pk)) ok = 0;
    fe_neg(A.X, A.X); fe_neg(A.T, A.T);                // -A
    ge_cached tab[8];                                  // (j+1)(-A)
    ge_p3_to_cached<F>(tab[0], A);
    {
        ge_p3 m; ge_p1p1 t;
        ge_dbl<F>(t, A.X, A.Y, A.Z); ge_p1p1_to_p3<F>(m, t);  // 2(-A)
        ge_p3_to_cached<F>(tab[1], m);
        for (int j = 2; j < 8; j++) {
            ge_addsub<F>(t, m, tab[0], 0); ge_p1p1_to_p3<F>(m, t);
            ge_p3_to_cached<F>(tab[j], m);
        }
    }
    uint32_t kt[8], st[8];
    sc_recode16(kt, k);
    sc_recode256(st, sig + 8);
    // Straus over one shared doubling chain.  The running point lives in P1xP1 form (t) between steps: it is completed
    // to P3 (4 mul) only right before an addition needs T, and to P2 (3 mul) before doublings.
    ge_p2 q;
    ge_p1p1 t;
    fe_0(t.X); fe_1(t.Y); fe_1(t.Z); fe_1(t.T);            // identity
#pragma unroll 1
    for (int i = 63; i >= 0; i--) {
        if (i != 63) {
#pragma unroll 1
            for (int d = 0; d < 4; d++) {
                ge_p1p1_to_p2<F>(q, t);
                ge_dbl<F>(t, q.X, q.Y, q.Z);
            }
        }
        int dk = sc_digit16(kt, i);
        if (dk != 0) {
            int neg = dk < 0;
            int m = neg ? -dk : dk;
            ge_p3 r;
            ge_p1p1_to_p3<F>(r, t);
            ge_addsub<F>(t, r, tab[m - 1], neg);
        }
        int ds = (i & 1) ? 0 : sc_digit256(st, i >> 1);     // S advances 8 bits every second 4-bit step
        if (ds != 0) {
            int neg = ds < 0;
            int m = neg ? -ds : ds;
            ge_p3 r;
            ge_p1p1_to_p3<F>(r, t);
            ge_maddsub<F>(t, r, b128[m - 1], neg);
        }
    }
    ge_p1p1_to_p2<F>(q, t);
    uint32_t enc[8];
    ge_encode<F>(enc, q.X, q.Y, q.Z);
    uint32_t diff = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) diff |= enc[i] ^ sig[i];
    return ok & (diff == 0);
}


// ---------------------------------------------------------------------------------- keyed verification (identity cache, N1)
// When the verifier already knows the issuer key (the reference resolves every issuer DID from its own registry,
// vc_service.go:259 -> did_service.go:368), a per-key radix-256 table of -A makes the variable-base half as cheap as
// the fixed-base half: R' = sum_i ks_i * (256^i B) + sum_i kk_i * (256^i (-A)) = 64 mixed additions, no doublings.
//
// One row of a key's table per thread: row[j] = (j+1) * 256^i * (-A), affine precomputed form.  Returns 0 if the key
// does not decode (Go: verification with that key is always false).
#ifndef AFC_KEYROW_CHUNK
#define AFC_KEYROW_CHUNK 64      // entries per inversion (8 KB of thread-local scratch): longer chunks, fewer inversions
#endif
// One row from its base point P = 256^i (-A): 128 consecutive multiples, converted to affine one chunk at a time with ONE
// field inversion per chunk (Montgomery's trick): 2 inversions per row instead of 128.
template <class F = FeInline>
AFC_HD void ge_key_row_from_base(ge_precomp* row, const ge_p3& P) {
    ge_cached c;
    ge_p3_to_cached<F>(c, P);
    ge_p3 M = P;
    constexpr int CH = AFC_KEYROW_CHUNK;
#pragma unroll 1
    for (int c0 = 0; c0 < COMB_COLS; c0 += CH) ge_affine_run<F, CH>(row + c0, M, c);
}
// A slice of a row: entries c0 .. c0+CH-1 = (c0+1 .. c0+CH) P, from the row's base point P (several threads per row: the
// slice's start point costs ~7 doublings and an addition, and one more inversion per slice).
template <class F, int CH>
AFC_HD void ge_key_row_slice(ge_precomp* row, const ge_p3& P, int c0) {
    ge_cached c;
    ge_p3_to_cached<F>(c, P);
    ge_p3 M;
    ge_small_multiple<F>(M, P, c, (uint32_t)c0 + 1);
    ge_affine_run<F, CH>(row + c0, M, c);
}
// The 32 row base points of one key, bases[i] = 256^i (-A): ONE doubling chain per key (248 doublings) instead of one per row
// (8 i doublings in row i: 3968 per key, and lanes of a warp that finish at different times).
template <class F = FeInline>
AFC_HD int ge_key_row_bases(ge_p3* bases, const uint32_t* pk) {
    ge_p3 P;
    int ok = ge_frombytes<F>(P, pk);
    fe_neg(P.X, P.X); fe_neg(P.T, P.T);
    ge_p1p1 t;
#pragma unroll 1
    for (int i = 0; i < COMB_ROWS; i++) {
        bases[i] = P;
        if (i + 1 < COMB_ROWS) {
#pragma unroll 1
            for (int k = 0; k < 8; k++) {
                ge_dbl<F>(t, P.X, P.Y, P.Z);
                if (k < 7) { ge_p2 q; ge_p1p1_to_p2<F>(q, t); fe_copy(P.X, q.X); fe_copy(P.Y, q.Y); fe_copy(P.Z, q.Z); }   // T only where it is kept
                else ge_p1p1_to_p3<F>(P, t);
            }
        }
    }
    return ok;
}
// ---- second construction of the per-key tables (round 2): what k_kc_chain / k_kc_rows run.
// (1) The doubling chain is walked in stages of `nr` rows (so that the rows of stage s can be filled while the chain of stage
//     s + 1 is still running) and leaves, per row i, three points in P3 form: P_i = 256^i (-A), 32 P_i and 64 P_i — the chain
//     passes through them anyway (5 and 6 doublings after P_i), keeping them costs one multiplication each (their T).
// (2) Row threads start their slice of 128 / KR_PARTS consecutive multiples from those helpers with at most two additions
//     (instead of a private double-and-add of up to 6 doublings + 2 additions), run forward storing (X, Y, Z, prefix product of Z),
//     take part in ONE field inversion per CTA (a product tree in shared memory, fe_invert_cta in k_ed25519.cu) and convert to
//     affine on the way back: one inversion per NT threads instead of one per thread (265 of the 809 multiplications a
//     32-entry slice used to cost).
static constexpr int KB_PTS = 3;                 // points kept per row by the chain: P, 32 P, 64 P
// Rows [r0, r0 + nr) of one key.  Stage 0 decodes the key; later stages continue from bases3[r0 * KB_PTS] (left there by the
// previous stage).  Returns 1 if the key decodes (meaningful for r0 == 0 only); an undecodable key gets the neutral element so
// that every later product stays well defined (its table is never used: lookups report ok = 0).
template <class F = FeInline>
AFC_HD int ge_key_chain_stage(ge_p3* bases3, const uint32_t* pk, int r0, int nr) {
    ge_p3 P;
    int ok = 1;
    if (r0 == 0) {
        ok = ge_frombytes<F>(P, pk);
        fe_neg(P.X, P.X); fe_neg(P.T, P.T);
        if (!ok) ge_p3_0(P);
    } else {
        P = bases3[r0 * KB_PTS];
    }
    ge_p1p1 t;
#pragma unroll 1
    for (int i = r0; i < r0 + nr; i++) {
        bases3[i * KB_PTS] = P;
        const int last = i + 1 >= COMB_ROWS;
#pragma unroll 1
        for (int k = 0; k < (last ? 6 : 8); k++) {
            ge_dbl<F>(t, P.X, P.Y, P.Z);
            if (k == 4 || k == 5 || k == 7) {
                ge_p1p1_to_p3<F>(P, t);
                if (k == 4) bases3[i * KB_PTS + 1] = P;
                if (k == 5) bases3[i * KB_PTS + 2] = P;
            } else {
                ge_p2 q; ge_p1p1_to_p2<F>(q, t); fe_copy(P.X, q.X); fe_copy(P.Y, q.Y); fe_copy(P.Z, q.Z);
            }
        }
    }
    if (r0 + nr < COMB_ROWS) bases3[(r0 + nr) * KB_PTS] = P;
    return ok;
}
// Start point of slice `part` (of PARTS) of a row: M = (part * 128 / PARTS + 1) P from the row's helpers; c = P in cached form.
template <class F, int PARTS>
AFC_HD void ge_key_slice_start(ge_p3& M, ge_cached& c, const ge_p3* row3, int part) {
    static_assert(PARTS == 1 || PARTS == 2 || PARTS == 4, "helpers cover 32 P and 64 P only");
    ge_p3_to_cached<F>(c, row3[0]);
    const int m = part * (COMB_COLS / PARTS);          // 0, 32, 64 or 96
    ge_p1p1 t;
    if (m == 0) { M = row3[0]; return; }
    M = (m & 64) ? row3[2] : row3[1];
    ge_addsub<F>(t, M, c, 0); ge_p1p1_to_p3<F>(M, t);  // 64 P + P  or  32 P + P
    if (m == 96) {
        ge_cached c32; ge_p3_to_cached<F>(c32, row3[1]);
        ge_addsub<F>(t, M, c32, 0); ge_p1p1_to_p3<F>(M, t);
    }
}
// Forward half of ge_affine_run: X/Y/Z[j] = M + j P, Pz[j] = Z_0 ... Z_j; the caller inverts Pz[CH-1] (alone or shared).
template <class F, int CH>
AFC_HD void ge_affine_run_fwd(fe* X, fe* Y, fe* Z, fe* Pz, ge_p3& M, const ge_cached& c) {
    ge_p1p1 t;
#pragma unroll 1
    for (int j = 0; j < CH; j++) {
        fe_copy(X[j], M.X); fe_copy(Y[j], M.Y); fe_copy(Z[j], M.Z);
        if (j == 0) fe_copy(Pz[0], M.Z); else F::mul(Pz[j], Pz[j - 1], M.Z);
        if (j + 1 < CH) { ge_addsub<F>(t, M, c, 0); ge_p1p1_to_p3<F>(M, t); }
    }
}
// Backward half: inv = 1 / Pz[CH-1] on entry.
template <class F, int CH>
AFC_HD void ge_affine_run_bwd(ge_precomp* out, const fe* X, const fe* Y, const fe* Z, const fe* Pz, fe inv) {
    fe d2; fe_const(d2, AFC_D2_32);
#pragma unroll 1
    for (int j = CH - 1; j >= 0; j--) {
        fe zi;
        if (j > 0) { F::mul(zi, inv, Pz[j - 1]); F::mul(inv, inv, Z[j]); } else fe_copy(zi, inv);
        fe x, y, xy;
        F::mul(x, X[j], zi); F::mul(y, Y[j], zi);
        ge_precomp& r = out[j];
        fe_add(r.ypx, y, x); fe_sub(r.ymx, y, x); F::mul(xy, x, y); F::mul(r.xy2d, xy, d2);
    }
}

// Single-thread form (one row, its own doubling chain): what the first build of the cache did; kept as the independent check
// of the two-step construction in tests/hostsim.
template <class F = FeInline>
AFC_HD int ge_build_key_row(ge_precomp* row, const uint32_t* pk, int i) {
    ge_p3 P;
    int ok = ge_frombytes<F>(P, pk);
    fe_neg(P.X, P.X); fe_neg(P.T, P.T);
    ge_p1p1 t;
#pragma unroll 1
    for (int k = 0; k < 8 * i; k++) { ge_dbl<F>(t, P.X, P.Y, P.Z); ge_p1p1_to_p3<F>(P, t); }
    ge_key_row_from_base<F>(row, P);
    return ok;
}

// Prefetch policy of the table-driven loop (AFC_KP_PREFETCH: 0 none, 1 both tables into L1, 2 both into L2, 3 key table L1 /
// base table L2).
#ifndef AFC_KP_PREFETCH
#define AFC_KP_PREFETCH 1
#endif
#ifndef AFC_KP_ARRANGED
#define AFC_KP_ARRANGED 1        // table entries loaded already arranged for the digit's sign (ge_load_precomp_arranged): no selects
#endif
#define AFC_PF_L1(p) asm volatile("prefetch.global.L1 [%0];" ::"l"(p))
#define AFC_PF_L2(p) asm volatile("prefetch.global.L2 [%0];" ::"l"(p))
#if AFC_KP_PREFETCH == 2
#define AFC_PREFETCH_A(p) AFC_PF_L2(p)
#define AFC_PREFETCH_B(p) AFC_PF_L2(p)
#elif AFC_KP_PREFETCH == 3
#define AFC_PREFETCH_A(p) AFC_PF_L1(p)
#define AFC_PREFETCH_B(p) AFC_PF_L2(p)
#else
#define AFC_PREFETCH_A(p) AFC_PF_L1(p)
#define AFC_PREFETCH_B(p) AFC_PF_L1(p)
#endif
// R' = [S]B + [k](-A) through the two tables, left in projective form (X : Y : Z): 32 mixed additions from the key's
// radix-256 table of -A and base.rows (12..16) from the base-point table, no doublings.  Base row j is added at key row
// floor(32 j / rows), so the two kinds of gather stay interleaved whatever the window.
template <class F = FeInline>
AFC_HD void ed25519_keyed_point(fe& X, fe& Y, fe& Z, const uint32_t* sig, const uint32_t* k, const ge_precomp* atab, const base_table& base) {
    uint32_t kt[8], st[8];
    sc_recode256(kt, k);
    sc_recode_wide(st, sig + 8, base.offset);
    const int w = base.w, rows = base.rows;
    ge_p3 h; ge_p3_0(h);
    ge_p1p1 t;
    int j = 0, at = 0;                                   // next base row, and the key row it is added at
#pragma unroll 1
    for (int i = 0; i < COMB_ROWS; i++) {
        int dk = sc_digit256(kt, i);
        int ds = 0;
        size_t brow = 0;
        if (i == at) {
            ds = sc_digit_wide(st, j, w, rows);
            brow = (size_t)j << (w - 1);
            j++;
            at = j < rows ? (j * COMB_ROWS) / rows : COMB_ROWS;
        }
#if AFC_DEVICE_CODE && AFC_KP_PREFETCH
        if (i + 1 < COMB_ROWS) {       // the next rows' entries are random 96-byte reads (HBM / L2): start them now
            int nk = sc_digit256(kt, i + 1), mk = nk < 0 ? -nk : nk;
            if (mk) { const char* p = (const char*)&atab[(i + 1) * COMB_COLS + (mk - 1)]; AFC_PREFETCH_A(p); AFC_PREFETCH_A(p + 95); }
            if (at == i + 1) {
                int ns = sc_digit_wide(st, j, w, rows), ms = ns < 0 ? -ns : ns;
                if (ms) { const char* p = (const char*)&base.tab[((size_t)j << (w - 1)) + (ms - 1)]; AFC_PREFETCH_B(p); AFC_PREFETCH_B(p + 95); }
            }
        }
#endif
        if (dk != 0) {
            int neg = dk < 0, m = neg ? -dk : dk;
            ge_precomp e;
#if AFC_KP_ARRANGED
            ge_load_precomp_arranged(e, &atab[i * COMB_COLS + (m - 1)], neg);
            ge_madd_arranged<F>(t, h, e, neg);
#else
            ge_load_precomp(e, &atab[i * COMB_COLS + (m - 1)]);
            ge_maddsub<F>(t, h, e, neg);
#endif
            ge_p1p1_to_p3<F>(h, t);
        }
        if (ds != 0) {
            int neg = ds < 0, m = neg ? -ds : ds;
            ge_precomp e;
#if AFC_KP_ARRANGED
            ge_load_precomp_arranged(e, &base.tab[brow + (m - 1)], neg);
            ge_madd_arranged<F>(t, h, e, neg);
#else
            ge_load_precomp(e, &base.tab[brow + (m - 1)]);
            ge_maddsub<F>(t, h, e, neg);
#endif
            ge_p1p1_to_p3<F>(h, t);
        }
    }
    fe_copy(X, h.X); fe_copy(Y, h.Y); fe_copy(Z, h.Z);
}

// pk_ok: the key decoded.  Single-credential form (used by the key-set kernel and the CPU checks).
template <class F = FeInline>
AFC_HD int ed25519_verify_keyed_core(int pk_ok, const uint32_t* sig, const uint32_t* k, const ge_precomp* atab, const ge_precomp* comb) {
    fe X, Y, Z;
    fe_0(X); fe_1(Y); fe_1(Z);
    // only a canonical S (< L < 2^253) keeps the top digit inside the base table's top row, as in the kernels
    if (ed25519_sig_wellformed(sig)) ed25519_keyed_point<F>(X, Y, Z, sig, k, atab, base_table_make(comb, BASE_W));
    uint32_t enc[1][8];
    if (!pk_ok) { fe_0(X); fe_1(Y); fe_1(Z); }          // garbage table: keep the arithmetic well defined, result is forced to 0
    ge_encode_many<F, 1>(enc, &X, &Y, &Z);
    uint32_t diff = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) diff |= enc[0][i] ^ sig[i];
    return (pk_ok != 0) & ed25519_sig_wellformed(sig) & (diff == 0);
}

// k = SHA-512(R || A || M) mod L
AFC_HD void ed25519_hram(uint32_t* k, const uint32_t* pk, const uint32_t* sig, const uint8_t* msg, uint64_t len) {
    uint32_t pre[16], dig[16];
#pragma unroll
    for (int i = 0; i < 8; i++) { pre[i] = sig[i]; pre[8 + i] = pk[i]; }
    sha512_prefixed<16>(dig, pre, msg, len);
    sc_reduce512(k, dig);
}

// ---------------------------------------------------------------------------------- key expansion / sign
// NewKeyFromSeed: s = clamp(SHA-512(seed)[0:32]) (unreduced), prefix = SHA-512(seed)[32:64], A = [s]B.
template <class F = FeInline>
AFC_HD void ed25519_expand(uint32_t* s, uint32_t* prefix, uint32_t* pk, const uint32_t* seed, const ge_precomp* comb) {
    uint32_t dig[16];
    sha512_prefixed<8>(dig, seed, (const uint8_t*)0, 0);
    dig[0] &= 0xfffffff8u;
    dig[7] &= 0x3fffffffu;
    dig[7] |= 0x40000000u;
#pragma unroll
    for (int i = 0; i < 8; i++) { s[i] = dig[i]; prefix[i] = dig[8 + i]; }
    uint32_t sr[8];
    sc_reduce256(sr, s);
    ge_p3 A;
    ge_scalarmult_base<F>(A, sr, comb);
    ge_encode<F>(pk, A.X, A.Y, A.Z);
}
// The two halves of signing either side of the point encodings, for kernels that share ONE field inversion between the
// encodings of several credentials (and of A = [s]B when signing from seeds):
//   seed -> (s clamped, prefix)                               NewKeyFromSeed without the public key
AFC_HD void ed25519_expand_scalar(uint32_t* s, uint32_t* prefix, const uint32_t* seed) {
    uint32_t dig[16];
    sha512_prefixed<8>(dig, seed, (const uint8_t*)0, 0);
    dig[0] &= 0xfffffff8u;
    dig[7] &= 0x3fffffffu;
    dig[7] |= 0x40000000u;
#pragma unroll
    for (int i = 0; i < 8; i++) { s[i] = dig[i]; prefix[i] = dig[8 + i]; }
}
//   r = SHA-512(prefix || M) mod L
AFC_HD void ed25519_nonce(uint32_t* r, const uint32_t* prefix, const uint8_t* msg, uint64_t len) {
    uint32_t dig[16];
    sha512_prefixed<8>(dig, prefix, msg, len);
    sc_reduce512(r, dig);
}
//   sig = encR || (H(encR || pk || M) s + r) mod L
AFC_HD void ed25519_sign_finish(uint32_t* sig, const uint32_t* encR, const uint32_t* pk, const uint32_t* s, const uint32_t* r,
                                const uint8_t* msg, uint64_t len) {
    uint32_t k[8];
#pragma unroll
    for (int i = 0; i < 8; i++) sig[i] = encR[i];
    ed25519_hram(k, pk, sig, msg, len);
    sc_muladd(sig + 8, k, s, r);
}
// Sign with an expanded key (s, prefix, pk)
template <class F = FeInline>
AFC_HD void ed25519_sign_expanded(uint32_t* sig, const uint32_t* s, const uint32_t* prefix, const uint32_t* pk,
                                   const uint8_t* msg, uint64_t len, const ge_precomp* comb) {
    uint32_t dig[16], r[8], k[8];
    sha512_prefixed<8>(dig, prefix, msg, len);
    sc_reduce512(r, dig);
    ge_p3 R;
    ge_scalarmult_base<F>(R, r, comb);
    ge_encode<F>(sig, R.X, R.Y, R.Z);
    ed25519_hram(k, pk, sig, msg, len);
    sc_muladd(sig + 8, k, s, r);
}

}  // namespace afc
