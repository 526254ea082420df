// Ed25519 kernels for sm_90a: batched verify (the headline metric), sign, key expansion.
//
// Reference call sites replaced (relative to /root/reference/control-plane):
//   ed25519.Verify            internal/services/vc_service.go:504,1624; internal/cli/vc_verification_enhanced.go:453
//   ed25519.Sign              internal/services/vc_service.go:463,715
//   ed25519.NewKeyFromSeed    internal/services/vc_service.go:460,712; internal/services/did_service.go:523
//
// Verify is two kernels so that each gets its own register/occupancy point:
//   k_ed_hram    k_i = SHA-512(R_i || A_i || M_i) mod L            (streams the message; 64-bit ALU work)
//   k_ed_verify  R'_i = [S_i]B + [k_i](-A_i); ok_i = enc(R'_i) == R_i  (pure 32-bit IMAD/IADD3 work,
//                ~2.9k field multiplications per credential — >99% of the time)
// One credential per thread; fixed 4-bit windows keep all 32 lanes on one instruction stream.
// When issuers repeat (the normal case) the second kernel is table-driven instead — per-issuer radix-256 tables built on the
// device (k_kc_*), 48 mixed additions and no doublings per credential, credentials handed to warps by a counter
// (k_ed_verify_cached_dyn / k_ed_verify_keyed_dyn) — and k_ed_verify only sees the keys that are too rare to deserve a table.
#include <cstdlib>

#include "afc_launch.h"
#include "afc_ge.cuh"

namespace afc {

static constexpr int ED_THREADS = 128;

__device__ __forceinline__ void load_words8(uint32_t* w, const uint8_t* p) {
    const uint4* q = (const uint4*)p;
    uint4 a = __ldg(q), b = __ldg(q + 1);
    w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
}
__device__ __forceinline__ void store_words8(uint8_t* p, const uint32_t* w) {
    uint4* q = (uint4*)p;
    q[0] = make_uint4(w[0], w[1], w[2], w[3]);
    q[1] = make_uint4(w[4], w[5], w[6], w[7]);
}

// One atomicAdd per distinct target among the lanes of a warp that call this together: the leader of each group of lanes
// with the same address adds the group's size and every lane gets its own slot (credentials of one issuer often arrive
// together, and the cold list has a single counter).
__device__ __forceinline__ uint32_t kc_grouped_add(uint32_t* addr) {
    const uint32_t mask = __match_any_sync(__activemask(), (unsigned long long)(uintptr_t)addr);
    const int leader = __ffs(mask) - 1, lane = threadIdx.x & 31;
    uint32_t base = 0;
    if (lane == leader) base = atomicAdd(addr, (uint32_t)__popc(mask));
    base = __shfl_sync(mask, base, leader);
    return base + (uint32_t)__popc(mask & ((1u << lane) - 1));
}

// Plain fills as kernels of our own: the cost of cudaMemsetAsync in these streams depends on what else the driver has in
// flight, from microseconds to a large share of a host call.
__global__ void __launch_bounds__(256)
k_fill_u32(uint32_t* __restrict__ p, uint32_t v, uint64_t n) {
    uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i + 3 < n) { *(uint4*)(p + i) = make_uint4(v, v, v, v); return; }
    for (; i < n; i++) p[i] = v;
}
// one thread per BASE_CHUNK consecutive entries of one row of the base-point table (afc_init, once per context)
__global__ void __launch_bounds__(32)
k_ed_build_tables(ge_precomp* base) {
    constexpr int CPR = BASE_COLS / BASE_CHUNK;      // chunks per row
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < BASE_ROWS * CPR) ge_build_base_chunk<FeCall>(base + (size_t)t * BASE_CHUNK, t / CPR, (t % CPR) * BASE_CHUNK);
}
// the same for the verify-only table of radix 2^w (base_table_entries(w) entries; at a context's first table-driven verify)
__global__ void __launch_bounds__(32)
k_ed_build_wide(ge_precomp* tab, int w, uint32_t chunks) {
    const uint32_t cpr = (1u << (w - 1)) / BASE_CHUNK, t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < chunks) ge_build_base_chunk<FeCall>(tab + (size_t)t * BASE_CHUNK, (int)(t / cpr), (int)(t % cpr) * BASE_CHUNK, w);
}

// the 512 entries of the constant-time signing table, copied out of the radix-65536 table (afc_init, once per context)
__global__ void __launch_bounds__(256)
k_ed_build_ct16(const ge_precomp* __restrict__ base, ge_precomp* __restrict__ ct16) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < CT_ROWS * CT_COLS) ct16[t] = base[ge_ct16_source(t / CT_COLS, t % CT_COLS)];
}

// (registers as the compiler leaves them: capping them for more CTAs per SM bought nothing, and a second launch-bounds argument
// of 1 makes ptxas spend registers and lose a CTA)
__global__ void __launch_bounds__(ED_THREADS)
k_ed_hram(const uint8_t* __restrict__ pks, const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ msgs,
          const uint64_t* __restrict__ off, uint32_t n, uint32_t* __restrict__ k_out, const uint32_t* __restrict__ list = nullptr,
          const uint32_t* __restrict__ n_list = nullptr) {
    // with a list: only the credentials the issuer-key cache left to the generic kernel (the four-lane kernel hashes its own)
    if (list) { n = *n_list; if (blockIdx.x * blockDim.x >= n) return; }
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (list) i = list[i];
    uint32_t pk[8], sig[16], k[8];
    load_words8(pk, pks + 32ull * i);
    load_words8(sig, sigs + 64ull * i);          // only R is hashed
    uint64_t o0 = off[i], o1 = off[i + 1];
    ed25519_hram(k, pk, sig, msgs + o0, o1 - o0);
    store_words8((uint8_t*)(k_out + 8ull * i), k);
}

// Variants (AFC_VERIFY_VARIANT: 0 = inline multiplies, 2 CTAs/SM — default; 1 = out-of-line multiplies, 3 CTAs/SM).  Also tried
// and dropped: inline at 168 registers (spills), inline 64-thread CTAs (no gain).  The variants differ only in how field multiplications are emitted and in the
// register budget: F = FeCall keeps the loop I-cache resident; MINB blocks/SM bounds registers (2 -> 255, 3 -> 168, 4 -> 128).
template <class F, int THREADS, int MINB>
__global__ void __launch_bounds__(THREADS, MINB)
k_ed_verify(const ge_precomp* __restrict__ comb, const uint8_t* __restrict__ pks, const uint8_t* __restrict__ sigs,
            const uint32_t* __restrict__ ks, uint32_t n, uint8_t* __restrict__ ok, const uint32_t* __restrict__ list,
            const uint32_t* __restrict__ n_list) {
    // with a list: only the credentials the issuer-key cache left to this kernel (the launch is sized for all n; CTAs past the
    // end of the list leave at once)
    if (list) { n = *n_list; if (blockIdx.x * blockDim.x >= n) return; }
    __shared__ ge_precomp sB[COMB_COLS];         // (j+1)B, j = 0..127: 12 KB, staged with 128-bit loads
    {
        const uint4* src = (const uint4*)comb;
        uint4* dst = (uint4*)sB;
        for (int t = threadIdx.x; t < (int)(sizeof(sB) / 16); t += blockDim.x) dst[t] = __ldg(src + t);
    }
    __syncthreads();
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (list) i = list[i];
    uint32_t pk[8], sig[16], k[8];
    load_words8(pk, pks + 32ull * i);
    load_words8(sig, sigs + 64ull * i);
    load_words8(sig + 8, sigs + 64ull * i + 32);
    load_words8(k, (const uint8_t*)(ks + 8ull * i));
    ok[i] = (uint8_t)ed25519_verify_core<F>(pk, sig, k, sB);
}

// ---- table-driven verification: per-key radix-256 tables of -A (identity cache N1 and the transparent issuer-key cache)
// Credentials per thread in the table-driven kernels (they share ONE field inversion, Montgomery's trick).  The group size is a
// launch parameter: every thread does the same work, so a launch runs in whole waves of `resident threads`; pick_group() chooses
// G in [1, KC_GMAX] so that the last wave is full and the inversion share small (1 M credentials on 132 SMs x 512 threads: G = 15,
// one 99 %-full wave; a 65 536-credential chunk of a host call: G = 1, one wave).
#ifndef AFC_KC_GMAX
#define AFC_KC_GMAX 32         // counter-driven kernels: at 1 M credentials a warp takes ~15 tiles, so no group is cut short
#endif
constexpr int KC_GMAX = AFC_KC_GMAX;
#ifndef AFC_CACHED_MINB
#define AFC_CACHED_MINB 3      // 5 (96 registers, 20 warps/SM) spills
#endif
#ifndef AFC_CACHED_THREADS
#define AFC_CACHED_THREADS 128
#endif
constexpr int KC_THREADS = AFC_CACHED_THREADS;

// Shared body: thread t of T handles positions t, t + T, t + 2T, ... of an ORDER of the credentials (G of them; lanes stay
// adjacent in that order).  item(p) -> credential index of position p: the identity for the key-set kernel without a
// permutation, or the issuer-bucketed permutation — consecutive positions then share their issuer, so the 32 lanes of a warp
// gather from ONE 12 KB table row per step instead of 32 different 384 KB tables (in credential order the gathers miss L2
// far more often).  lookup(i, atab) -> false when credential i's key is unknown or does not decode (ok = 0).
template <class Item, class Lookup>
__device__ __forceinline__ void table_verify_group(Item item, Lookup lookup, const base_table& base, const uint8_t* __restrict__ sigs,
                                                   const uint32_t* __restrict__ ks, uint32_t n, uint32_t T, int G, uint8_t* __restrict__ ok) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    fe X[KC_GMAX], Y[KC_GMAX], Z[KC_GMAX];
    uint32_t good = 0;
    static_assert(KC_GMAX <= 32, "one bit of `good` per credential of a thread");
#pragma unroll 1
    for (int g = 0; g < G; g++) {
        uint64_t p = (uint64_t)t + (uint64_t)g * T;
        fe_0(X[g]); fe_1(Y[g]); fe_1(Z[g]);
        if (p >= n) continue;
        const uint32_t i = item((uint32_t)p);
        const ge_precomp* atab;
        if (!lookup(i, atab)) continue;
        uint32_t sig[16], k[8];
        load_words8(sig, sigs + 64ull * i);
        load_words8(sig + 8, sigs + 64ull * i + 32);
        load_words8(k, (const uint8_t*)(ks + 8ull * i));
        if (!ed25519_sig_wellformed(sig)) continue;
        ed25519_keyed_point<FeInline>(X[g], Y[g], Z[g], sig, k, atab, base);
        good |= 1u << g;
    }
    uint32_t enc[KC_GMAX][8];
    ge_encode_group<FeInline, KC_GMAX>(enc, X, Y, Z, G);
#pragma unroll 1
    for (int g = 0; g < G; g++) {
        uint64_t p = (uint64_t)t + (uint64_t)g * T;
        if (p >= n) break;
        const uint32_t i = item((uint32_t)p);
        uint32_t r[8];
        load_words8(r, sigs + 64ull * i);
        uint32_t diff = 0;
#pragma unroll
        for (int w = 0; w < 8; w++) diff |= enc[g][w] ^ r[w];
        ok[i] = (uint8_t)(((good >> g) & 1u) && diff == 0);
    }
}

// The same work handed out by a counter instead of by position: every warp of a PERSISTENT grid (one CTA per resident slot) takes
// 32 consecutive positions of the order at a time until none are left, up to KC_GMAX per group, then shares the group's inversion.
// A static split runs in whole waves of the resident threads (67 584 on an H100) and G is chosen to make the waves come out
// even; here every SM stays full until the counter runs dry and the groups are as long as the batch allows (~15 credentials per
// inversion for 1 M).
// The inversion is shared by the whole CTA (product tree in shared memory, fe_invert_cta below): at 1 M credentials a thread has
// ~15 of its own to share one with and the CTA-wide form buys little; in a 65 536-credential chunk of a host call a warp gets ONE
// tile, and an inversion per credential would be a third of the work.
template <class F, int NT> __device__ __forceinline__ void fe_invert_cta(fe& inv, const fe& q, fe* tree);
template <int NT, class Item, class Lookup>
__device__ __forceinline__ void table_verify_dynamic(Item item, Lookup lookup, const base_table& base, const uint8_t* __restrict__ sigs,
                                                     const uint32_t* __restrict__ ks, uint32_t n, uint32_t* __restrict__ counter,
                                                     uint8_t* __restrict__ ok, int share_inv) {
    __shared__ fe tree[2 * NT];
    const int lane = threadIdx.x & 31;
    for (;;) {
        fe X[KC_GMAX], Y[KC_GMAX], Z[KC_GMAX], pz[KC_GMAX];        // pz[g] = Z_0 ... Z_g (Montgomery's trick)
        uint32_t idx[KC_GMAX];
        uint32_t good = 0;
        int G = 0;
#pragma unroll 1
        for (; G < KC_GMAX; G++) {
            uint32_t first = 0;
            if (lane == 0) first = atomicAdd(counter, 32u);
            first = __shfl_sync(0xffffffffu, first, 0);
            if (first >= n) break;
            const uint32_t p = first + (uint32_t)lane;
            fe_0(X[G]); fe_1(Y[G]); fe_1(Z[G]);
            idx[G] = 0xffffffffu;
            if (p < n) {
                const uint32_t i = item(p);
                idx[G] = i;
                const ge_precomp* atab;
                if (lookup(i, atab)) {
                    uint32_t sig[16], k[8];
                    load_words8(sig, sigs + 64ull * i);
                    load_words8(sig + 8, sigs + 64ull * i + 32);
                    load_words8(k, (const uint8_t*)(ks + 8ull * i));
                    if (ed25519_sig_wellformed(sig)) {
                        ed25519_keyed_point<FeInline>(X[G], Y[G], Z[G], sig, k, atab, base);
                        good |= 1u << G;
                    }
                }
            }
            if (G == 0) fe_copy(pz[0], Z[0]); else fe_mul(pz[G], pz[G - 1], Z[G]);
        }
        fe inv, q;
        if (G) fe_copy(q, pz[G - 1]); else fe_1(q);                  // a warp that found the counter dry still takes part in the tree
        if (share_inv) fe_invert_cta<FeCall, NT>(inv, q, tree);
        else fe_invert<FeCall>(inv, q);                              // small launch, idle SMs: redundant inversions in parallel are the shorter path
#pragma unroll 1
        for (int g = G - 1; g >= 0; g--) {
            fe zi, x, y;
            if (g > 0) { fe_mul(zi, inv, pz[g - 1]); fe_mul(inv, inv, Z[g]); } else fe_copy(zi, inv);
            fe_mul(x, X[g], zi); fe_mul(y, Y[g], zi);
            const uint32_t i = idx[g];
            if (i == 0xffffffffu) continue;
            uint32_t enc[8], r[8];
            fe_towords(enc, y);
            enc[7] |= (uint32_t)fe_isnegative(x) << 31;
            load_words8(r, sigs + 64ull * i);
            uint32_t diff = 0;
#pragma unroll
            for (int w = 0; w < 8; w++) diff |= enc[w] ^ r[w];
            ok[i] = (uint8_t)(((good >> g) & 1u) && diff == 0);
        }
        if (share_inv) { if (!__syncthreads_or(G == KC_GMAX)) return; }     // every warp saw the counter run dry (and nobody still reads the tree)
        else if (G < KC_GMAX) return;
    }
}

// ---- building per-key tables --------------------------------------------------------------------------------------------
// Two kernels per stage of rows (ge_key_chain_stage / ge_key_slice_start + ge_affine_run_fwd/bwd in afc_ge.cuh):
//   k_kc_chain  one thread per key walks the doubling chain through the stage's rows (latency-bound: a handful of warps)
//   k_kc_rows   one thread per slice of 128 / KR_PARTS table entries; ONE field inversion per CTA
// `list` maps build position -> table id (nullptr: identity), `count` the number of keys (device value if count_dev).
#ifndef AFC_BASES_FE
#define AFC_BASES_FE FeInline      // the chain is latency-bound (one warp per 32 keys): inlined multiplies let the 4 squarings of a doubling overlap
#endif
#ifndef AFC_KEYROW_PARTS
#define AFC_KEYROW_PARTS 4          // threads per table row (128 / PARTS entries each)
#endif
#ifndef AFC_ROWS_THREADS
#define AFC_ROWS_THREADS 256        // CTA size of k_kc_rows = slices that share one field inversion
#endif
#ifndef AFC_ROWS_MINB
#define AFC_ROWS_MINB 2             // CTAs per SM the register budget of k_kc_rows is capped for (2 x 256 threads: <= 128 registers)
#endif
#ifndef AFC_ROWS_FE
#define AFC_ROWS_FE FeInline        // multiplies of the forward / backward runs inlined (FeCall: out of line)
#endif
constexpr int KR_PARTS = AFC_KEYROW_PARTS, KR_SLICE = COMB_COLS / KR_PARTS, KR_NT = AFC_ROWS_THREADS;

struct KeyBuild {
    const uint8_t* pks;          // 32-byte keys, indexed by table id
    const uint32_t* list;        // build position -> table id, or nullptr (identity)
    const uint32_t* count_dev;   // number of keys to build (device), or nullptr
    uint32_t count;              // number of keys to build when count_dev is nullptr; otherwise the launch bound
    ge_p3* bases3;               // count x COMB_ROWS x KB_PTS (indexed by build position)
    ge_precomp* tabs;            // indexed by table id
    uint8_t* valid;              // indexed by table id
};
__device__ __forceinline__ uint32_t kb_count(const KeyBuild& b) { return b.count_dev ? min(*b.count_dev, b.count) : b.count; }

__global__ void __launch_bounds__(32)
k_kc_chain(KeyBuild b, int r0, int nr) {
    const uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= kb_count(b)) return;
    const uint32_t id = b.list ? b.list[pos] : pos;
    uint32_t pk[8];
    load_words8(pk, b.pks + 32ull * id);
    const int ok = ge_key_chain_stage<AFC_BASES_FE>(b.bases3 + (size_t)pos * COMB_ROWS * KB_PTS, pk, r0, nr);
    if (r0 == 0) b.valid[id] = (uint8_t)ok;
}

// The same chain with FOUR lanes per key (Hisil-Wong-Carter-Dawson: the four squarings of a doubling are independent, and so
// are the four products that complete it).  Lane `role` of a quad owns one coordinate (0 X, 1 Y, 2 Z, 3 T): per doubling every
// lane does ONE squaring and ONE multiplication instead of four and three-to-four, and the quad exchanges 48 words by shuffle.
// The chain is pure latency (248 dependent doublings per key, a handful of warps on the whole GPU): 2.6x fewer instructions
// per warp is 2.6x less of it.  T comes for free (lane 3), so every point the rows need is already in P3 form.
__device__ __forceinline__ void fe_shfl(fe& r, const fe& v, int src) {
#pragma unroll
    for (int w = 0; w < 8; w++) r.v[w] = __shfl_sync(0xffffffffu, v.v[w], src);
}
__device__ __forceinline__ void quad_double(fe& C, int role, int q0) {
    fe xs, ys, in, t;
    fe_shfl(xs, C, q0); fe_shfl(ys, C, q0 + 1);
    fe_add(t, xs, ys);
    fe_select(in, C, t, role == 3);                    // X, Y, Z, X + Y
    fe_sq(in, in);
    fe_dbl(t, in);
    fe_select(in, in, t, role == 2);                   // X^2, Y^2, 2 Z^2, (X + Y)^2
    fe xx, yy, bb, aa;
    fe_shfl(xx, in, q0); fe_shfl(yy, in, q0 + 1); fe_shfl(bb, in, q0 + 2); fe_shfl(aa, in, q0 + 3);
    fe rX, rY, rZ, rT, u, v;
    fe_add(rY, yy, xx); fe_sub(rZ, yy, xx); fe_sub(rX, aa, rY); fe_sub(rT, bb, rZ);
    fe_select(u, rX, rY, role == 1); fe_select(u, u, rZ, role == 2);            // rX rY rZ rX
    fe_select(v, rT, rZ, role == 1); fe_select(v, v, rY, role == 3);            // rT rZ rT rY
    fe_mul(C, u, v);                                   // X3 = rX rT, Y3 = rY rZ, Z3 = rZ rT, T3 = rX rY
}
__global__ void __launch_bounds__(32)
k_kc_chain4(KeyBuild b) {
    const int lane = threadIdx.x & 31, role = lane & 3, q0 = lane & ~3;
    const uint32_t pos = (blockIdx.x * blockDim.x + threadIdx.x) >> 2;
    if (blockIdx.x * (blockDim.x >> 2) >= kb_count(b)) return;             // whole warp out of range
    const bool live = pos < kb_count(b);
    const uint32_t id = live ? (b.list ? b.list[pos] : pos) : 0;
    uint32_t pk[8] = {1, 0, 0, 0, 0, 0, 0, 0};                             // idle quads walk the neutral element
    if (live) load_words8(pk, b.pks + 32ull * id);
    ge_p3 P;
    const int ok = ge_frombytes<AFC_BASES_FE>(P, pk);
    fe_neg(P.X, P.X); fe_neg(P.T, P.T);
    if (!ok) ge_p3_0(P);
    if (live && role == 0) b.valid[id] = (uint8_t)ok;
    fe C;
    fe_select(C, P.X, P.Y, role == 1); fe_select(C, C, P.Z, role == 2); fe_select(C, C, P.T, role == 3);
    fe* out = (fe*)(b.bases3 + (size_t)pos * COMB_ROWS * KB_PTS);          // ge_p3 = {X, Y, Z, T}: lane `role` writes field `role`
#pragma unroll 1
    for (int i = 0; i < COMB_ROWS; i++) {
        if (live) out[(i * KB_PTS + 0) * 4 + role] = C;
        const int nd = i + 1 < COMB_ROWS ? 8 : 6;
#pragma unroll 1
        for (int k = 0; k < nd; k++) {
            quad_double(C, role, q0);
            if (live && k == 4) out[(i * KB_PTS + 1) * 4 + role] = C;
            if (live && k == 5) out[(i * KB_PTS + 2) * 4 + role] = C;
        }
    }
}

// 1 / q for every thread of the CTA with ONE field inversion: product tree in shared memory (tree[2 NT]), the root inverted by
// thread 0, inverses pushed back down (inv(left) = inv(parent) x right, inv(right) = inv(parent) x left).  Every q must be
// non-zero (Z coordinates of curve points: the addition law is complete; undecodable keys were replaced by the neutral element).
template <class F, int NT>
__device__ __forceinline__ void fe_invert_cta(fe& inv, const fe& q, fe* tree) {
    const int tid = threadIdx.x;
    tree[tid] = q;
    int off = 0, cnt = NT;
    while (cnt > 1) {
        __syncthreads();
        const int half = cnt >> 1;
        if (tid < half) { fe r; F::mul(r, tree[off + 2 * tid], tree[off + 2 * tid + 1]); tree[off + cnt + tid] = r; }
        off += cnt; cnt = half;
    }
    __syncthreads();
    if (tid == 0) { fe r; fe_invert<F>(r, tree[off]); tree[off] = r; }
    while (cnt < NT) {
        __syncthreads();
        const int cnt2 = cnt << 1, off2 = off - cnt2;
        if (tid < cnt) {
            fe iv = tree[off + tid], L = tree[off2 + 2 * tid], R = tree[off2 + 2 * tid + 1], a, c;
            F::mul(a, iv, R); F::mul(c, iv, L);
            tree[off2 + 2 * tid] = a; tree[off2 + 2 * tid + 1] = c;
        }
        off = off2; cnt = cnt2;
    }
    __syncthreads();
    inv = tree[tid];
}

__global__ void __launch_bounds__(KR_NT, AFC_ROWS_MINB)
k_kc_rows(KeyBuild b, int r0, int nr) {
    __shared__ fe tree[2 * KR_NT];
    const uint32_t per_key = (uint32_t)nr * KR_PARTS;
    const uint64_t total = (uint64_t)kb_count(b) * per_key;
    if ((uint64_t)blockIdx.x * KR_NT >= total) return;                     // whole CTA out of range (uniform)
    const uint64_t g = (uint64_t)blockIdx.x * KR_NT + threadIdx.x;
    const bool live = g < total;
    fe X[KR_SLICE], Y[KR_SLICE], Z[KR_SLICE], Pz[KR_SLICE];
    fe q; fe_1(q);
    ge_precomp* out = nullptr;
    if (live) {
        const uint32_t pos = (uint32_t)(g / per_key), within = (uint32_t)(g % per_key);
        const int row = r0 + (int)(within / KR_PARTS), part = (int)(within % KR_PARTS);
        const uint32_t id = b.list ? b.list[pos] : pos;
        ge_p3 M; ge_cached c;
        ge_key_slice_start<FeCall, KR_PARTS>(M, c, b.bases3 + ((size_t)pos * COMB_ROWS + row) * KB_PTS, part);
        ge_affine_run_fwd<AFC_ROWS_FE, KR_SLICE>(X, Y, Z, Pz, M, c);
        fe_copy(q, Pz[KR_SLICE - 1]);
        out = b.tabs + ((size_t)id * COMB_ROWS + row) * COMB_COLS + part * KR_SLICE;
    }
    fe inv;
    fe_invert_cta<FeCall, KR_NT>(inv, q, tree);
    if (live) ge_affine_run_bwd<AFC_ROWS_FE, KR_SLICE>(out, X, Y, Z, Pz, inv);
}

__global__ void __launch_bounds__(ED_THREADS)
k_ed_hram_keyed(const uint8_t* __restrict__ key_pks, const uint32_t* __restrict__ key_index, uint32_t n_keys,
                const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ msgs, const uint64_t* __restrict__ off, uint32_t n,
                uint32_t* __restrict__ k_out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t key = key_index[i];
    if (key >= n_keys) key = 0;                   // result is forced to 0 in k_ed_verify_keyed
    uint32_t pk[8], sig[16], k[8];
    load_words8(pk, key_pks + 32ull * key);
    load_words8(sig, sigs + 64ull * i);
    uint64_t o0 = off[i], o1 = off[i + 1];
    ed25519_hram(k, pk, sig, msgs + o0, o1 - o0);
    store_words8((uint8_t*)(k_out + 8ull * i), k);
}

// bucketing of an explicit key set's batch by key index (counting sort: histogram, scan, scatter), so that the table-driven kernel
// walks it issuer by issuer like the transparent cache does; indices past the key set share one extra bucket (their ok is 0 anyway)
__global__ void __launch_bounds__(256)
k_ks_hist(const uint32_t* __restrict__ key_index, uint32_t n_keys, uint32_t n, uint32_t* __restrict__ bucket) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t k = key_index[i];
    kc_grouped_add(&bucket[k < n_keys ? k : n_keys]);
}
__global__ void __launch_bounds__(1024)
k_ks_scan(uint32_t* __restrict__ bucket, uint32_t m) {          // exclusive scan of m counters in place, ONE CTA
    __shared__ uint32_t s_part[32], s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < m; base += 1024) {
        const uint32_t id = base + threadIdx.x, v = id < m ? bucket[id] : 0;
        uint32_t x = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, d); if ((threadIdx.x & 31) >= d) x += y; }
        if ((threadIdx.x & 31) == 31) s_part[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            uint32_t p = s_part[threadIdx.x];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, p, d); if (threadIdx.x >= d) p += y; }
            s_part[threadIdx.x] = p;
        }
        __syncthreads();
        const uint32_t warp_off = (threadIdx.x >> 5) ? s_part[(threadIdx.x >> 5) - 1] : 0;
        if (id < m) bucket[id] = s_carry + warp_off + x - v;
        __syncthreads();
        if (threadIdx.x == 0) s_carry += s_part[31];
        __syncthreads();
    }
}
__global__ void __launch_bounds__(256)
k_ks_scatter(const uint32_t* __restrict__ key_index, uint32_t n_keys, uint32_t n, uint32_t* __restrict__ bucket, uint32_t* __restrict__ perm) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t k = key_index[i];
    perm[kc_grouped_add(&bucket[k < n_keys ? k : n_keys])] = i;
}

__global__ void __launch_bounds__(ED_THREADS, AFC_CACHED_MINB)
k_ed_verify_keyed(const base_table base, const ge_precomp* __restrict__ tabs, const uint8_t* __restrict__ valid,
                  const uint32_t* __restrict__ key_index, uint32_t n_keys, const uint8_t* __restrict__ sigs,
                  const uint32_t* __restrict__ ks, uint32_t n, uint32_t T, int G, uint8_t* __restrict__ ok, const uint32_t* __restrict__ perm) {
    table_verify_group([&](uint32_t p) { return perm ? perm[p] : p; }, [&](uint32_t i, const ge_precomp*& atab) {
        uint32_t key = key_index[i];
        if (key >= n_keys || !valid[key]) return false;      // unknown index or undecodable key: ok = 0
        atab = tabs + (size_t)key * COMB_ROWS * COMB_COLS;
        return true;
    }, base, sigs, ks, n, T, G, ok);
}

__global__ void __launch_bounds__(ED_THREADS, AFC_CACHED_MINB)
k_ed_verify_keyed_dyn(const base_table base, const ge_precomp* __restrict__ tabs, const uint8_t* __restrict__ valid,
                      const uint32_t* __restrict__ key_index, uint32_t n_keys, const uint8_t* __restrict__ sigs,
                      const uint32_t* __restrict__ ks, uint32_t n, uint8_t* __restrict__ ok, const uint32_t* __restrict__ perm,
                      uint32_t* __restrict__ counter, int share_inv) {
    table_verify_dynamic<ED_THREADS>([&](uint32_t p) { return perm ? perm[p] : p; }, [&](uint32_t i, const ge_precomp*& atab) {
        uint32_t key = key_index[i];
        if (key >= n_keys || !valid[key]) return false;
        atab = tabs + (size_t)key * COMB_ROWS * COMB_COLS;
        return true;
    }, base, sigs, ks, n, counter, ok, share_inv);
}

// ---- transparent issuer-key cache behind afc_ed25519_verify_batch -----------------------------------------------
// Issuers repeat: the reference verifies against the DIDs its own registry derived (vc_service.go:259), BASELINE's
// configs[1] draws 10^6 credentials from 1024 keys.  The generic entry point therefore, on the device and without a host
// synchronisation:
//   (1) de-duplicates the batch's public keys in a hash table and counts the credentials of each        k_kc_dedup
//   (2) looks the distinct keys up in a persistent per-context cache of radix-256 tables                 k_kc_dedup
//   (3) decides PER KEY: cached -> hot; not cached but used >= KC_AMORTISE times in this batch -> gets a table (evicting the
//       least recently used tables if the cache is full) -> hot; everything else -> cold                k_kc_plan1 / k_kc_plan2
//   (4) builds the missing tables                                                                        k_kc_chain / k_kc_rows
//   (5) buckets the hot credentials by table id, lists the cold ones                                    k_kc_scan / k_kc_scatter
//   (6) runs the table-driven kernel over the hot order and the generic Straus kernel over the cold list — in the same call.
// Results are bit-identical whichever way a credential goes (same group element, same canonical comparison).
using KeyCacheDev = launch::KeyCache;     // POD descriptor of the device buffers (afc_launch.h)
using namespace launch;                   // KS_* state indices
constexpr uint32_t KC_EMPTY = 0xffffffffu, KC_COLD = 0xfffffffeu;
#ifndef AFC_KC_AMORTISE
#define AFC_KC_AMORTISE 48
#endif
constexpr uint32_t KC_AMORTISE = AFC_KC_AMORTISE;      // a table costs about this many generic verifications

__device__ __forceinline__ uint32_t kc_hash(const uint32_t* w) {
    uint32_t h = w[0] * 0x9E3779B1u ^ w[1];
    h = (h ^ (h >> 15)) * 0x85EBCA77u ^ w[2];
    h = (h ^ (h >> 13)) * 0xC2B2AE3Du ^ w[5];
    return h ^ (h >> 16);
}
__device__ __forceinline__ bool kc_equal(const uint32_t* a, const uint8_t* p) {
    uint32_t b[8];
    load_words8(b, p);
    uint32_t d = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) d |= a[i] ^ b[i];
    return d == 0;
}
// start of a call: per-call counters, next epoch, per-id credential counts zeroed
__global__ void __launch_bounds__(256)
k_kc_begin(KeyCacheDev kc) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    for (uint32_t i = t; i <= kc.max_keys; i += gridDim.x * blockDim.x) kc.bucket[i] = 0;
    if (t == 0) {
        kc.state[KS_NHOT] = 0; kc.state[KS_NCOLD] = 0; kc.state[KS_DISTINCT] = 0; kc.state[KS_NBUILD] = 0; kc.state[KS_NCAND] = 0;
        kc.state[KS_REBUILD] = 0; kc.state[KS_EVICTED] = 0; kc.state[KS_QTILE] = 0;
        kc.state[KS_EPOCH] += 1; kc.state[KS_CALLS] += 1;
    }
}
// pass 1: in-batch de-duplication + use counts; representatives also probe the persistent cache (lookup only)
__global__ void __launch_bounds__(256)
k_kc_dedup(KeyCacheDev kc, const uint8_t* __restrict__ pks, uint32_t n) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t w[8];
    load_words8(w, pks + 32ull * i);
    uint32_t h0 = kc_hash(w), h = h0 & kc.bmask;
    uint32_t r = i;
    for (;;) {
        uint32_t cur = kc.bslots[h];
        if (cur == KC_EMPTY) {
            cur = atomicCAS(&kc.bslots[h], KC_EMPTY, i);
            if (cur == KC_EMPTY) break;                       // i is the representative
        }
        if (kc_equal(w, pks + 32ull * cur)) { r = cur; break; }
        h = (h + 1) & kc.bmask;
    }
    kc.rep[i] = r;
    kc_grouped_add(&kc.cnt[r]);
    if (r != i) return;
    kc.dlist[atomicAdd(&kc.state[KS_DISTINCT], 1u)] = i;
    // persistent lookup (the table holds live ids only: evictions rebuild it)
    uint32_t id = KC_EMPTY;
    h = h0 & kc.slot_mask;
    for (uint32_t probes = 0; probes <= kc.slot_mask; probes++) {
        uint32_t cur = kc.slots[h];
        if (cur == KC_EMPTY) break;
        if (kc_equal(w, kc.cpks + 32ull * cur)) { id = cur; break; }
        h = (h + 1) & kc.slot_mask;
    }
    kc.kid[i] = id;
}
// pass 2a, one thread per distinct key: cached -> touch it; frequent enough -> candidate for a table; else cold
__global__ void __launch_bounds__(256)
k_kc_plan1(KeyCacheDev kc) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= kc.state[KS_DISTINCT]) return;
    const uint32_t r = kc.dlist[j], id = kc.kid[r], c = kc.cnt[r];
    if (id != KC_EMPTY) { kc.stamp[id] = kc.state[KS_EPOCH]; kc.bucket[id] = c; }
    else if (c >= KC_AMORTISE) kc.cand[atomicAdd(&kc.state[KS_NCAND], 1u)] = r;
    else kc.kid[r] = KC_COLD;
}
// pass 2b, ONE CTA: make room (least recently used tables first, never one that this call uses), hand out ids
constexpr int KC_PLAN_THREADS = 1024;
__device__ __forceinline__ uint32_t kc_block_count_older(const KeyCacheDev& kc, uint32_t high, uint32_t epoch, uint32_t thr, uint32_t* s_cnt) {
    __syncthreads();
    if (threadIdx.x == 0) *s_cnt = 0;
    __syncthreads();
    uint32_t c = 0;
    for (uint32_t id = threadIdx.x; id < high; id += blockDim.x) { const uint32_t st = kc.stamp[id]; c += (st != 0 && st != epoch && st <= thr); }
    if (c) atomicAdd(s_cnt, c);
    __syncthreads();
    return *s_cnt;
}
__global__ void __launch_bounds__(KC_PLAN_THREADS)
k_kc_plan2(KeyCacheDev kc, const uint8_t* __restrict__ pks) {
    __shared__ uint32_t s_cnt, s_taken, s_pushed;
    const uint32_t ncand = kc.state[KS_NCAND], high = kc.state[KS_HIGH], epoch = kc.state[KS_EPOCH];
    uint32_t nfree = kc.state[KS_NFREE];
    if (ncand == 0) return;
    const uint32_t avail0 = (kc.max_keys - high) + nfree;
    if (ncand > avail0 && epoch > 1) {
        const uint32_t want = ncand - avail0;
        // smallest stamp threshold that frees `want` tables (stamps are call numbers: older = smaller)
        uint32_t lo = 1, hi = epoch - 1;
        const uint32_t evictable = kc_block_count_older(kc, high, epoch, hi, &s_cnt);
        if (evictable) {
            const uint32_t goal = want < evictable ? want : evictable;
            while (lo < hi) {
                const uint32_t mid = lo + (hi - lo) / 2;
                if (kc_block_count_older(kc, high, epoch, mid, &s_cnt) >= goal) hi = mid; else lo = mid + 1;
            }
            const uint32_t below = lo > 1 ? kc_block_count_older(kc, high, epoch, lo - 1, &s_cnt) : 0;   // all of these go
            __syncthreads();
            if (threadIdx.x == 0) { s_taken = 0; s_pushed = 0; }
            __syncthreads();
            const uint32_t at_thr = goal - below;                                                        // and this many with stamp == lo
            for (uint32_t id = threadIdx.x; id < high; id += blockDim.x) {
                const uint32_t st = kc.stamp[id];
                if (st == 0 || st == epoch || st > lo) continue;
                if (st == lo && atomicAdd(&s_taken, 1u) >= at_thr) continue;
                kc.stamp[id] = 0; kc.valid[id] = 0;
                kc.free_list[nfree + atomicAdd(&s_pushed, 1u)] = id;
            }
            __syncthreads();
            nfree += s_pushed;
            if (threadIdx.x == 0) { kc.state[KS_REBUILD] = 1; kc.state[KS_EVICTED] = s_pushed; kc.state[KS_TOTAL_EVICTED] += s_pushed; }
        }
    }
    __syncthreads();
    const uint32_t avail = (kc.max_keys - high) + nfree;
    const uint32_t take = ncand < avail ? ncand : avail;
    for (uint32_t j = threadIdx.x; j < ncand; j += blockDim.x) {
        const uint32_t r = kc.cand[j];
        if (j >= take) { kc.kid[r] = KC_COLD; continue; }
        const uint32_t id = j < nfree ? kc.free_list[nfree - 1 - j] : high + (j - nfree);
        uint32_t w[8];
        load_words8(w, pks + 32ull * r);
        store_words8(kc.cpks + 32ull * id, w);
        kc.kid[r] = id; kc.stamp[id] = epoch; kc.bucket[id] = kc.cnt[r]; kc.build_list[j] = id;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t from_free = take < nfree ? take : nfree;
        kc.state[KS_NBUILD] = take; kc.state[KS_NFREE] = nfree - from_free; kc.state[KS_HIGH] = high + (take - from_free);
        kc.state[KS_TOTAL_BUILT] += take;
    }
}
// the persistent hash table: after an eviction it is cleared and every live id re-inserted, otherwise only the new ids go in
__global__ void __launch_bounds__(256)
k_kc_rehash_clear(KeyCacheDev kc) {
    if (!kc.state[KS_REBUILD]) return;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    for (uint32_t s = t; s <= kc.slot_mask; s += gridDim.x * blockDim.x) kc.slots[s] = KC_EMPTY;
}
__global__ void __launch_bounds__(256)
k_kc_rehash_insert(KeyCacheDev kc) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t id;
    if (kc.state[KS_REBUILD]) { if (t >= kc.state[KS_HIGH] || kc.stamp[t] == 0) return; id = t; }
    else { if (t >= kc.state[KS_NBUILD]) return; id = kc.build_list[t]; }
    uint32_t w[8];
    load_words8(w, kc.cpks + 32ull * id);
    uint32_t h = kc_hash(w) & kc.slot_mask;
    while (atomicCAS(&kc.slots[h], KC_EMPTY, id) != KC_EMPTY) h = (h + 1) & kc.slot_mask;   // distinct keys: no equality test needed
}
// pass 3: exclusive scan of the per-id credential counts -> scatter cursors; ONE CTA
__global__ void __launch_bounds__(1024)
k_kc_scan(KeyCacheDev kc) {
    __shared__ uint32_t s_part[32], s_carry;
    const uint32_t high = kc.state[KS_HIGH];
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < high; base += 1024) {
        const uint32_t id = base + threadIdx.x, v = id < high ? kc.bucket[id] : 0;
        uint32_t x = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, d); if ((threadIdx.x & 31) >= d) x += y; }
        if ((threadIdx.x & 31) == 31) s_part[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            uint32_t p = s_part[threadIdx.x];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, p, d); if (threadIdx.x >= d) p += y; }
            s_part[threadIdx.x] = p;
        }
        __syncthreads();
        const uint32_t warp_off = (threadIdx.x >> 5) ? s_part[(threadIdx.x >> 5) - 1] : 0;
        if (id < high) kc.bucket[id] = s_carry + warp_off + x - v;
        __syncthreads();
        if (threadIdx.x == 0) s_carry += s_part[31];
        __syncthreads();
    }
    if (threadIdx.x == 0) kc.state[KS_NHOT] = s_carry;
}
__global__ void __launch_bounds__(256)
k_kc_scatter(KeyCacheDev kc, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t id = kc.kid[kc.rep[i]];
    if (id >= KC_COLD) kc.cold[kc_grouped_add(&kc.state[KS_NCOLD])] = i;
    else kc.perm[kc_grouped_add(&kc.bucket[id])] = i;
}
// (Fusing k_ed_hram into this kernel was tried and dropped: the SHA-512 state pushes the register allocation of the curve loop
// around and nothing overlaps that did not already.)
__global__ void __launch_bounds__(KC_THREADS, AFC_CACHED_MINB)
k_ed_verify_cached(KeyCacheDev kc, const base_table base, const uint8_t* __restrict__ sigs, const uint32_t* __restrict__ ks,
                   int G, uint8_t* __restrict__ ok) {
    const uint32_t n_hot = kc.state[KS_NHOT];
    if (!n_hot) return;
    const uint32_t T = (n_hot + (uint32_t)G - 1) / (uint32_t)G;
    table_verify_group([&](uint32_t p) { return kc.perm[p]; }, [&](uint32_t i, const ge_precomp*& atab) {
        const uint32_t id = kc.kid[kc.rep[i]];
        if (!kc.valid[id]) return false;                     // key does not decode: ok = 0
        atab = (const ge_precomp*)kc.tabs + (size_t)id * COMB_ROWS * COMB_COLS;
        return true;
    }, base, sigs, ks, n_hot, T, G, ok);
}

// ---- table-driven verification on FOUR lanes per credential (experiment, AFC_VERIFY_QUAD=1|2) --------------------------------
// k_ed_verify_cached / _keyed above keep a whole point, a table entry and the multiplier's accumulators in one thread: ~115
// registers, 4 warps per scheduler and no room on the SM for the hashing to run beside it
// (DESIGN.md §4).  Here a QUAD of lanes shares one credential (ge_quad_plan, afc_ge.cuh): each lane owns one coordinate and does 2
// of the 8 multiplication slots of a mixed addition (7 used), operands arrive by shuffle, and the lane loads only its own 32 bytes
// of the 96-byte table entry.  A lane needs 80 registers, so six warps per scheduler are resident, and (mode 2) the SAME warps do
// the hashing: a warp takes 32 consecutive positions of the issuer-bucketed order, every lane first hashes ONE credential
// (H(R || A || M) mod L, ALU pipe) and leaves its recoded scalars in shared memory, then every quad walks four credentials
// through the tables (multiplier pipe).  The projective result goes to `pts` (3 field elements per position); k_ed_quad_finish
// shares one field inversion per CTA of 2048 credentials, encodes and compares with R.
// Why it loses: the multiplier is busier but has more to do — 8 slots for 7 products and the moves ptxas puts on the same pipe;
// fused, hashing in bucketed order reads its messages at random and the two code bodies miss the instruction cache.  Not the
// default (DESIGN.md §4 has the H100 times).
#ifndef AFC_QUAD_THREADS
#define AFC_QUAD_THREADS 128
#endif
#ifndef AFC_QUAD_MINB
#define AFC_QUAD_MINB 6
#endif
constexpr int QD_THREADS = AFC_QUAD_THREADS;
constexpr int QF_THREADS = 256, QF_G = 8;
static_assert(BASE_W == 16, "the quad kernel walks one base-table row per two key-table rows");

struct QuadSlot {                 // what the owner lane of a credential leaves for the quad that walks it
    uint32_t kt[8], st[8];        // signed radix-256 digits of k, signed radix-65536 digits of S
    const ge_precomp* atab;       // the issuer's table
};
// where the credentials, their order and their keys come from
struct QuadCached {               // transparent cache: hot credentials in bucketed order
    KeyCacheDev kc; const uint8_t* pks;
    __device__ __forceinline__ uint32_t count() const { return kc.state[KS_NHOT]; }
    __device__ __forceinline__ uint32_t item(uint32_t p) const { return kc.perm[p]; }
    __device__ __forceinline__ bool key(uint32_t i, const ge_precomp*& atab, const uint8_t*& pk) const {
        const uint32_t id = kc.kid[kc.rep[i]];
        pk = pks + 32ull * i;
        if (!kc.valid[id]) return false;
        atab = (const ge_precomp*)kc.tabs + (size_t)id * COMB_ROWS * COMB_COLS;
        return true;
    }
};
struct QuadKeyed {                // explicit key set
    const ge_precomp* tabs; const uint8_t* valid; const uint8_t* key_pks; const uint32_t* key_index; uint32_t n_keys;
    const uint32_t* perm; uint32_t n;
    __device__ __forceinline__ uint32_t count() const { return n; }
    __device__ __forceinline__ uint32_t item(uint32_t p) const { return perm ? perm[p] : p; }
    __device__ __forceinline__ bool key(uint32_t i, const ge_precomp*& atab, const uint8_t*& pk) const {
        const uint32_t k = key_index[i];
        if (k >= n_keys) return false;
        pk = key_pks + 32ull * k;
        if (!valid[k]) return false;
        atab = tabs + (size_t)k * COMB_ROWS * COMB_COLS;
        return true;
    }
};

// The neutral table entry {y + x, y - x, 2dxy} = {1, 1, 0}: what a digit 0 adds, and (its first element) what the Z lane multiplies by.
// Loading it like any other entry keeps the loads unconditional and the instruction stream free of selects.
__device__ __align__(32) const uint32_t g_quad_neutral[24] ={1, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};

// ge_quad_plan(role, neg) as per-lane constants (absolute source lanes; the two things that depend on the digit's sign as base ^ flip)
struct QuadLane {
    int s1, sA2, sB2, s3;
    uint32_t keep1, sgn1, s2base, s2flip, voff_base, voff_flip;
    bool zlane;
};
__device__ __forceinline__ QuadLane quad_lane(int role, int q0) {
    const quad_plan a = ge_quad_plan(role, 0), b = ge_quad_plan(role, 1);
    QuadLane L;
    L.s1 = q0 + a.src1; L.sA2 = q0 + a.srcA2; L.sB2 = q0 + a.srcB2; L.s3 = q0 + a.src3;
    L.keep1 = a.keep1; L.sgn1 = a.sgn1;
    L.s2base = a.sgn2; L.s2flip = a.sgn2 ^ b.sgn2;
    L.voff_base = a.v_off; L.voff_flip = a.v_off ^ b.v_off;
    L.zlane = !a.v_load;
    if (L.zlane) { L.voff_base = 0; L.voff_flip = 0; }
    return L;
}
// the lane's 32 bytes of row[|d| - 1], or of the neutral entry (d == 0, Z lane)
__device__ __forceinline__ void quad_load(fe& v, const ge_precomp* row, int d, const QuadLane& L) {
    const uint32_t nm = (uint32_t)(d >> 31);
    const int m = d < 0 ? -d : d;
    const char* e = (m == 0 || L.zlane) ? (const char*)g_quad_neutral : (const char*)(row + (m - 1));
    const uint32_t* p = (const uint32_t*)(e + (L.voff_base ^ (L.voff_flip & nm)));
    asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.v[0]), "=r"(v.v[1]), "=r"(v.v[2]), "=r"(v.v[3]) : "l"(p));
    asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.v[4]), "=r"(v.v[5]), "=r"(v.v[6]), "=r"(v.v[7]) : "l"(p + 4));
}
__device__ __forceinline__ void quad_madd(fe& C, const fe& v, int d, const QuadLane& L) {
    const uint32_t nm = (uint32_t)(d >> 31);
    fe p, u, m, a, b, w, x;
    fe_shfl(p, C, L.s1);
    fe_addsub_m(u, C, p, L.keep1, L.sgn1);
    fe_mul(m, u, v);
    fe_shfl(a, m, L.sA2); fe_shfl(b, m, L.sB2);
    fe_addsub_m(w, a, b, 0xffffffffu, L.s2base ^ (L.s2flip & nm));
    fe_shfl(x, w, L.s3);
    fe_mul(C, w, x);
}

// Warps take tiles of the order from a counter: 32 positions at a time, except the first tile of a warp, which is 8, 16, 24 or 32
// positions depending on where the warp sits — identical warps started together would otherwise hash together and multiply
// together for the whole launch, and the two pipes would never be busy at the same time.
template <class Src, bool FUSED>
__global__ void __launch_bounds__(QD_THREADS, AFC_QUAD_MINB)
k_ed_verify_quad(Src src, const ge_precomp* __restrict__ base, const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ msgs,
                 const uint64_t* __restrict__ off, const uint32_t* __restrict__ ks, fe* __restrict__ pts, uint8_t* __restrict__ ok,
                 uint32_t* __restrict__ tile_counter, uint32_t sms) {
    __shared__ QuadSlot slots[QD_THREADS];
    const uint32_t n = src.count();
    const int lane = threadIdx.x & 31, role = lane & 3, quad = lane >> 2;
    const QuadLane L = quad_lane(role, lane & ~3);
    QuadSlot* wslots = slots + (threadIdx.x & ~31u);
    uint32_t take = 8u * (1u + ((blockIdx.x / sms + (threadIdx.x >> 5)) & 3u));
    for (;;) {
        uint32_t first = 0;
        if (lane == 0) first = atomicAdd(tile_counter, take);
        first = __shfl_sync(0xffffffffu, first, 0);
        if (first >= n) break;
        // ---- every lane prepares ONE credential: checks, k = H(R || A || M) mod L, recoded scalars
        if ((uint32_t)lane < take) {
            const uint32_t p = first + lane;
            uint32_t k[8] = {0, 0, 0, 0, 0, 0, 0, 0}, S[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            const ge_precomp* atab = base;                                  // never read: all digits are 0 when the credential is bad
            if (p < n) {
                const uint32_t i = src.item(p);
                const uint8_t* pkp = nullptr;
                uint32_t sig[16];
                load_words8(sig, sigs + 64ull * i);
                load_words8(sig + 8, sigs + 64ull * i + 32);
                const bool good = src.key(i, atab, pkp) && ed25519_sig_wellformed(sig);
                if (good) {
                    if (FUSED) {
                        uint32_t pk[8];
                        load_words8(pk, pkp);
                        const uint64_t o0 = off[i], o1 = off[i + 1];
                        ed25519_hram(k, pk, sig, msgs + o0, o1 - o0);
                    } else load_words8(k, (const uint8_t*)(ks + 8ull * i));
#pragma unroll
                    for (int w = 0; w < 8; w++) S[w] = sig[8 + w];
                } else atab = base;
                ok[i] = (uint8_t)good;                                      // k_ed_quad_finish ands the comparison in
            }
            QuadSlot& mine = wslots[lane];
            sc_recode256(mine.kt, k);
            sc_recode_base(mine.st, S);
#pragma unroll
            for (int w = 0; w < 8; w++) { mine.kt[w] ^= 0x80808080u; mine.st[w] ^= 0x80008000u; }     // stored as signed digits
            mine.atab = atab;
        }
        __syncwarp();
        // ---- every quad walks up to four credentials: 32 additions from the issuer's table, 16 from the base-point table
        const int nj = (int)(take >> 3);
#pragma unroll 1
        for (int j = 0; j < nj; j++) {
            const uint32_t p = first + (uint32_t)(quad + 8 * j);
            const QuadSlot& c = wslots[quad + 8 * j];
            const int8_t* kb = (const int8_t*)c.kt;
            const int16_t* sb = (const int16_t*)c.st;
            const ge_precomp* atab = c.atab;
            fe C; fe_0(C); C.v[0] = (role == 1 || role == 2) ? 1u : 0u;   // (0 : 1 : 1 : 0)
            int d = kb[0];
            fe v; quad_load(v, atab, d, L);
#pragma unroll 1
            for (int r = 0; r < BASE_ROWS; r++) {
                const int d1 = kb[2 * r + 1];
                fe v1; quad_load(v1, atab + (2 * r + 1) * COMB_COLS, d1, L);
                quad_madd(C, v, d, L);
                const int d2 = sb[r];
                fe v2; quad_load(v2, base + (size_t)r * BASE_COLS, d2, L);
                quad_madd(C, v1, d1, L);
                if (r + 1 < BASE_ROWS) { d = kb[2 * r + 2]; quad_load(v, atab + (2 * r + 2) * COMB_COLS, d, L); }
                quad_madd(C, v2, d2, L);
            }
            if (role < 3 && p < n) pts[3ull * p + role] = C;
        }
        __syncwarp();
        take = 32;
    }
}

// enc(X/Z, Y/Z) == R for every position, ONE field inversion per CTA (QF_THREADS x QF_G positions)
template <class Src>
__global__ void __launch_bounds__(QF_THREADS)
k_ed_quad_finish(Src src, const fe* __restrict__ pts, const uint8_t* __restrict__ sigs, uint8_t* __restrict__ ok) {
    __shared__ fe tree[2 * QF_THREADS];
    const uint32_t n = src.count();
    const uint32_t T = (n + QF_G - 1) / QF_G;
    if (blockIdx.x * QF_THREADS >= T) return;                               // whole CTA past the end
    const uint32_t t = blockIdx.x * QF_THREADS + threadIdx.x;
    fe pz[QF_G], acc; fe_1(acc);
#pragma unroll 1
    for (int g = 0; g < QF_G; g++) {
        const uint64_t p = (uint64_t)t + (uint64_t)g * T;
        if (t < T && p < n) { fe z = pts[3 * p + 2]; FeCall::mul(acc, acc, z); }
        pz[g] = acc;
    }
    fe inv;
    fe_invert_cta<FeCall, QF_THREADS>(inv, acc, tree);
    if (t >= T) return;
#pragma unroll 1
    for (int g = QF_G - 1; g >= 0; g--) {
        const uint64_t p = (uint64_t)t + (uint64_t)g * T;
        if (p >= n) continue;
        fe zi, z = pts[3 * p + 2];
        if (g > 0) FeCall::mul(zi, inv, pz[g - 1]); else fe_copy(zi, inv);
        FeCall::mul(inv, inv, z);
        fe x = pts[3 * p], y = pts[3 * p + 1];
        FeCall::mul(x, x, zi); FeCall::mul(y, y, zi);
        uint32_t enc[8], r[8];
        fe_towords(enc, y);
        enc[7] |= (uint32_t)fe_isnegative(x) << 31;
        const uint32_t i = src.item((uint32_t)p);
        load_words8(r, sigs + 64ull * i);
        uint32_t diff = 0;
#pragma unroll
        for (int w = 0; w < 8; w++) diff |= enc[w] ^ r[w];
        if (diff) ok[i] = 0;
    }
}

__global__ void __launch_bounds__(KC_THREADS, AFC_CACHED_MINB)
k_ed_verify_cached_dyn(KeyCacheDev kc, const base_table base, const uint8_t* __restrict__ sigs, const uint32_t* __restrict__ ks,
                       uint8_t* __restrict__ ok, int share_inv) {
    const uint32_t n_hot = kc.state[KS_NHOT];
    if (!n_hot) return;
    table_verify_dynamic<KC_THREADS>([&](uint32_t p) { return kc.perm[p]; }, [&](uint32_t i, const ge_precomp*& atab) {
        const uint32_t id = kc.kid[kc.rep[i]];
        if (!kc.valid[id]) return false;
        atab = (const ge_precomp*)kc.tabs + (size_t)id * COMB_ROWS * COMB_COLS;
        return true;
    }, base, sigs, ks, n_hot, kc.state + KS_QTILE, ok, share_inv);
}

// mode 0: seeds (32 B each) -> expand then sign;  mode 1: expanded keys (96 B each) selected by key_index.
// Thread t of T signs credentials t, t + T, ... (G <= SIGN_GMAX of them, chosen per launch by pick_sign_group).  All their points — R = [r]B and, from seeds, A = [s]B —
// are computed first and encoded with ONE field inversion (Montgomery's trick): per credential the inversion was 70 % of the
// field work of a signature from an expanded key (16 mixed additions = 112 multiplications against 265) and twice that from a seed.
constexpr int SIGN_GMAX = 8;
#ifndef AFC_SIGN_FE
#define AFC_SIGN_FE FeCall          // field multiplications of the signing kernels out of line (FeInline: inlined, more registers)
#endif
// CT = true: `comb` is the 48 KB constant-time table (ge_scalarmult_base_ct), staged in shared memory; every scalar that is
// multiplied here is secret (the nonce r, and the private scalar s when signing from seeds).
template <bool CT>
__device__ __forceinline__ const ge_precomp* stage_ct_table(const ge_precomp* comb) {
    if (!CT) return comb;
    extern __shared__ uint4 s_ct_raw[];
    const uint4* src = (const uint4*)comb;
    for (int i = threadIdx.x; i < (int)(sizeof(ge_precomp) * CT_ROWS * CT_COLS / 16); i += blockDim.x) s_ct_raw[i] = __ldg(src + i);
    __syncthreads();
    return (const ge_precomp*)s_ct_raw;
}
template <bool CT, class F>
__device__ __forceinline__ void base_mult(ge_p3& h, const uint32_t* a, const ge_precomp* tab) {
    if (CT) ge_scalarmult_base_ct<F>(h, a, tab); else ge_scalarmult_base<F>(h, a, tab);
}
// (4 CTAs per SM, <= 128 registers: left alone, ptxas spends 163 on the in-register SHA-512 and a CTA per SM is lost)
template <bool CT>
__global__ void __launch_bounds__(ED_THREADS, 4)
k_ed_sign(const ge_precomp* __restrict__ comb_in, const uint8_t* __restrict__ keys, const uint32_t* __restrict__ key_index, uint32_t n_keys,
          const uint8_t* __restrict__ msgs, const uint64_t* __restrict__ off, uint32_t n, uint32_t T, int G, uint8_t* __restrict__ sigs) {
    const ge_precomp* comb = stage_ct_table<CT>(comb_in);
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const int mode = n_keys != 0;                                 // n_keys = 0: `keys` are seeds, one per credential
    fe X[2 * SIGN_GMAX], Y[2 * SIGN_GMAX], Z[2 * SIGN_GMAX];     // [0, G): R points; [G, 2G): A points (mode 0)
    uint32_t sc[SIGN_GMAX][8], rr[SIGN_GMAX][8], pks[SIGN_GMAX][8];
#pragma unroll 1
    for (int g = 0; g < G; g++) {
        const uint64_t i = (uint64_t)t + (uint64_t)g * T;
        fe_0(X[g]); fe_1(Y[g]); fe_1(Z[g]); fe_0(X[G + g]); fe_1(Y[G + g]); fe_1(Z[G + g]);
        if (i >= n) continue;
        uint32_t prefix[8];
        if (mode == 0) {
            uint32_t seed[8], sr[8];
            load_words8(seed, keys + 32ull * i);
            ed25519_expand_scalar(sc[g], prefix, seed);
            sc_reduce256(sr, sc[g]);
            ge_p3 A;
            base_mult<CT, AFC_SIGN_FE>(A, sr, comb);
            fe_copy(X[G + g], A.X); fe_copy(Y[G + g], A.Y); fe_copy(Z[G + g], A.Z);
        } else {
            uint32_t kidx = key_index ? key_index[i] : (uint32_t)i;
            if (kidx >= n_keys) kidx = 0;                         // never read key material out of bounds
            const uint8_t* e = keys + 96ull * kidx;
            load_words8(sc[g], e); load_words8(prefix, e + 32); load_words8(pks[g], e + 64);
        }
        const uint64_t o0 = off[i], o1 = off[i + 1];
        ed25519_nonce(rr[g], prefix, msgs + o0, o1 - o0);
        ge_p3 R;
        base_mult<CT, AFC_SIGN_FE>(R, rr[g], comb);
        fe_copy(X[g], R.X); fe_copy(Y[g], R.Y); fe_copy(Z[g], R.Z);
    }
    uint32_t enc[2 * SIGN_GMAX][8];
    ge_encode_group<AFC_SIGN_FE, 2 * SIGN_GMAX>(enc, X, Y, Z, mode == 0 ? 2 * G : G);
#pragma unroll 1
    for (int g = 0; g < G; g++) {
        const uint64_t i = (uint64_t)t + (uint64_t)g * T;
        if (i >= n) break;
        const uint64_t o0 = off[i], o1 = off[i + 1];
        uint32_t sig[16];
        ed25519_sign_finish(sig, enc[g], mode == 0 ? enc[G + g] : pks[g], sc[g], rr[g], msgs + o0, o1 - o0);
        store_words8(sigs + 64ull * i, sig);
        store_words8(sigs + 64ull * i + 32, sig + 8);
    }
}

// seeds -> expanded96 (s || prefix || pk) and/or pks (32 B each); G seeds per thread share one inversion, as in k_ed_sign
template <bool CT>
__global__ void __launch_bounds__(ED_THREADS)
k_ed_expand(const ge_precomp* __restrict__ comb_in, const uint8_t* __restrict__ seeds, uint32_t n, uint32_t T, int G,
            uint8_t* __restrict__ expanded96, uint8_t* __restrict__ pks) {
    const ge_precomp* comb = stage_ct_table<CT>(comb_in);
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    fe X[SIGN_GMAX], Y[SIGN_GMAX], Z[SIGN_GMAX];
    uint32_t sc[SIGN_GMAX][8], pre[SIGN_GMAX][8];
#pragma unroll 1
    for (int g = 0; g < G; g++) {
        const uint64_t i = (uint64_t)t + (uint64_t)g * T;
        fe_0(X[g]); fe_1(Y[g]); fe_1(Z[g]);
        if (i >= n) continue;
        uint32_t seed[8], sr[8];
        load_words8(seed, seeds + 32ull * i);
        ed25519_expand_scalar(sc[g], pre[g], seed);
        sc_reduce256(sr, sc[g]);
        ge_p3 A;
        base_mult<CT, AFC_SIGN_FE>(A, sr, comb);
        fe_copy(X[g], A.X); fe_copy(Y[g], A.Y); fe_copy(Z[g], A.Z);
    }
    uint32_t enc[SIGN_GMAX][8];
    ge_encode_group<AFC_SIGN_FE, SIGN_GMAX>(enc, X, Y, Z, G);
#pragma unroll 1
    for (int g = 0; g < G; g++) {
        const uint64_t i = (uint64_t)t + (uint64_t)g * T;
        if (i >= n) break;
        if (expanded96) {
            uint8_t* e = expanded96 + 96ull * i;
            store_words8(e, sc[g]); store_words8(e + 32, pre[g]); store_words8(e + 64, enc[g]);
        }
        if (pks) store_words8(pks + 32ull * i, enc[g]);
    }
}

// ---- diagnostics ------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t xorshift(uint32_t& x) { x ^= x << 13; x ^= x >> 17; x ^= x << 5; return x; }

// PTX field arithmetic vs the portable versions, on random and boundary operands
__global__ void k_ed_selftest(uint32_t iters, uint32_t* mismatch) {
    uint32_t rs = 0x9E3779B9u * (blockIdx.x * blockDim.x + threadIdx.x + 1);
    uint32_t bad = 0;
    for (uint32_t it = 0; it < iters; it++) {
        fe a, b;
#pragma unroll
        for (int i = 0; i < 8; i++) { a.v[i] = xorshift(rs); b.v[i] = xorshift(rs); }
        uint32_t sel = xorshift(rs);
        if ((sel & 15) == 0) {
#pragma unroll
            for (int i = 0; i < 8; i++) a.v[i] = 0xffffffffu;
        }
        if ((sel & 0xf0) == 0) {
#pragma unroll
            for (int i = 0; i < 8; i++) b.v[i] = 0xffffffffu;
        }
        if ((sel & 0xf00) == 0) { fe_0(a); a.v[0] = sel >> 26; }
        if ((sel & 0xf000) == 0) {
#pragma unroll
            for (int i = 1; i < 8; i++) b.v[i] = 0xffffffffu;
            b.v[0] = 0xffffffffu - (sel >> 26);
        }
        fe r1, r2;
        uint32_t w1[8], w2[8];
        fe_mul(r1, a, b); fe_mul_c(r2, a, b); fe_towords(w1, r1); fe_towords(w2, r2);
#pragma unroll
        for (int i = 0; i < 8; i++) bad |= w1[i] ^ w2[i];
        fe_mul_schoolbook(r1, a, b); fe_towords(w1, r1);
#pragma unroll
        for (int i = 0; i < 8; i++) bad |= w1[i] ^ w2[i];
        fe_sq(r1, a); fe_mul_c(r2, a, a); fe_towords(w1, r1); fe_towords(w2, r2);
#pragma unroll
        for (int i = 0; i < 8; i++) bad |= w1[i] ^ w2[i];
        fe_add(r1, a, b); fe_add_c(r2, a, b);
#pragma unroll
        for (int i = 0; i < 8; i++) bad |= r1.v[i] ^ r2.v[i];
        fe_sub(r1, a, b); fe_sub_c(r2, a, b);
#pragma unroll
        for (int i = 0; i < 8; i++) bad |= r1.v[i] ^ r2.v[i];
    }
    if (bad) atomicAdd(mismatch, 1u);
}


// Issue-model probe: per iteration 8 dependent-by-own-accumulator IMAD.WIDE.U32 plus NADD ALU instructions of a given
// kind on 8 other registers (KIND 0: add.u32, 1: add.cc/addc carry pairs, 2: lop3-type xor, 3: IMAD.WIDE with carry (.X) chain).
template <int NADD, int KIND>
__device__ __forceinline__ void probe_mix(uint32_t iters, fe& a, fe& b) {
    uint64_t acc[8];
    uint32_t x[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { acc[i] = ((uint64_t)a.v[i] << 32) | b.v[i]; x[i] = a.v[i] ^ b.v[7 - i]; }
    uint32_t m = a.v[0] | 1u, y = b.v[1] | 1u;
    for (uint32_t it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < 8; i++) {
            if (KIND == 3) {
                uint32_t lo = (uint32_t)acc[i], hi = (uint32_t)(acc[i] >> 32);
                if (i == 0) asm volatile("mad.lo.cc.u32 %0, %2, %3, %0;\n\tmadc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(lo), "r"(m));
                else if (i < 7) asm volatile("madc.lo.cc.u32 %0, %2, %3, %0;\n\tmadc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(lo), "r"(m));
                else asm volatile("madc.lo.cc.u32 %0, %2, %3, %0;\n\tmadc.hi.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(lo), "r"(m));
                acc[i] = ((uint64_t)hi << 32) | lo;
            } else {
                asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[i]) : "r"((uint32_t)acc[i]), "r"(m));
            }
#pragma unroll
            for (int j = 0; j < NADD / 8; j++) {
                if (KIND == 1) asm volatile("add.cc.u32 %0, %0, %1;\n\taddc.u32 %0, %0, 0;" : "+r"(x[(i + j) & 7]) : "r"(y));   // counts as 2
                else if (KIND == 2) asm volatile("xor.b32 %0, %0, %1;" : "+r"(x[(i + j) & 7]) : "r"(y));
                else asm volatile("add.u32 %0, %0, %1;" : "+r"(x[(i + j) & 7]) : "r"(y));
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 8; i++) { a.v[i] ^= (uint32_t)acc[i] ^ x[i]; b.v[i] ^= (uint32_t)(acc[i] >> 32); }
}

// register-only throughput probes: which = 0 fe_mul, 1 fe_sq, 2 fe_add+fe_sub, 5 fe_mul_c, 6 fe_sq via mul
__global__ void k_microbench_fe(int which, uint32_t iters, uint32_t* sink) {
    uint32_t rs = 0x9E3779B9u * (blockIdx.x * blockDim.x + threadIdx.x + 1);
    fe a, b;
#pragma unroll
    for (int i = 0; i < 8; i++) { a.v[i] = xorshift(rs); b.v[i] = xorshift(rs); }
    if (which == 0) {
        for (uint32_t it = 0; it < iters; it++) { fe_mul(a, a, b); fe_mul(b, b, a); }
    } else if (which == 1) {
        for (uint32_t it = 0; it < iters; it++) { fe_sq(a, a); fe_sq(b, b); }
    } else if (which == 2) {
        for (uint32_t it = 0; it < iters; it++) { fe_add(a, a, b); fe_sub(b, b, a); }
    } else if (which == 5) {
        for (uint32_t it = 0; it < iters; it++) { fe_mul_c(a, a, b); fe_mul_c(b, b, a); }
    } else if (which == 6) {
        for (uint32_t it = 0; it < iters; it++) { fe_mul(a, a, a); fe_mul(b, b, b); }
    } else if (which == 7) {
        for (uint32_t it = 0; it < iters; it++) { fe_mul_schoolbook(a, a, b); fe_mul_schoolbook(b, b, a); }
    } else if (which == 20) { probe_mix<0, 0>(iters, a, b);
    } else if (which == 21) { probe_mix<8, 0>(iters, a, b);
    } else if (which == 22) { probe_mix<16, 0>(iters, a, b);
    } else if (which == 23) { probe_mix<24, 0>(iters, a, b);
    } else if (which == 24) { probe_mix<32, 0>(iters, a, b);
    } else if (which == 25) { probe_mix<16, 1>(iters, a, b);
    } else if (which == 26) { probe_mix<16, 2>(iters, a, b);
    } else if (which == 27) { probe_mix<0, 3>(iters, a, b);
    } else if (which == 28) { probe_mix<16, 3>(iters, a, b);
    } else if (which == 29) { probe_mix<48, 0>(iters, a, b);
    } else if (which == 11) {
        // raw pipe probes: 16 dependent 32-bit IMAD per iteration (8 independent chains)
        uint32_t acc[8];
#pragma unroll
        for (int i = 0; i < 8; i++) acc[i] = a.v[i];
        uint32_t m0 = a.v[0] | 1;
        for (uint32_t it = 0; it < iters; it++) {
#pragma unroll
            for (int r = 0; r < 2; r++)
#pragma unroll
                for (int i = 0; i < 8; i++) acc[i] = acc[i] * m0 + b.v[i];
        }
#pragma unroll
        for (int i = 0; i < 8; i++) a.v[i] ^= acc[i];
    } else if (which == 12) {
        // 16 LOP3/IADD3-class ALU instructions per iteration
        uint32_t acc[8];
#pragma unroll
        for (int i = 0; i < 8; i++) acc[i] = a.v[i];
        for (uint32_t it = 0; it < iters; it++) {
#pragma unroll
            for (int r = 0; r < 2; r++)
#pragma unroll
                for (int i = 0; i < 8; i++) acc[i] = (acc[i] + b.v[i]) ^ (acc[(i + 1) & 7] & b.v[(i + 3) & 7]);
        }
#pragma unroll
        for (int i = 0; i < 8; i++) a.v[i] ^= acc[i];
    } else {
        for (uint32_t it = 0; it < iters; it++) { fe_mul(a, a, a); fe_mul(b, b, b); }
    }
    uint32_t x = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) x ^= a.v[i] ^ b.v[i];
    if (x == 0x12345678u) sink[0] = x;
}

namespace launch {

static inline uint32_t blocks_for(uint64_t n, int t) { return (uint32_t)((n + t - 1) / t); }

// Group size for a launch of n credentials whose threads share one field inversion per G credentials: every thread does the
// same work, so the launch runs in whole waves of `resident threads`; minimise waves(G) x (G x main + inversion), both in field
// multiplications (SHA-512 work counted at its measured equivalent).
static int pick_group_for(uint32_t n, const void* kernel, int slot, uint64_t c_main, uint64_t c_inv, int gmax, const char* env) {
    static int forced[4] = {-1, -1, -1, -1};
    if (forced[slot] < 0) { const char* e = getenv(env); forced[slot] = e ? atoi(e) : 0; }
    if (forced[slot] >= 1 && forced[slot] <= gmax) return forced[slot];
    static thread_local int resident[4] = {0, 0, 0, 0};
    if (!resident[slot]) {
        int dev = 0, sms = 0, per_sm = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        const int threads = slot == 0 ? KC_THREADS : ED_THREADS;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0) != cudaSuccess || per_sm < 1) { cudaGetLastError(); per_sm = 3; }
        resident[slot] = sms * per_sm * threads;
    }
    const uint64_t R = (uint64_t)resident[slot];
    int best = 1; uint64_t best_cost = ~0ull;
    for (int G = 1; G <= gmax; G++) {
        uint64_t T = ((uint64_t)n + G - 1) / G, waves = (T + R - 1) / R;
        uint64_t cost = waves * (G * c_main + c_inv);
        if (cost < best_cost) { best_cost = cost; best = G; }
    }
    return best;
}
static int pick_group(uint32_t n, const void* kernel) {          // table-driven verification: 48 mixed additions per credential
    return pick_group_for(n, kernel, kernel == (const void*)k_ed_verify_cached ? 0 : 1, (uint64_t)(COMB_ROWS + BASE_ROWS) * 7 + 12, 270, KC_GMAX,
                          "AFC_KC_GROUP");
}
// signing / key expansion: 16 mixed additions + two (one) SHA-512 passes worth ~240 (~60) multiplications of time
static int pick_sign_group(uint32_t n) { return pick_group_for(n, (const void*)k_ed_sign<false>, 2, 362, 270, SIGN_GMAX, "AFC_SIGN_GROUP"); }
static int pick_expand_group(uint32_t n) { return pick_group_for(n, (const void*)k_ed_expand<false>, 3, 180, 270, SIGN_GMAX, "AFC_SIGN_GROUP"); }
// constant-time signing: 64 mixed additions + masked table scans instead of 16 additions (occupancy taken from the fast kernel's
// register count: the shared-memory table allows 4 CTAs per SM, which the registers do not exceed)
static int pick_sign_group_ct(uint32_t n) { return pick_group_for(n, (const void*)k_ed_sign<false>, 2, 362 + 48 * 7 + 200, 270, SIGN_GMAX, "AFC_SIGN_GROUP"); }

cudaError_t ed_keycache_clear(const KeyCache& kc, cudaStream_t s, LaunchLog* lg) {
    const uint64_t cnt = (uint64_t)kc.slot_mask + 1;
    AFC_LAUNCH(lg, "k_fill_u32", s, k_fill_u32<<<blocks_for((cnt + 3) / 4, 256), 256, 0, s>>>(kc.slots, 0xffffffffu, cnt));
    AFC_LAUNCH(lg, "k_fill_u32", s, k_fill_u32<<<blocks_for(((uint64_t)kc.max_keys + 3) / 4, 256), 256, 0, s>>>(kc.stamp, 0u, kc.max_keys));
    AFC_LAUNCH(lg, "k_fill_u32", s, k_fill_u32<<<1, 256, 0, s>>>(kc.state, 0u, KS_WORDS));
    return cudaGetLastError();
}

size_t ed_tables_bytes() { return sizeof(ge_precomp) * (size_t)BASE_ROWS * BASE_COLS; }

cudaError_t ed_build_tables(void* comb, cudaStream_t s, LaunchLog* lg) {
    AFC_LAUNCH(lg, "k_ed_build_tables", s, k_ed_build_tables<<<blocks_for((uint64_t)BASE_ROWS * BASE_COLS / BASE_CHUNK, 32), 32, 0, s>>>((ge_precomp*)comb));
    return cudaGetLastError();
}
size_t ed_wide_table_bytes(int w) { return sizeof(ge_precomp) * base_table_entries(w); }
cudaError_t ed_build_wide_table(void* tab, int w, cudaStream_t s, LaunchLog* lg) {
    const uint32_t chunks = (uint32_t)(base_table_entries(w) / BASE_CHUNK);
    AFC_LAUNCH(lg, "k_ed_build_wide", s, k_ed_build_wide<<<blocks_for(chunks, 32), 32, 0, s>>>((ge_precomp*)tab, w, chunks));
    return cudaGetLastError();
}
static base_table verify_table(const VerifyBase& vb) { return base_table_make((const ge_precomp*)vb.tab, vb.w); }
// AFC_VERIFY_QUAD: 0 = one thread per credential (k_ed_verify_cached_dyn / _keyed_dyn; default), 1 = four lanes per credential after
// k_ed_hram, 2 = four lanes per credential with the hashing fused.  The four-lane form spends 8 multiplication slots on the 7
// products of a mixed addition and more of the same pipe on register moves (DESIGN.md §4).  Kept as an experiment; same results.
static int quad_mode() {
    static int m = -1;
    if (m < 0) { const char* e = getenv("AFC_VERIFY_QUAD"); m = e ? atoi(e) : 0; if (m < 0 || m > 2) m = 0; }
    return m;
}
// AFC_VERIFY_DYNAMIC: 1 = the table-driven kernels take their credentials from a counter (persistent grid), 0 = static split
static int dynamic_mode() {
    static int m = -1;
    if (m < 0) { const char* e = getenv("AFC_VERIFY_DYNAMIC"); m = e ? atoi(e) : 1; }
    return m;
}
static uint32_t dynamic_grid(uint32_t n, const void* kernel, int threads) {
    static thread_local int per_sm[2] = {0, 0};
    const int slot = kernel == (const void*)k_ed_verify_cached_dyn ? 0 : 1;
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (!per_sm[slot]) {
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm[slot], kernel, threads, 0) != cudaSuccess || per_sm[slot] < 1) { cudaGetLastError(); per_sm[slot] = AFC_CACHED_MINB; }
    }
    // AFC_DYN_GRID_CAP (tests): at most this many CTAs, so that a small batch already makes every warp go through several groups
    static const uint32_t cap = [] { const char* e = getenv("AFC_DYN_GRID_CAP"); return e ? (uint32_t)strtoul(e, nullptr, 10) : 0u; }();
    uint32_t full = (uint32_t)(sms * per_sm[slot]);
    if (cap && cap < full) full = cap;
    const uint32_t need = blocks_for(n, threads);
    return need < full ? need : full;
}
// one inversion per CTA (less work) or per thread (shorter critical path): small batches leave SMs idle and a warp gets one
// tile, so there the redundant per-thread path is the shorter one
static int dynamic_share_inv(uint32_t n) { return n > 32768u; }
static uint32_t quad_sms() {
    static thread_local int sms = 0;
    if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); if (sms < 1) sms = 132; }
    return (uint32_t)sms;
}
// persistent grid of the four-lane kernel: every resident CTA slot, or fewer when the batch is small
static uint32_t quad_grid(uint32_t n) {
    const uint32_t full = quad_sms() * AFC_QUAD_MINB, need = blocks_for(((uint64_t)n + 7) / 8, QD_THREADS / 32);
    return need < full ? need : full;
}
static void launch_generic_verify(const ge_precomp* cb, const uint8_t* pks, const uint8_t* sigs, const uint32_t* ks, uint32_t n, uint8_t* ok,
                                  const uint32_t* list, const uint32_t* n_list, cudaStream_t s, LaunchLog* lg) {
    static int variant = -1;
    if (variant < 0) { const char* e = getenv("AFC_VERIFY_VARIANT"); variant = e ? atoi(e) : 0; }
    const uint32_t nb = blocks_for(n, ED_THREADS);
    switch (variant) {
    case 1: AFC_LAUNCH(lg, "k_ed_verify", s, k_ed_verify<FeCall, 128, 3><<<nb, 128, 0, s>>>(cb, pks, sigs, ks, n, ok, list, n_list)); break;
    default: AFC_LAUNCH(lg, "k_ed_verify", s, k_ed_verify<FeInline, 128, 2><<<nb, 128, 0, s>>>(cb, pks, sigs, ks, n, ok, list, n_list)); break;
    }
}
// Stages the table build is cut into (rows per stage = 32 / stages): the rows of stage s are filled on kc.side2 while the
// doubling chain of stage s + 1 runs on kc.side.
static int kc_stages() {
    static int st = -1;
    if (st < 0) { const char* e = getenv("AFC_KC_STAGES"); st = e ? atoi(e) : 1; if (st != 1 && st != 2 && st != 4) st = 1; }
    return st;
}
static void launch_key_build(const KeyBuild& b, uint32_t max_build, cudaStream_t chain, cudaStream_t rows, const cudaEvent_t* ev_chain,
                             LaunchLog* lg) {
    static int chain4 = -1;
    if (chain4 < 0) { const char* e = getenv("AFC_KC_CHAIN4"); chain4 = e ? atoi(e) : 1; }
    if (chain4) {
        // four lanes per key, eight keys per warp, one warp per CTA
        AFC_LAUNCH(lg, "k_kc_chain4", chain, k_kc_chain4<<<blocks_for((uint64_t)max_build * 4, 32), 32, 0, chain>>>(b));
        if (chain != rows) { cudaEventRecord(ev_chain[0], chain); cudaStreamWaitEvent(rows, ev_chain[0], 0); }
        AFC_LAUNCH(lg, "k_kc_rows", rows, k_kc_rows<<<blocks_for((uint64_t)max_build * COMB_ROWS * KR_PARTS, KR_NT), KR_NT, 0, rows>>>(b, 0, COMB_ROWS));
        return;
    }
    const int stages = (chain == rows) ? 1 : kc_stages(), nr = COMB_ROWS / stages;
    for (int st = 0; st < stages; st++) {
        // one warp per CTA for the chain: 32 x keys small CTAs spread evenly over the SMs
        AFC_LAUNCH(lg, "k_kc_chain", chain, k_kc_chain<<<blocks_for(max_build, 32), 32, 0, chain>>>(b, st * nr, nr));
        if (chain != rows) { cudaEventRecord(ev_chain[st], chain); cudaStreamWaitEvent(rows, ev_chain[st], 0); }
        AFC_LAUNCH(lg, "k_kc_rows", rows, k_kc_rows<<<blocks_for((uint64_t)max_build * nr * KR_PARTS, KR_NT), KR_NT, 0, rows>>>(b, st * nr, nr));
    }
}
cudaError_t ed_verify_batch(const void* comb, const VerifyBase& vb, const uint8_t* pks, const uint8_t* sigs, const uint8_t* msgs, const uint64_t* off,
                            uint32_t n, uint8_t* ok, uint32_t* scratch_k, const KeyCache* kcp, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    const ge_precomp* cb = (const ge_precomp*)comb;
    const uint32_t nb = blocks_for(n, ED_THREADS);
    if (!kcp) {
        AFC_LAUNCH(lg, "k_ed_hram", s, k_ed_hram<<<nb, ED_THREADS, 0, s>>>(pks, sigs, msgs, off, n, scratch_k));
        launch_generic_verify(cb, pks, sigs, scratch_k, n, ok, nullptr, nullptr, s, lg);
        return cudaGetLastError();
    }
    // Issuer-key cache: de-duplicate, look up, decide per key on the device, build what is missing, bucket by issuer.
    // The cache work runs on kc.side / kc.side2 (HIGH-priority streams: their small CTAs are dispatched as soon as SM slots free
    // up) while H(R||A||M), which does not depend on the cache, runs on the caller's stream: the table build (IMAD.WIDE-bound)
    // and the hashing (ALU-bound) share the SMs.  With equal priorities the block dispatcher drains the hashing grid first
    // and nothing overlaps (measured).
    const KeyCache kc = *kcp;
    const cudaStream_t q = kc.side, q2 = kc.side2;
    cudaError_t e = cudaEventRecord(kc.ev_fork, s);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(q, kc.ev_fork, 0);
    if (e != cudaSuccess) return e;
    {
        const uint64_t cnt = (uint64_t)kc.bmask + 1;
        AFC_LAUNCH(lg, "k_fill_u32", q, k_fill_u32<<<blocks_for((cnt + 3) / 4, 256), 256, 0, q>>>(kc.bslots, 0xffffffffu, cnt));
        AFC_LAUNCH(lg, "k_fill_u32", q, k_fill_u32<<<blocks_for(((uint64_t)n + 3) / 4, 256), 256, 0, q>>>(kc.cnt, 0u, n));
    }
    AFC_LAUNCH(lg, "k_kc_begin", q, k_kc_begin<<<blocks_for((uint64_t)kc.max_keys + 1, 256), 256, 0, q>>>(kc));
    AFC_LAUNCH(lg, "k_kc_dedup", q, k_kc_dedup<<<blocks_for(n, 256), 256, 0, q>>>(kc, pks, n));
    AFC_LAUNCH(lg, "k_kc_plan1", q, k_kc_plan1<<<blocks_for(n, 256), 256, 0, q>>>(kc));
    AFC_LAUNCH(lg, "k_kc_plan2", q, k_kc_plan2<<<1, KC_PLAN_THREADS, 0, q>>>(kc, pks));
    AFC_LAUNCH(lg, "k_kc_rehash_clear", q, k_kc_rehash_clear<<<64, 256, 0, q>>>(kc));
    AFC_LAUNCH(lg, "k_kc_rehash_insert", q, k_kc_rehash_insert<<<blocks_for(kc.max_keys, 256), 256, 0, q>>>(kc));
    // at most min(max_keys, n / KC_AMORTISE) tables can be due in one call
    const uint32_t max_build = kc.max_keys < n / KC_AMORTISE ? kc.max_keys : n / KC_AMORTISE;
    if (max_build) {
        KeyBuild b{kc.cpks, kc.build_list, kc.state + KS_NBUILD, max_build, (ge_p3*)kc.bases, (ge_precomp*)kc.tabs, kc.valid};
        launch_key_build(b, max_build, q, q2, kc.ev_chain, lg);
    }
    AFC_LAUNCH(lg, "k_kc_scan", q, k_kc_scan<<<1, 1024, 0, q>>>(kc));
    AFC_LAUNCH(lg, "k_kc_scatter", q, k_kc_scatter<<<blocks_for(n, 256), 256, 0, q>>>(kc, n));
    if (max_build) {
        if ((e = cudaEventRecord(kc.ev_rows, q2)) != cudaSuccess) return e;
        if ((e = cudaStreamWaitEvent(q, kc.ev_rows, 0)) != cudaSuccess) return e;
    }
    if ((e = cudaEventRecord(kc.ev_join, q)) != cudaSuccess) return e;
    const int quad = kc.pts ? quad_mode() : 0;
    if (quad != 2) AFC_LAUNCH(lg, "k_ed_hram", s, k_ed_hram<<<nb, ED_THREADS, 0, s>>>(pks, sigs, msgs, off, n, scratch_k));
    if ((e = cudaStreamWaitEvent(s, kc.ev_join, 0)) != cudaSuccess) return e;
    if (quad) {
        const QuadCached src{kc, pks};
        if (quad == 2) {
            AFC_LAUNCH(lg, "k_ed_verify_quad", s, (k_ed_verify_quad<QuadCached, true><<<quad_grid(n), QD_THREADS, 0, s>>>(src, cb, sigs, msgs, off, scratch_k, (fe*)kc.pts, ok, kc.state + KS_QTILE, quad_sms())));
            AFC_LAUNCH(lg, "k_ed_hram", s, k_ed_hram<<<nb, ED_THREADS, 0, s>>>(pks, sigs, msgs, off, n, scratch_k, kc.cold, kc.state + KS_NCOLD));
        } else AFC_LAUNCH(lg, "k_ed_verify_quad", s, (k_ed_verify_quad<QuadCached, false><<<quad_grid(n), QD_THREADS, 0, s>>>(src, cb, sigs, msgs, off, scratch_k, (fe*)kc.pts, ok, kc.state + KS_QTILE, quad_sms())));
        AFC_LAUNCH(lg, "k_ed_quad_finish", s, k_ed_quad_finish<QuadCached><<<blocks_for(((uint64_t)n + QF_G - 1) / QF_G, QF_THREADS), QF_THREADS, 0, s>>>(src, (const fe*)kc.pts, sigs, ok));
    } else {
        if (dynamic_mode()) {
            AFC_LAUNCH(lg, "k_ed_verify_cached_dyn", s, k_ed_verify_cached_dyn<<<dynamic_grid(n, (const void*)k_ed_verify_cached_dyn, KC_THREADS), KC_THREADS, 0, s>>>(kc, verify_table(vb), sigs, scratch_k, ok, dynamic_share_inv(n)));
        } else {
            const int G = pick_group(n, (const void*)k_ed_verify_cached);
            const uint32_t Tmax = (uint32_t)(((uint64_t)n + G - 1) / G);
            AFC_LAUNCH(lg, "k_ed_verify_cached", s, k_ed_verify_cached<<<blocks_for(Tmax, KC_THREADS), KC_THREADS, 0, s>>>(kc, verify_table(vb), sigs, scratch_k, G, ok));
        }
    }
    launch_generic_verify(cb, pks, sigs, scratch_k, n, ok, kc.cold, kc.state + KS_NCOLD, s, lg);
    return cudaGetLastError();
}
size_t ed_key_table_bytes(uint32_t n_keys) { return sizeof(ge_precomp) * (size_t)n_keys * COMB_ROWS * COMB_COLS; }
size_t ed_key_bases_bytes(uint32_t n_keys) { return sizeof(ge_p3) * (size_t)n_keys * COMB_ROWS * KB_PTS; }
cudaError_t ed_build_key_tables(const uint8_t* pks, uint32_t n_keys, void* tabs, uint8_t* valid, void* bases_scratch, cudaStream_t s, LaunchLog* lg) {
    if (n_keys == 0) return cudaSuccess;
    KeyBuild b{pks, nullptr, nullptr, n_keys, (ge_p3*)bases_scratch, (ge_precomp*)tabs, valid};
    launch_key_build(b, n_keys, s, s, nullptr, lg);
    return cudaGetLastError();
}
static inline size_t keyed_bucket_words(uint32_t n_keys) { return ((size_t)n_keys + 1 + 3) & ~(size_t)3; }     // keeps what follows 16-byte aligned
// the projective results of the four-lane kernel: only when that experiment is switched on (AFC_VERIFY_QUAD)
size_t ed_verify_pts_bytes(uint64_t n) { return quad_mode() ? (size_t)n * 96 : 0; }
size_t ed_keyed_scratch_bytes(uint32_t n_keys, uint32_t n) { return ed_verify_pts_bytes(n) + (4 + keyed_bucket_words(n_keys) + (size_t)n) * 4; }
// scratch_perm: ed_keyed_scratch_bytes(n_keys, n) bytes, 32-byte aligned ([pts[3 n] field elements,] 4 counter words, bucket[n_keys + 1], perm[n]), or
// nullptr = credential order and the one-thread kernel
cudaError_t ed_verify_keyed_batch(const void* comb, const VerifyBase& vb, const void* tabs, const uint8_t* valid, const uint8_t* key_pks, uint32_t n_keys,
                                  const uint32_t* key_index, const uint8_t* sigs, const uint8_t* msgs, const uint64_t* off, uint32_t n,
                                  uint8_t* ok, uint32_t* scratch_k, uint32_t* scratch_perm, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    const uint32_t* perm = nullptr;
    fe* pts = (fe*)scratch_perm;
    const int quad = scratch_perm ? quad_mode() : 0;
    if (scratch_perm && n >= 4096) {                     // small batches: one wave anyway, the three extra launches would cost more
        uint32_t* bucket = scratch_perm + ed_verify_pts_bytes(n) / 4 + 4;
        uint32_t* perm_w = bucket + keyed_bucket_words(n_keys);
        AFC_LAUNCH(lg, "k_fill_u32", s, k_fill_u32<<<blocks_for(((uint64_t)n_keys + 4) / 4, 256), 256, 0, s>>>(bucket, 0u, (uint64_t)n_keys + 1));
        AFC_LAUNCH(lg, "k_ks_hist", s, k_ks_hist<<<blocks_for(n, 256), 256, 0, s>>>(key_index, n_keys, n, bucket));
        AFC_LAUNCH(lg, "k_ks_scan", s, k_ks_scan<<<1, 1024, 0, s>>>(bucket, n_keys + 1));
        AFC_LAUNCH(lg, "k_ks_scatter", s, k_ks_scatter<<<blocks_for(n, 256), 256, 0, s>>>(key_index, n_keys, n, bucket, perm_w));
        perm = perm_w;
    }
    if (quad) {
        uint32_t* tile_ctr = scratch_perm + ed_verify_pts_bytes(n) / 4;
        AFC_LAUNCH(lg, "k_fill_u32", s, k_fill_u32<<<1, 256, 0, s>>>(tile_ctr, 0u, 4));
        const QuadKeyed src{(const ge_precomp*)tabs, valid, key_pks, key_index, n_keys, perm, n};
        if (quad == 2) AFC_LAUNCH(lg, "k_ed_verify_quad", s, (k_ed_verify_quad<QuadKeyed, true><<<quad_grid(n), QD_THREADS, 0, s>>>(src, (const ge_precomp*)comb, sigs, msgs, off, scratch_k, pts, ok, tile_ctr, quad_sms())));
        else {
            AFC_LAUNCH(lg, "k_ed_hram_keyed", s, k_ed_hram_keyed<<<blocks_for(n, ED_THREADS), ED_THREADS, 0, s>>>(key_pks, key_index, n_keys, sigs, msgs, off, n, scratch_k));
            AFC_LAUNCH(lg, "k_ed_verify_quad", s, (k_ed_verify_quad<QuadKeyed, false><<<quad_grid(n), QD_THREADS, 0, s>>>(src, (const ge_precomp*)comb, sigs, msgs, off, scratch_k, pts, ok, tile_ctr, quad_sms())));
        }
        AFC_LAUNCH(lg, "k_ed_quad_finish", s, k_ed_quad_finish<QuadKeyed><<<blocks_for(((uint64_t)n + QF_G - 1) / QF_G, QF_THREADS), QF_THREADS, 0, s>>>(src, pts, sigs, ok));
        return cudaGetLastError();
    }
    AFC_LAUNCH(lg, "k_ed_hram_keyed", s, k_ed_hram_keyed<<<blocks_for(n, ED_THREADS), ED_THREADS, 0, s>>>(key_pks, key_index, n_keys, sigs, msgs, off, n, scratch_k));
    if (scratch_perm && dynamic_mode()) {
        uint32_t* tile_ctr = scratch_perm + ed_verify_pts_bytes(n) / 4;
        AFC_LAUNCH(lg, "k_fill_u32", s, k_fill_u32<<<1, 256, 0, s>>>(tile_ctr, 0u, 4));
        AFC_LAUNCH(lg, "k_ed_verify_keyed_dyn", s, k_ed_verify_keyed_dyn<<<dynamic_grid(n, (const void*)k_ed_verify_keyed_dyn, ED_THREADS), ED_THREADS, 0, s>>>(verify_table(vb), (const ge_precomp*)tabs, valid, key_index, n_keys, sigs, scratch_k, n, ok, perm, tile_ctr, dynamic_share_inv(n)));
        return cudaGetLastError();
    }
    const int G = pick_group(n, (const void*)k_ed_verify_keyed);
    const uint32_t T = (uint32_t)(((uint64_t)n + G - 1) / G);
    AFC_LAUNCH(lg, "k_ed_verify_keyed", s, k_ed_verify_keyed<<<blocks_for(T, ED_THREADS), ED_THREADS, 0, s>>>(verify_table(vb), (const ge_precomp*)tabs, valid, key_index, n_keys, sigs, scratch_k, n, T, G, ok, perm));
    return cudaGetLastError();
}
// ct16 != nullptr selects the constant-time kernels (48 KB of dynamic shared memory for the table)
constexpr size_t CT_SMEM = sizeof(ge_precomp) * CT_ROWS * CT_COLS;
size_t ed_ct_table_bytes() { return CT_SMEM; }
cudaError_t ed_build_ct_table(const void* comb, void* ct16, cudaStream_t s, LaunchLog* lg) {
    static_assert(BASE_W == 16, "the constant-time table is gathered from the radix-65536 table");
    AFC_LAUNCH(lg, "k_ed_build_ct16", s, k_ed_build_ct16<<<blocks_for(CT_ROWS * CT_COLS, 256), 256, 0, s>>>((const ge_precomp*)comb, (ge_precomp*)ct16));
    return cudaGetLastError();
}
static void launch_sign(const void* comb, const void* ct16, const uint8_t* keys, const uint32_t* key_index, uint32_t n_keys, const uint8_t* msgs,
                        const uint64_t* off, uint32_t n, uint8_t* sigs, cudaStream_t s, LaunchLog* lg) {
    const int G = ct16 ? pick_sign_group_ct(n) : pick_sign_group(n);
    const uint32_t T = (uint32_t)(((uint64_t)n + G - 1) / G);
    if (ct16) AFC_LAUNCH(lg, "k_ed_sign_ct", s, k_ed_sign<true><<<blocks_for(T, ED_THREADS), ED_THREADS, CT_SMEM, s>>>((const ge_precomp*)ct16, keys, key_index, n_keys, msgs, off, n, T, G, sigs));
    else AFC_LAUNCH(lg, "k_ed_sign", s, k_ed_sign<false><<<blocks_for(T, ED_THREADS), ED_THREADS, 0, s>>>((const ge_precomp*)comb, keys, key_index, n_keys, msgs, off, n, T, G, sigs));
}
cudaError_t ed_sign_batch(const void* comb, const void* ct16, const uint8_t* seeds, const uint8_t* msgs, const uint64_t* off, uint32_t n,
                          uint8_t* sigs, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    launch_sign(comb, ct16, seeds, nullptr, 0u, msgs, off, n, sigs, s, lg);
    return cudaGetLastError();
}
cudaError_t ed_sign_expanded_batch(const void* comb, const void* ct16, const uint8_t* expanded96, uint32_t n_keys, const uint32_t* key_index,
                                   const uint8_t* msgs, const uint64_t* off, uint32_t n, uint8_t* sigs, cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    launch_sign(comb, ct16, expanded96, key_index, n_keys, msgs, off, n, sigs, s, lg);
    return cudaGetLastError();
}
cudaError_t ed_expand_batch(const void* comb, const void* ct16, const uint8_t* seeds, uint32_t n, uint8_t* expanded96, uint8_t* pks_only,
                            cudaStream_t s, LaunchLog* lg) {
    if (n == 0) return cudaSuccess;
    const int G = pick_expand_group(n);
    const uint32_t T = (uint32_t)(((uint64_t)n + G - 1) / G);
    if (ct16) AFC_LAUNCH(lg, "k_ed_expand_ct", s, k_ed_expand<true><<<blocks_for(T, ED_THREADS), ED_THREADS, CT_SMEM, s>>>((const ge_precomp*)ct16, seeds, n, T, G, expanded96, pks_only));
    else AFC_LAUNCH(lg, "k_ed_expand", s, k_ed_expand<false><<<blocks_for(T, ED_THREADS), ED_THREADS, 0, s>>>((const ge_precomp*)comb, seeds, n, T, G, expanded96, pks_only));
    return cudaGetLastError();
}
cudaError_t ed_selftest(uint32_t iters, uint32_t* d_mismatch, cudaStream_t s, LaunchLog* lg) {
    AFC_LAUNCH(lg, "k_ed_selftest", s, k_ed_selftest<<<64, 128, 0, s>>>(iters, d_mismatch));
    return cudaGetLastError();
}
cudaError_t microbench_fe(int which, uint32_t iters, uint32_t blocks, uint32_t threads, uint32_t* sink, cudaStream_t s, LaunchLog* lg) {
    AFC_LAUNCH(lg, "k_microbench_fe", s, k_microbench_fe<<<blocks, threads, 0, s>>>(which, iters, sink));
    return cudaGetLastError();
}

}  // namespace launch
}  // namespace afc
