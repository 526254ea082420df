// Known agents re-registered on the device (afc_did_reregister_batch, include/afcrypto.h; afc_didrereg.cuh).
//
// Reference call sites replaced (relative to /root/reference/control-plane):
//   k_didrr_reg / k_didrr_ids   PerformDifferentialAnalysis, setDifference, extractReasonerIDs   internal/services/did_service.go:757-847
//   k_didrr_ranks               the maps of buildExistingIdentityPackage and PartialRegisterAgent, sorted as json.Marshal writes them
//   k_didrr_sizes               the state RegisterAgent picks (:154-179) and handlePartialRegistration's branches (:991-1045)
//   k_didrr_derive              generateReasonerPath / generateSkillPath, derivePrivateKey         internal/services/did_service.go:870-937, 515-525
//   (then the expansion kernel of k_ed25519.cu, unchanged: ed25519.NewKeyFromSeed)
//   k_didrr_emit / _emit_new    the identities of both maps, at their final offsets                   internal/services/did_service.go:940-986, 1084-1190
//   k_didrr_frame               the text around them, and each request's two key slots
//
// The batch is n requests, the m ids of their 2n request lists and the G registered components of their 2n registered lists.
//   k_didrr_reg     one thread per registered component: GONE and DUP (the request is then refused), its stored entry's length
//   k_didrr_ids     one thread per request id: NEW, SHADOWED, its escaped length
//   k_didrr_ranks   one thread per registered component (rank among the survivors) and per request id (rank among the kept new ids); the
//                   last of each map writes its size.  O(list) per thread, as k_didr_ranks.
//   k_didrr_sizes   one thread per request: state, counts, body length; then the scan gives the body offsets
//   k_didrr_derive  one thread per key slot (2 per request): the path and SHA-256(masterSeed || path), or zeros where no new component
//                   of that kind is added
//   ed_expand_batch over the 2n seeds, into the caller's expanded96
//   k_didrr_emit    one thread per registered component: its GONE flag, and its stored identity when the body lists the survivors
//   k_didrr_emit_new  one thread per request id: its NEW and KEPT flags, and a kept new id's identity (with its private JWK)
//   k_didrr_frame   one thread per request: its key slots' pks and DIDs (zeros for unused slots) and the text around the maps
#include "afc_launch.h"
#include "afc_didrereg.cuh"

namespace afc {

static constexpr int DIDRR_THREADS = 128;

__global__ void __launch_bounds__(DIDRR_THREADS)
k_didrr_reg(const uint8_t* __restrict__ reg_cols, const uint64_t* __restrict__ reg_col_off, const uint64_t* __restrict__ reg_idx,
            const uint8_t* __restrict__ ids, const uint64_t* __restrict__ id_off, const uint64_t* __restrict__ id_idx, uint32_t n, uint32_t G,
            uint8_t* __restrict__ rflags, uint64_t* __restrict__ ebytes, uint32_t* __restrict__ bad) {
    const uint32_t gg = blockIdx.x * blockDim.x + threadIdx.x;
    if (gg >= G) return;
    const uint64_t g = reg_idx[0] + gg;
    const uint32_t L = didr_list_of(reg_idx, n, g);
    const uint32_t f = didrr_reg_flags(reg_cols, reg_col_off, g, reg_idx[L], reg_idx[L + 1], ids, id_off, id_idx[L], id_idx[L + 1]);
    rflags[gg] = (uint8_t)f;
    ebytes[gg] = (f & DIDRR_R_GONE) ? 0 : didrr_stored_entry_bytes((L & 1) ? DIDR_SKILL : DIDR_REASONER, reg_cols, reg_col_off, g);
    if (f & DIDRR_R_DUP) bad[L >> 1] = 1;
}

__global__ void __launch_bounds__(DIDRR_THREADS)
k_didrr_ids(const uint8_t* __restrict__ ids, const uint64_t* __restrict__ id_off, const uint64_t* __restrict__ id_idx, const uint8_t* __restrict__ reg_cols,
            const uint64_t* __restrict__ reg_col_off, const uint64_t* __restrict__ reg_idx, uint32_t n, uint32_t m, uint8_t* __restrict__ iflags,
            uint64_t* __restrict__ esc) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint64_t r = id_idx[0] + j;
    const uint32_t L = didr_list_of(id_idx, n, r);
    const uint32_t f = didrr_id_flags(ids, id_off, r, id_idx[L + 1], reg_cols, reg_col_off, reg_idx[L], reg_idx[L + 1]);
    iflags[j] = (uint8_t)f;
    esc[j] = f == (DIDRR_I_NONEMPTY | DIDRR_I_NEW) ? didr_esc_len(ids + id_off[r], id_off[r + 1] - id_off[r]) : 0;
}

__global__ void __launch_bounds__(DIDRR_THREADS)
k_didrr_ranks(const uint8_t* __restrict__ reg_cols, const uint64_t* __restrict__ reg_col_off, const uint64_t* __restrict__ reg_idx,
              const uint8_t* __restrict__ ids, const uint64_t* __restrict__ id_off, const uint64_t* __restrict__ id_idx,
              const uint32_t* __restrict__ agent_index, uint32_t h, uint32_t n, uint32_t G, uint32_t m, const uint8_t* __restrict__ rflags,
              const uint64_t* __restrict__ ebytes, const uint8_t* __restrict__ iflags, const uint64_t* __restrict__ esc, uint32_t* __restrict__ rank,
              uint64_t* __restrict__ before, uint64_t* __restrict__ map_bytes, uint32_t* __restrict__ map_cnt) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (uint64_t)G + m) return;
    const uint64_t gbase = reg_idx[0];
    if (t < G) {                                                  // a survivor: old map (map_bytes / map_cnt [0, 2n))
        if (rflags[t] & DIDRR_R_GONE) return;
        const uint64_t g = gbase + t;
        const uint32_t L = didr_list_of(reg_idx, n, g);
        const DidrRank q = didrr_reg_rank(reg_cols, reg_col_off, rflags, ebytes, gbase, g, reg_idx[L], reg_idx[L + 1]);
        rank[t] = q.rank;
        before[t] = q.before;
        if (q.rank + 1 == q.kept) { map_bytes[L] = q.before + ebytes[t] + q.rank; map_cnt[L] = q.kept; }
        return;
    }
    const uint64_t j = t - G;                                     // a kept new id: new map ([2n, 4n))
    if (iflags[j] != (DIDRR_I_NONEMPTY | DIDRR_I_NEW)) return;
    const uint64_t base = id_idx[0], r = base + j;
    const uint32_t L = didr_list_of(id_idx, n, r), kind = (L & 1) ? DIDR_SKILL : DIDR_REASONER;
    const uint32_t plen = didr_path_len(kind, h, agent_index[L >> 1], didrr_survivors(rflags, gbase, reg_idx[L], reg_idx[L + 1]));
    const DidrRank q = didrr_id_rank(ids, id_off, iflags, esc, base, r, id_idx[L], id_idx[L + 1], kind, plen);
    rank[t] = q.rank;
    before[t] = q.before;
    if (q.rank + 1 == q.kept) {
        map_bytes[2 * (size_t)n + L] = q.before + didr_entry_bytes(kind, plen, esc[j]) + q.rank;
        map_cnt[2 * (size_t)n + L] = q.kept;
    }
}

__global__ void __launch_bounds__(DIDRR_THREADS)
k_didrr_sizes(const uint8_t* __restrict__ agent_cols, const uint64_t* __restrict__ agent_col_off, const uint64_t* __restrict__ reg_idx,
              const uint8_t* __restrict__ server, uint64_t server_len, uint32_t n, const uint32_t* __restrict__ bad, const uint64_t* __restrict__ map_bytes,
              const uint32_t* __restrict__ map_cnt, uint8_t* __restrict__ state, uint32_t* __restrict__ counts, uint64_t* __restrict__ agent_bytes,
              uint64_t* __restrict__ body_len) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t l = 2 * (size_t)i;
    uint32_t c[4] = {map_cnt[2 * (size_t)n + l], map_cnt[2 * (size_t)n + l + 1], (uint32_t)(reg_idx[l + 1] - reg_idx[l]) - map_cnt[l],
                     (uint32_t)(reg_idx[l + 2] - reg_idx[l + 1]) - map_cnt[l + 1]};
    const uint8_t st = didrr_state(bad[i] != 0, c[0], c[1], c[2], c[3]);
    state[i] = st;
    if (st == DIDRR_INVALID) { c[0] = c[1] = c[2] = c[3] = 0; }
    for (int k = 0; k < 4; k++) counts[4 * (size_t)i + k] = c[k];
    if (st == DIDRR_INVALID) { agent_bytes[i] = 0; body_len[i] = 0; return; }
    const uint64_t agent = didrr_agent_bytes(agent_cols, agent_col_off, i);
    agent_bytes[i] = agent;
    ByteCounter t; t.init();
    didrr_tail(t, server, server_len, st, c);
    body_len[i] = didr_layout(agent, didrr_map_bytes(map_bytes, n, st, i, 0), didrr_map_bytes(map_bytes, n, st, i, 1)).tail + t.n;
}

__global__ void __launch_bounds__(DIDRR_THREADS)
k_didrr_derive(const uint8_t* __restrict__ master, const uint32_t* __restrict__ agent_index, uint32_t h, uint32_t n, const uint8_t* __restrict__ state,
               const uint32_t* __restrict__ counts, const uint32_t* __restrict__ map_cnt, uint8_t* __restrict__ paths, uint8_t* __restrict__ seeds) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * n) return;
    const uint32_t i = t >> 1, kind = (t & 1) ? DIDR_SKILL : DIDR_REASONER;
    uint4* sd = (uint4*)(seeds + 32 * (size_t)t);
    uint8_t* slot = paths + (size_t)DIDR_PATH_SLOT * t;
    if (state[i] != DIDRR_PARTIAL || counts[4 * (size_t)i + (t & 1)] == 0) {
        sd[0] = make_uint4(0, 0, 0, 0); sd[1] = make_uint4(0, 0, 0, 0);
        uint4* ps = (uint4*)slot;
        ps[0] = make_uint4(0, 0, 0, 0); ps[1] = make_uint4(0, 0, 0, 0); ps[2] = make_uint4(0, 0, 0, 0);
        return;
    }
    const uint32_t a = agent_index[i], j0 = map_cnt[t];
    {
        ByteWriter w; w.init(slot);
        didr_put_path(w, kind, h, a, j0);
        for (uint32_t k = didr_path_len(kind, h, a, j0); k < DIDR_PATH_SLOT; k++) w.put(0);
        w.finish();
    }
    uint32_t ms[8], seed[8];
    const word4 m0 = ld_u128(master), m1 = ld_u128(master + 16);
    ms[0] = bswap32(m0.x); ms[1] = bswap32(m0.y); ms[2] = bswap32(m0.z); ms[3] = bswap32(m0.w);
    ms[4] = bswap32(m1.x); ms[5] = bswap32(m1.y); ms[6] = bswap32(m1.z); ms[7] = bswap32(m1.w);
    didr_derive(ms, slot, didr_path_len(kind, h, a, j0), seed);
    sd[0] = make_uint4(seed[0], seed[1], seed[2], seed[3]);
    sd[1] = make_uint4(seed[4], seed[5], seed[6], seed[7]);
}

__global__ void __launch_bounds__(DIDRR_THREADS)
k_didrr_emit(const uint8_t* __restrict__ reg_cols, const uint64_t* __restrict__ reg_col_off, const uint64_t* __restrict__ reg_idx, uint32_t n, uint32_t G,
             const uint8_t* __restrict__ rflags, const uint32_t* __restrict__ rank, const uint64_t* __restrict__ before,
             const uint64_t* __restrict__ map_bytes, const uint64_t* __restrict__ agent_bytes, const uint8_t* __restrict__ state,
             uint8_t* __restrict__ reg_flags, const uint64_t* __restrict__ body_off, uint8_t* __restrict__ bodies) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= G) return;
    const uint64_t g = reg_idx[0] + t;
    const uint32_t L = didr_list_of(reg_idx, n, g), i = L >> 1, kind = (L & 1) ? DIDR_SKILL : DIDR_REASONER;
    const uint8_t st = state[i];
    const bool gone = (rflags[t] & DIDRR_R_GONE) != 0;
    reg_flags[t] = st != DIDRR_INVALID && gone ? DIDRR_GONE : 0;
    if (!((st == DIDRR_UNCHANGED || st == DIDRR_REMOVED) && !gone)) return;
    const uint64_t at = didrr_at(map_bytes, agent_bytes, rank, before, n, st, i, kind, t);
    ByteWriter w; w.init(bodies + body_off[i] + at - (rank[t] ? 1 : 0));
    if (rank[t]) w.put(',');
    didrr_stored_entry(w, kind, reg_cols, reg_col_off, g);
    w.finish();
}

__global__ void __launch_bounds__(DIDRR_THREADS)
k_didrr_emit_new(const uint8_t* __restrict__ ids, const uint64_t* __restrict__ id_off, const uint64_t* __restrict__ id_idx,
                 const uint32_t* __restrict__ agent_index, uint32_t h, uint32_t n, uint32_t G, uint32_t m, const uint8_t* __restrict__ iflags,
                 const uint32_t* __restrict__ rank, const uint64_t* __restrict__ before, const uint64_t* __restrict__ map_bytes,
                 const uint32_t* __restrict__ map_cnt, const uint64_t* __restrict__ agent_bytes, const uint8_t* __restrict__ state,
                 const uint8_t* __restrict__ seeds, const uint8_t* __restrict__ expanded96, uint8_t* __restrict__ id_flags,
                 const uint64_t* __restrict__ body_off, uint8_t* __restrict__ bodies) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint64_t r = id_idx[0] + j, t = (uint64_t)G + j;
    const uint32_t L = didr_list_of(id_idx, n, r), i = L >> 1, kind = (L & 1) ? DIDR_SKILL : DIDR_REASONER;
    const uint8_t st = state[i];
    const uint32_t f = iflags[j];
    const bool nw = st == DIDRR_PARTIAL && (f & DIDRR_I_NEW);
    id_flags[j] = nw ? (uint8_t)(DIDRR_NEW | ((f & DIDRR_I_SHADOWED) ? 0 : 1)) : 0;      // 1: AFC_DID_KEPT
    if (!nw || (f & DIDRR_I_SHADOWED)) return;
    const uint64_t at = didrr_at(map_bytes, agent_bytes, rank, before, n, st, i, kind, t);
    const size_t slot = 2 * (size_t)i + (L & 1);
    uint32_t pk[8], seed[8];
    {
        const word4 p0 = ld_u128(expanded96 + 96 * slot + 64), p1 = ld_u128(expanded96 + 96 * slot + 80);
        pk[0] = p0.x; pk[1] = p0.y; pk[2] = p0.z; pk[3] = p0.w; pk[4] = p1.x; pk[5] = p1.y; pk[6] = p1.z; pk[7] = p1.w;
        const word4 s0 = ld_u128(seeds + 32 * slot), s1 = ld_u128(seeds + 32 * slot + 16);
        seed[0] = s0.x; seed[1] = s0.y; seed[2] = s0.z; seed[3] = s0.w; seed[4] = s1.x; seed[5] = s1.y; seed[6] = s1.z; seed[7] = s1.w;
    }
    ByteWriter w; w.init(bodies + body_off[i] + at - (rank[t] ? 1 : 0));
    if (rank[t]) w.put(',');
    didr_entry(w, kind, h, agent_index[i], map_cnt[L], pk, seed, ids + id_off[r], id_off[r + 1] - id_off[r]);
    w.finish();
}

__global__ void __launch_bounds__(DIDRR_THREADS)
k_didrr_frame(const uint8_t* __restrict__ agent_cols, const uint64_t* __restrict__ agent_col_off, const uint8_t* __restrict__ server, uint64_t server_len,
              uint32_t n, const uint8_t* __restrict__ state, const uint32_t* __restrict__ counts, const uint64_t* __restrict__ map_bytes,
              const uint64_t* __restrict__ agent_bytes, uint8_t* __restrict__ expanded96, uint8_t* __restrict__ pks, uint8_t* __restrict__ dids,
              const uint64_t* __restrict__ body_off, uint8_t* __restrict__ bodies) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t st = state[i];
    uint32_t c[4];
    for (int k = 0; k < 4; k++) c[k] = counts[4 * (size_t)i + k];
    for (uint32_t kind = 0; kind < 2; kind++) {                   // the key slots
        const size_t slot = 2 * (size_t)i + kind;
        uint4* po = (uint4*)(pks + 32 * slot);
        if (st == DIDRR_PARTIAL && c[kind]) {
            const word4 p0 = ld_u128(expanded96 + 96 * slot + 64), p1 = ld_u128(expanded96 + 96 * slot + 80);
            const uint32_t pk[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
            po[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]); po[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
            ByteWriter w; w.init(dids + DIDR_DID_CHARS * slot);
            didr_put_did(w, pk);
            w.finish();
        } else {                                                  // no stale byte stays in an unused slot
            uint4* e = (uint4*)(expanded96 + 96 * slot);
            for (int q = 0; q < 6; q++) e[q] = make_uint4(0, 0, 0, 0);
            po[0] = make_uint4(0, 0, 0, 0); po[1] = make_uint4(0, 0, 0, 0);
            for (int k = 0; k < DIDR_DID_CHARS; k++) dids[DIDR_DID_CHARS * slot + k] = 0;
        }
    }
    if (st == DIDRR_INVALID) return;
    const uint64_t agent = agent_bytes[i], rb = didrr_map_bytes(map_bytes, n, st, i, 0), sb = didrr_map_bytes(map_bytes, n, st, i, 1);
    const DidrLayout Lo = didr_layout(agent, rb, sb);
    uint8_t* body = bodies + body_off[i];
    { ByteWriter w; w.init(body); vci_put_text(w, DIDR_L_HEAD); w.finish(); }
    { ByteWriter w; w.init(body + Lo.agent); didrr_agent(w, agent_cols, agent_col_off, i); vci_put_text(w, DIDR_L_RMAP); w.finish(); }
    { ByteWriter w; w.init(body + Lo.rmap + rb); vci_put_text(w, DIDR_L_SMAP); w.finish(); }
    ByteWriter w; w.init(body + Lo.tail);
    didrr_tail(w, server, server_len, st, c);
    w.finish();
}

namespace launch {

static inline uint32_t didrr_blocks(uint64_t n) { return (uint32_t)((n + DIDRR_THREADS - 1) / DIDRR_THREADS); }

cudaError_t didrr_reregister(const DidrrArgs& A, cudaStream_t s, LaunchLog* lg) {
    const uint32_t n = A.n, m = A.m, G = A.G;
    cudaError_t e = cudaMemsetAsync(A.bad, 0, (size_t)n * 4, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(A.map_bytes, 0, (size_t)4 * n * 8, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(A.map_cnt, 0, (size_t)4 * n * 4, s);
    if (e == cudaSuccess && G) {
        AFC_LAUNCH(lg, "k_didrr_reg", s, k_didrr_reg<<<didrr_blocks(G), DIDRR_THREADS, 0, s>>>(A.reg_cols, A.reg_col_off, A.reg_idx, A.ids, A.id_off,
                                                                                               A.id_idx, n, G, A.rflags, A.ebytes, A.bad));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && m) {
        AFC_LAUNCH(lg, "k_didrr_ids", s, k_didrr_ids<<<didrr_blocks(m), DIDRR_THREADS, 0, s>>>(A.ids, A.id_off, A.id_idx, A.reg_cols, A.reg_col_off,
                                                                                               A.reg_idx, n, m, A.iflags, A.esc));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && (uint64_t)G + m) {
        AFC_LAUNCH(lg, "k_didrr_ranks", s, k_didrr_ranks<<<didrr_blocks((uint64_t)G + m), DIDRR_THREADS, 0, s>>>(
                                               A.reg_cols, A.reg_col_off, A.reg_idx, A.ids, A.id_off, A.id_idx, A.agent_index, A.h, n, G, m, A.rflags,
                                               A.ebytes, A.iflags, A.esc, A.rank, A.before, A.map_bytes, A.map_cnt));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        AFC_LAUNCH(lg, "k_didrr_sizes", s, k_didrr_sizes<<<didrr_blocks(n), DIDRR_THREADS, 0, s>>>(A.agent_cols, A.agent_col_off, A.reg_idx, A.server,
                                                                                                   A.server_len, n, A.bad, A.map_bytes, A.map_cnt,
                                                                                                   A.state, A.counts, A.agent_bytes, A.body_off + 1));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = offsets_from_lengths(A.body_off, n, A.scan, s, lg);
    if (e == cudaSuccess) {
        AFC_LAUNCH(lg, "k_didrr_derive", s, k_didrr_derive<<<didrr_blocks(2 * (uint64_t)n), DIDRR_THREADS, 0, s>>>(A.master, A.agent_index, A.h, n,
                                                                                                                   A.state, A.counts, A.map_cnt,
                                                                                                                   A.paths, A.seeds));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = ed_expand_batch(A.comb, A.ct16, A.seeds, 2 * n, A.expanded96, nullptr, s, lg);
    if (e == cudaSuccess && G) {
        AFC_LAUNCH(lg, "k_didrr_emit", s, k_didrr_emit<<<didrr_blocks(G), DIDRR_THREADS, 0, s>>>(A.reg_cols, A.reg_col_off, A.reg_idx, n, G, A.rflags,
                                                                                                 A.rank, A.before, A.map_bytes, A.agent_bytes, A.state,
                                                                                                 A.reg_flags, A.body_off, A.body));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && m) {
        AFC_LAUNCH(lg, "k_didrr_emit_new", s, k_didrr_emit_new<<<didrr_blocks(m), DIDRR_THREADS, 0, s>>>(
                                                  A.ids, A.id_off, A.id_idx, A.agent_index, A.h, n, G, m, A.iflags, A.rank, A.before, A.map_bytes,
                                                  A.map_cnt, A.agent_bytes, A.state, A.seeds, A.expanded96, A.id_flags, A.body_off, A.body));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        AFC_LAUNCH(lg, "k_didrr_frame", s, k_didrr_frame<<<didrr_blocks(n), DIDRR_THREADS, 0, s>>>(A.agent_cols, A.agent_col_off, A.server, A.server_len,
                                                                                                   n, A.state, A.counts, A.map_bytes, A.agent_bytes,
                                                                                                   A.expanded96, A.pks, A.dids, A.body_off, A.body));
        e = cudaGetLastError();
    }
    return e;
}
uint64_t didrr_req_fixed() { return DIDRR_REQ_FIXED; }
uint64_t didrr_per_reg_fixed() { return DIDRR_PER_REG_FIXED; }

}  // namespace launch
}  // namespace afc
