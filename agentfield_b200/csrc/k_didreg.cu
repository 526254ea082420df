// Agent DIDs registered on the device (afc_did_register_batch, include/afcrypto.h; afc_didreg.cuh).
//
// Reference call sites replaced (relative to /root/reference/control-plane):
//   k_didr_ids / k_didr_ranks   the reasoner and skill loops and their maps             internal/services/did_service.go:227-311
//   k_didr_derive               generateDIDWithKeys: derivePrivateKey                  internal/services/did_service.go:476-525
//   (then the expansion kernel of k_ed25519.cu, unchanged: ed25519.NewKeyFromSeed)
//   k_didr_emit                 generateDIDKey, both JWK encoders, the DIDIdentity entries   internal/services/did_service.go:528-575
//   k_didr_sizes / k_didr_frame c.JSON of the DIDRegistrationResponse                   internal/services/did_service.go:330-365
//
// The batch is n requests and the m ids of their 2n lists.  A component is a request's agent or one of its non-empty ids; its slot is
// t < n (agent t) or n + j (id j), and its index c (the order of the outputs) is the agent, then the request's non-empty reasoners, then
// its non-empty skills.  The empty ids' slots map to the C.. n + m - 1 tail, which holds zeros on return.
//   k_didr_ids      one thread per id: its list (binary search of id_idx), non-empty and shadowed flags, escaped length
//   the existing scan over the non-empty flags: nz, from which every index above follows
//   k_didr_ranks    one thread per id: rank among its list's kept keys and the bytes of the entries before it (O(list) per id, so a
//                   request of 1024 reasoners spreads over 1024 threads instead of holding one)
//   k_didr_sizes    one thread per request: component offsets, body length; then the scan gives the body offsets
//   k_didr_derive   one thread per slot: the path into its slot, SHA-256(masterSeed || path) into the seed scratch (a zero seed for the tail)
//   ed_expand_batch over the n + m seeds, into the caller's expanded96
//   k_didr_emit     one thread per slot: pk, DID, flags; a kept component's identity (and map key) at its final place in its body; the tail zeroed
//   k_didr_frame    one thread per request: the text around the identities and maps
#include "afc_launch.h"
#include "afc_didreg.cuh"

namespace afc {

static constexpr int DIDR_THREADS = 128;

__global__ void __launch_bounds__(DIDR_THREADS)
k_didr_ids(const uint8_t* __restrict__ ids, const uint64_t* __restrict__ id_off, const uint64_t* __restrict__ id_idx, uint32_t n, uint32_t m,
           uint32_t* __restrict__ list, uint8_t* __restrict__ flags, uint64_t* __restrict__ esc, uint64_t* __restrict__ nz_len) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint64_t r = id_idx[0] + j;
    const uint32_t L = didr_list_of(id_idx, n, r);
    const uint32_t f = didr_id_flags(ids, id_off, r, id_idx[L + 1]);
    list[j] = L;
    flags[j] = (uint8_t)f;
    esc[j] = f ? didr_esc_len(ids + id_off[r], id_off[r + 1] - id_off[r]) : 0;
    nz_len[j] = f ? 1 : 0;
}

__global__ void __launch_bounds__(DIDR_THREADS)
k_didr_ranks(const uint8_t* __restrict__ ids, const uint64_t* __restrict__ id_off, const uint64_t* __restrict__ id_idx, const uint32_t* __restrict__ agent_index,
             uint32_t h, uint32_t m, const uint32_t* __restrict__ list, const uint8_t* __restrict__ flags, const uint64_t* __restrict__ esc,
             const uint64_t* __restrict__ nz, uint32_t* __restrict__ rank, uint64_t* __restrict__ before, uint64_t* __restrict__ map_bytes,
             uint32_t* __restrict__ map_cnt) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m || flags[j] != DIDR_F_NONEMPTY) return;
    const uint64_t base = id_idx[0], r = base + j;
    const uint32_t L = list[j], kind = (L & 1) ? DIDR_SKILL : DIDR_REASONER, a = agent_index[L >> 1];
    const DidrRank q = didr_rank(ids, id_off, flags, esc, nz, base, r, id_idx[L], id_idx[L + 1], kind, h, a);
    rank[j] = q.rank;
    before[j] = q.before;
    if (q.rank + 1 == q.kept) {                                   // the last key writes its map's size and count
        map_bytes[L] = q.before + didr_entry_bytes(kind, didr_path_len(kind, h, a, (uint32_t)(nz[j] - nz[id_idx[L] - base])), esc[j]) + q.rank;
        map_cnt[L] = q.kept;
    }
}

__global__ void __launch_bounds__(DIDR_THREADS)
k_didr_sizes(const uint8_t* __restrict__ server, uint64_t server_len, const uint8_t* __restrict__ nodes, const uint64_t* __restrict__ node_off,
             const uint32_t* __restrict__ agent_index, const uint64_t* __restrict__ id_idx, uint32_t h, uint32_t n, const uint64_t* __restrict__ nz,
             const uint64_t* __restrict__ map_bytes, const uint32_t* __restrict__ map_cnt, uint64_t* __restrict__ comp_off,
             uint64_t* __restrict__ body_len) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (i == 0) comp_off[0] = 0;
    comp_off[i + 1] = (uint64_t)i + 1 + nz[id_idx[2 * (size_t)i + 2] - id_idx[0]];
    ByteCounter c; c.init();
    didr_tail(c, server, server_len, nodes + node_off[i], node_off[i + 1] - node_off[i], map_cnt[2 * (size_t)i], map_cnt[2 * (size_t)i + 1]);
    const uint64_t agent = didr_identity_bytes(DIDR_AGENT, didr_path_len(DIDR_AGENT, h, agent_index[i], 0), 0);
    body_len[i] = didr_layout(agent, map_bytes[2 * (size_t)i], map_bytes[2 * (size_t)i + 1]).tail + c.n;
}

__global__ void __launch_bounds__(DIDR_THREADS)
k_didr_derive(const uint8_t* __restrict__ master, const uint32_t* __restrict__ agent_index, const uint64_t* __restrict__ id_idx, uint32_t h,
              uint32_t n, uint32_t m, const uint32_t* __restrict__ list, const uint8_t* __restrict__ flags, const uint64_t* __restrict__ nz,
              uint8_t* __restrict__ paths, uint8_t* __restrict__ seeds) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (uint64_t)n + m) return;
    const DidrSlot s = didr_slot(id_idx, list, flags, nz, n, m, t);
    uint4* sd = (uint4*)(seeds + 32 * s.c);
    if (!s.comp) { sd[0] = make_uint4(0, 0, 0, 0); sd[1] = make_uint4(0, 0, 0, 0); return; }
    uint8_t* slot = paths + (size_t)DIDR_PATH_SLOT * s.c;
    const uint32_t a = agent_index[s.i];
    {
        ByteWriter w; w.init(slot);
        didr_put_path(w, s.kind, h, a, s.j);
        const uint32_t len = didr_path_len(s.kind, h, a, s.j);
        for (uint32_t k = len; k < DIDR_PATH_SLOT; k++) w.put(0);
        w.finish();
    }
    uint32_t ms[8], seed[8];
    const word4 m0 = ld_u128(master), m1 = ld_u128(master + 16);
    ms[0] = bswap32(m0.x); ms[1] = bswap32(m0.y); ms[2] = bswap32(m0.z); ms[3] = bswap32(m0.w);
    ms[4] = bswap32(m1.x); ms[5] = bswap32(m1.y); ms[6] = bswap32(m1.z); ms[7] = bswap32(m1.w);
    didr_derive(ms, slot, didr_path_len(s.kind, h, a, s.j), seed);
    sd[0] = make_uint4(seed[0], seed[1], seed[2], seed[3]);
    sd[1] = make_uint4(seed[4], seed[5], seed[6], seed[7]);
}

__global__ void __launch_bounds__(DIDR_THREADS)
k_didr_emit(const uint8_t* __restrict__ ids, const uint64_t* __restrict__ id_off, const uint32_t* __restrict__ agent_index,
            const uint64_t* __restrict__ id_idx, uint32_t h, uint32_t n, uint32_t m, const uint32_t* __restrict__ list,
            const uint8_t* __restrict__ flags, const uint64_t* __restrict__ nz, const uint32_t* __restrict__ rank, const uint64_t* __restrict__ before,
            const uint64_t* __restrict__ map_bytes, const uint8_t* __restrict__ seeds, uint8_t* __restrict__ expanded96, uint8_t* __restrict__ pks,
            uint8_t* __restrict__ dids, uint8_t* __restrict__ paths, uint8_t* __restrict__ comp_flags, const uint64_t* __restrict__ body_off,
            uint8_t* __restrict__ bodies) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (uint64_t)n + m) return;
    const DidrSlot s = didr_slot(id_idx, list, flags, nz, n, m, t);
    if (!s.comp) {                                                // the tail: no secret or stale byte stays there
        uint4* e = (uint4*)(expanded96 + 96 * s.c);
        for (int q = 0; q < 6; q++) e[q] = make_uint4(0, 0, 0, 0);
        uint4* p = (uint4*)(pks + 32 * s.c);
        p[0] = make_uint4(0, 0, 0, 0); p[1] = make_uint4(0, 0, 0, 0);
        uint4* ps = (uint4*)(paths + (size_t)DIDR_PATH_SLOT * s.c);
        ps[0] = make_uint4(0, 0, 0, 0); ps[1] = make_uint4(0, 0, 0, 0); ps[2] = make_uint4(0, 0, 0, 0);
        for (int k = 0; k < DIDR_DID_CHARS; k++) dids[DIDR_DID_CHARS * s.c + k] = 0;
        comp_flags[s.c] = 0;
        return;
    }
    uint32_t pk[8], seed[8];
    {
        const word4 p0 = ld_u128(expanded96 + 96 * s.c + 64), p1 = ld_u128(expanded96 + 96 * s.c + 80);
        pk[0] = p0.x; pk[1] = p0.y; pk[2] = p0.z; pk[3] = p0.w; pk[4] = p1.x; pk[5] = p1.y; pk[6] = p1.z; pk[7] = p1.w;
        uint4* po = (uint4*)(pks + 32 * s.c);
        po[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]); po[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
        const word4 s0 = ld_u128(seeds + 32 * s.c), s1 = ld_u128(seeds + 32 * s.c + 16);
        seed[0] = s0.x; seed[1] = s0.y; seed[2] = s0.z; seed[3] = s0.w; seed[4] = s1.x; seed[5] = s1.y; seed[6] = s1.z; seed[7] = s1.w;
    }
    {
        ByteWriter w; w.init(dids + DIDR_DID_CHARS * s.c);
        didr_put_did(w, pk);
        w.finish();
    }
    const uint64_t jj = t - n;
    const bool kept = s.kind == DIDR_AGENT || flags[jj] == DIDR_F_NONEMPTY;
    comp_flags[s.c] = kept ? 1 : 0;
    if (!kept) return;
    const uint32_t a = agent_index[s.i];
    const uint64_t agent = didr_identity_bytes(DIDR_AGENT, didr_path_len(DIDR_AGENT, h, a, 0), 0);
    const DidrLayout Lo = didr_layout(agent, map_bytes[2 * (size_t)s.i], map_bytes[2 * (size_t)s.i + 1]);
    uint8_t* body = bodies + body_off[s.i];
    if (s.kind == DIDR_AGENT) {
        ByteWriter w; w.init(body + Lo.agent);
        didr_identity(w, DIDR_AGENT, h, a, 0, pk, seed, nullptr, 0);
        w.finish();
        return;
    }
    const uint64_t at = (s.kind == DIDR_REASONER ? Lo.rmap : Lo.smap) + before[jj] + rank[jj];
    ByteWriter w; w.init(body + at - (rank[jj] ? 1 : 0));
    if (rank[jj]) w.put(',');
    didr_entry(w, s.kind, h, a, s.j, pk, seed, ids + id_off[s.r], id_off[s.r + 1] - id_off[s.r]);
    w.finish();
}

__global__ void __launch_bounds__(DIDR_THREADS)
k_didr_frame(const uint8_t* __restrict__ server, uint64_t server_len, const uint8_t* __restrict__ nodes, const uint64_t* __restrict__ node_off,
             const uint32_t* __restrict__ agent_index, uint32_t h, uint32_t n, const uint64_t* __restrict__ map_bytes,
             const uint32_t* __restrict__ map_cnt, const uint64_t* __restrict__ body_off, uint8_t* __restrict__ bodies) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t agent = didr_identity_bytes(DIDR_AGENT, didr_path_len(DIDR_AGENT, h, agent_index[i], 0), 0);
    const uint64_t rb = map_bytes[2 * (size_t)i], sb = map_bytes[2 * (size_t)i + 1];
    const DidrLayout Lo = didr_layout(agent, rb, sb);
    uint8_t* body = bodies + body_off[i];
    { ByteWriter w; w.init(body); vci_put_text(w, DIDR_L_HEAD); w.finish(); }
    { ByteWriter w; w.init(body + Lo.agent + agent); vci_put_text(w, DIDR_L_RMAP); w.finish(); }
    { ByteWriter w; w.init(body + Lo.rmap + rb); vci_put_text(w, DIDR_L_SMAP); w.finish(); }
    ByteWriter w; w.init(body + Lo.tail);
    didr_tail(w, server, server_len, nodes + node_off[i], node_off[i + 1] - node_off[i], map_cnt[2 * (size_t)i], map_cnt[2 * (size_t)i + 1]);
    w.finish();
}

namespace launch {

static inline uint32_t didr_blocks(uint64_t n) { return (uint32_t)((n + DIDR_THREADS - 1) / DIDR_THREADS); }

cudaError_t didr_register(const DidrArgs& A, cudaStream_t s, LaunchLog* lg) {
    const uint32_t n = A.n, m = A.m;
    const uint64_t slots = (uint64_t)n + m;
    cudaError_t e = cudaSuccess;
    if (m) {
        AFC_LAUNCH(lg, "k_didr_ids", s, k_didr_ids<<<didr_blocks(m), DIDR_THREADS, 0, s>>>(A.ids, A.id_off, A.id_idx, n, m, A.list, A.flags, A.esc,
                                                                                          A.nz + 1));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = offsets_from_lengths(A.nz, m, A.scan, s, lg);
    if (e == cudaSuccess) e = cudaMemsetAsync(A.map_bytes, 0, (size_t)2 * n * 8, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(A.map_cnt, 0, (size_t)2 * n * 4, s);
    if (e == cudaSuccess && m) {
        AFC_LAUNCH(lg, "k_didr_ranks", s, k_didr_ranks<<<didr_blocks(m), DIDR_THREADS, 0, s>>>(A.ids, A.id_off, A.id_idx, A.agent_index, A.h, m, A.list,
                                                                                              A.flags, A.esc, A.nz, A.rank, A.before, A.map_bytes,
                                                                                              A.map_cnt));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        AFC_LAUNCH(lg, "k_didr_sizes", s, k_didr_sizes<<<didr_blocks(n), DIDR_THREADS, 0, s>>>(A.server, A.server_len, A.nodes, A.node_off, A.agent_index,
                                                                                              A.id_idx, A.h, n, A.nz, A.map_bytes, A.map_cnt,
                                                                                              A.comp_off, A.body_off + 1));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = offsets_from_lengths(A.body_off, n, A.scan, s, lg);
    if (e == cudaSuccess) {
        AFC_LAUNCH(lg, "k_didr_derive", s, k_didr_derive<<<didr_blocks(slots), DIDR_THREADS, 0, s>>>(A.master, A.agent_index, A.id_idx, A.h, n, m, A.list,
                                                                                                    A.flags, A.nz, A.paths, A.seeds));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = ed_expand_batch(A.comb, A.ct16, A.seeds, (uint32_t)slots, A.expanded96, nullptr, s, lg);
    if (e == cudaSuccess) {
        AFC_LAUNCH(lg, "k_didr_emit", s, k_didr_emit<<<didr_blocks(slots), DIDR_THREADS, 0, s>>>(A.ids, A.id_off, A.agent_index, A.id_idx, A.h, n, m, A.list,
                                                                                                A.flags, A.nz, A.rank, A.before, A.map_bytes, A.seeds,
                                                                                                A.expanded96, A.pks, A.dids, A.paths, A.comp_flags,
                                                                                                A.body_off, A.body));
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        AFC_LAUNCH(lg, "k_didr_frame", s, k_didr_frame<<<didr_blocks(n), DIDR_THREADS, 0, s>>>(A.server, A.server_len, A.nodes, A.node_off, A.agent_index,
                                                                                              A.h, n, A.map_bytes, A.map_cnt, A.body_off, A.body));
        e = cudaGetLastError();
    }
    return e;
}
uint64_t didr_req_fixed() { return DIDR_REQ_FIXED; }
uint64_t didr_per_id_fixed() { return DIDR_PER_ID_FIXED; }

}  // namespace launch
}  // namespace afc
