// TEST-ONLY CPU build of the re-registration routines (agentfield_b200/csrc/afc_didrereg.cuh): what the threads of k_didrr_reg,
// k_didrr_ids, k_didrr_ranks, k_didrr_sizes, k_didrr_derive, k_didrr_emit, k_didrr_emit_new and k_didrr_frame do, run one after another
// over a whole batch, with the kernels' own list mapping (didr_list_of).  The Ed25519 expansion is not here: the caller passes the public
// keys of the key slots.  Compiled on its own by tests/test_didrereg_hostsim.py.
#define AFC_HOSTSIM 1
#include <vector>

#include "../../agentfield_b200/csrc/afc_didrereg.cuh"

using namespace afc;

extern "C" {

// The batch, as the kernels compute it.  Outputs: state (n), counts (4n), per key slot (2n) seeds (32), paths (48), dids (55), per
// component reg_flags, per id id_flags; with pks (2n x 32) also the bodies: body_off (n + 1), body (the sizes pass's total) — the caller
// reads body_off[n] from a first call without pks.
int hs_didrr_run(const uint8_t* master, const uint8_t* server, uint64_t server_len, const uint8_t* agent_cols, const uint64_t* agent_col_off,
                 const uint32_t* agent_index, const uint64_t* id_idx, const uint8_t* ids, const uint64_t* id_off, const uint64_t* reg_idx,
                 const uint8_t* reg_cols, const uint64_t* reg_col_off, uint32_t n, const uint8_t* pks, uint8_t* state, uint32_t* counts,
                 uint8_t* seeds, uint8_t* paths, uint8_t* dids, uint8_t* reg_flags, uint8_t* id_flags, uint8_t* body, uint64_t* body_off) {
    const uint64_t ibase = id_idx[0], gbase = reg_idx[0];
    const uint32_t m = (uint32_t)(id_idx[2 * (size_t)n] - ibase), G = (uint32_t)(reg_idx[2 * (size_t)n] - gbase);
    const uint32_t h = didr_server_hash(server, server_len);
    std::vector<uint8_t> rflags(G + 1), iflags(m + 1);
    std::vector<uint64_t> ebytes(G + 1), esc(m + 1), before((size_t)G + m + 1), map_bytes(4 * (size_t)n), agent_bytes(n);
    std::vector<uint32_t> rank((size_t)G + m + 1), map_cnt(4 * (size_t)n), bad(n);
    for (uint32_t t = 0; t < G; t++) {                            // k_didrr_reg
        const uint64_t g = gbase + t;
        const uint32_t L = didr_list_of(reg_idx, n, g);
        const uint32_t f = didrr_reg_flags(reg_cols, reg_col_off, g, reg_idx[L], reg_idx[L + 1], ids, id_off, id_idx[L], id_idx[L + 1]);
        rflags[t] = (uint8_t)f;
        ebytes[t] = (f & DIDRR_R_GONE) ? 0 : didrr_stored_entry_bytes((L & 1) ? DIDR_SKILL : DIDR_REASONER, reg_cols, reg_col_off, g);
        if (f & DIDRR_R_DUP) bad[L >> 1] = 1;
    }
    for (uint32_t j = 0; j < m; j++) {                            // k_didrr_ids
        const uint64_t r = ibase + j;
        const uint32_t L = didr_list_of(id_idx, n, r);
        const uint32_t f = didrr_id_flags(ids, id_off, r, id_idx[L + 1], reg_cols, reg_col_off, reg_idx[L], reg_idx[L + 1]);
        iflags[j] = (uint8_t)f;
        esc[j] = f == (DIDRR_I_NONEMPTY | DIDRR_I_NEW) ? didr_esc_len(ids + id_off[r], id_off[r + 1] - id_off[r]) : 0;
    }
    for (uint64_t t = 0; t < (uint64_t)G + m; t++) {              // k_didrr_ranks
        if (t < G) {
            if (rflags[t] & DIDRR_R_GONE) continue;
            const uint64_t g = gbase + t;
            const uint32_t L = didr_list_of(reg_idx, n, g);
            const DidrRank q = didrr_reg_rank(reg_cols, reg_col_off, rflags.data(), ebytes.data(), gbase, g, reg_idx[L], reg_idx[L + 1]);
            rank[t] = q.rank; before[t] = q.before;
            if (q.rank + 1 == q.kept) { map_bytes[L] = q.before + ebytes[t] + q.rank; map_cnt[L] = q.kept; }
            continue;
        }
        const uint64_t j = t - G, r = ibase + j;
        if (iflags[j] != (DIDRR_I_NONEMPTY | DIDRR_I_NEW)) continue;
        const uint32_t L = didr_list_of(id_idx, n, r), kind = (L & 1) ? DIDR_SKILL : DIDR_REASONER;
        const uint32_t plen = didr_path_len(kind, h, agent_index[L >> 1], didrr_survivors(rflags.data(), gbase, reg_idx[L], reg_idx[L + 1]));
        const DidrRank q = didrr_id_rank(ids, id_off, iflags.data(), esc.data(), ibase, r, id_idx[L], id_idx[L + 1], kind, plen);
        rank[t] = q.rank; before[t] = q.before;
        if (q.rank + 1 == q.kept) { map_bytes[2 * (size_t)n + L] = q.before + didr_entry_bytes(kind, plen, esc[j]) + q.rank; map_cnt[2 * (size_t)n + L] = q.kept; }
    }
    body_off[0] = 0;
    for (uint32_t i = 0; i < n; i++) {                            // k_didrr_sizes, then the scan
        const size_t l = 2 * (size_t)i;
        uint32_t c[4] = {map_cnt[2 * (size_t)n + l], map_cnt[2 * (size_t)n + l + 1], (uint32_t)(reg_idx[l + 1] - reg_idx[l]) - map_cnt[l],
                         (uint32_t)(reg_idx[l + 2] - reg_idx[l + 1]) - map_cnt[l + 1]};
        const uint8_t st = didrr_state(bad[i] != 0, c[0], c[1], c[2], c[3]);
        state[i] = st;
        if (st == DIDRR_INVALID) c[0] = c[1] = c[2] = c[3] = 0;
        for (int k = 0; k < 4; k++) counts[4 * (size_t)i + k] = c[k];
        uint64_t len = 0;
        if (st != DIDRR_INVALID) {
            agent_bytes[i] = didrr_agent_bytes(agent_cols, agent_col_off, i);
            ByteCounter t; t.init();
            didrr_tail(t, server, server_len, st, c);
            len = didr_layout(agent_bytes[i], didrr_map_bytes(map_bytes.data(), n, st, i, 0), didrr_map_bytes(map_bytes.data(), n, st, i, 1)).tail + t.n;
        }
        body_off[i + 1] = body_off[i] + len;
    }
    uint32_t ms[8];
    for (int k = 0; k < 8; k++) ms[k] = bswap32(load_le32(master + 4 * k));
    for (uint32_t t = 0; t < 2 * n; t++) {                        // k_didrr_derive
        const uint32_t i = t >> 1, kind = (t & 1) ? DIDR_SKILL : DIDR_REASONER;
        memset(seeds + 32 * (size_t)t, 0, 32); memset(paths + 48 * (size_t)t, 0, 48);
        if (state[i] != DIDRR_PARTIAL || counts[4 * (size_t)i + (t & 1)] == 0) continue;
        const uint32_t a = agent_index[i], j0 = map_cnt[t];
        alignas(16) uint8_t tmp[48];
        { ByteWriter w; w.init(tmp); didr_put_path(w, kind, h, a, j0); for (uint32_t k = didr_path_len(kind, h, a, j0); k < 48; k++) w.put(0); w.finish(); }
        memcpy(paths + 48 * (size_t)t, tmp, 48);
        uint32_t seed[8];
        didr_derive(ms, tmp, didr_path_len(kind, h, a, j0), seed);
        for (int k = 0; k < 8; k++) store_le32(seeds + 32 * (size_t)t + 4 * k, seed[k]);
    }
    for (uint32_t t = 0; t < G; t++) {                            // k_didrr_emit
        const uint64_t g = gbase + t;
        const uint32_t L = didr_list_of(reg_idx, n, g), i = L >> 1, kind = (L & 1) ? DIDR_SKILL : DIDR_REASONER;
        const uint8_t st = state[i];
        const bool gone = (rflags[t] & DIDRR_R_GONE) != 0;
        reg_flags[t] = st != DIDRR_INVALID && gone ? DIDRR_GONE : 0;
        if (!pks || !((st == DIDRR_UNCHANGED || st == DIDRR_REMOVED) && !gone)) continue;
        const uint64_t at = didrr_at(map_bytes.data(), agent_bytes.data(), rank.data(), before.data(), n, st, i, kind, t);
        ByteWriter w; w.init(body + body_off[i] + at - (rank[t] ? 1 : 0));
        if (rank[t]) w.put(',');
        didrr_stored_entry(w, kind, reg_cols, reg_col_off, g);
        w.finish();
    }
    for (uint32_t j = 0; j < m; j++) {                            // k_didrr_emit_new
        const uint64_t r = ibase + j, t = (uint64_t)G + j;
        const uint32_t L = didr_list_of(id_idx, n, r), i = L >> 1, kind = (L & 1) ? DIDR_SKILL : DIDR_REASONER;
        const uint8_t st = state[i];
        const uint32_t f = iflags[j];
        const bool nw = st == DIDRR_PARTIAL && (f & DIDRR_I_NEW);
        id_flags[j] = nw ? (uint8_t)(DIDRR_NEW | ((f & DIDRR_I_SHADOWED) ? 0 : 1)) : 0;
        if (!pks || !nw || (f & DIDRR_I_SHADOWED)) continue;
        const uint64_t at = didrr_at(map_bytes.data(), agent_bytes.data(), rank.data(), before.data(), n, st, i, kind, t);
        const size_t slot = 2 * (size_t)i + (L & 1);
        uint32_t pk[8], seed[8];
        for (int k = 0; k < 8; k++) { pk[k] = load_le32(pks + 32 * slot + 4 * k); seed[k] = load_le32(seeds + 32 * slot + 4 * k); }
        ByteWriter w; w.init(body + body_off[i] + at - (rank[t] ? 1 : 0));
        if (rank[t]) w.put(',');
        didr_entry(w, kind, h, agent_index[i], map_cnt[L], pk, seed, ids + id_off[r], id_off[r + 1] - id_off[r]);
        w.finish();
    }
    if (!pks) return 0;
    for (uint32_t i = 0; i < n; i++) {                            // k_didrr_frame
        const uint8_t st = state[i];
        uint32_t c[4];
        for (int k = 0; k < 4; k++) c[k] = counts[4 * (size_t)i + k];
        for (uint32_t kind = 0; kind < 2; kind++) {
            const size_t slot = 2 * (size_t)i + kind;
            memset(dids + 55 * slot, 0, 55);
            if (st != DIDRR_PARTIAL || !c[kind]) continue;
            uint32_t pk[8];
            for (int k = 0; k < 8; k++) pk[k] = load_le32(pks + 32 * slot + 4 * k);
            ByteWriter w; w.init(dids + 55 * slot); didr_put_did(w, pk); w.finish();
        }
        if (st == DIDRR_INVALID) continue;
        const uint64_t rb = didrr_map_bytes(map_bytes.data(), n, st, i, 0), sb = didrr_map_bytes(map_bytes.data(), n, st, i, 1);
        const DidrLayout Lo = didr_layout(agent_bytes[i], rb, sb);
        uint8_t* b = body + body_off[i];
        { ByteWriter w; w.init(b); vci_put_text(w, DIDR_L_HEAD); w.finish(); }
        { ByteWriter w; w.init(b + Lo.agent); didrr_agent(w, agent_cols, agent_col_off, i); vci_put_text(w, DIDR_L_RMAP); w.finish(); }
        { ByteWriter w; w.init(b + Lo.rmap + rb); vci_put_text(w, DIDR_L_SMAP); w.finish(); }
        ByteWriter w; w.init(b + Lo.tail);
        didrr_tail(w, server, server_len, st, c);
        w.finish();
    }
    return 0;
}

}  // extern "C"
