// TEST-ONLY CPU build of the DID-registration routines (agentfield_b200/csrc/afc_didreg.cuh): what the threads of k_didr_ids,
// k_didr_ranks, k_didr_sizes, k_didr_derive, k_didr_emit and k_didr_frame do, run one after another over a whole batch, with the
// kernels' own list and slot mapping (didr_list_of, didr_slot).  The Ed25519
// expansion is not here: the caller passes the public keys.  Compiled on its own by tests/test_didreg_hostsim.py.
#define AFC_HOSTSIM 1
#include <vector>

#include "../../agentfield_b200/csrc/afc_didreg.cuh"

using namespace afc;

extern "C" {

uint32_t hs_didr_fnv1a(const uint8_t* p, uint64_t n) { return didr_fnv1a(p, n); }
uint32_t hs_didr_server_hash(const uint8_t* p, uint64_t n) { return didr_server_hash(p, n); }

// the path text into out (at least 48 bytes); returns its length, and -1 if didr_path_len disagrees
int hs_didr_path(uint32_t kind, uint32_t h, uint32_t a, uint32_t j, uint8_t* out) {
    ByteWriter w; w.init(out);
    didr_put_path(w, kind, h, a, j);
    w.finish();
    ByteCounter c; c.init();
    didr_put_path(c, kind, h, a, j);
    return c.n == didr_path_len(kind, h, a, j) ? (int)c.n : -1;
}

// base64url of n x 32 bytes: 43 characters each
void hs_didr_b64_32(const uint8_t* in, uint64_t n, uint8_t* out) {
    for (uint64_t i = 0; i < n; i++) {
        uint32_t w[8];
        for (int k = 0; k < 8; k++) w[k] = load_le32(in + 32 * i + 4 * k);
        ByteWriter b; b.init(out + 43 * i);
        didr_b64_32(b, w);
        b.finish();
    }
}
void hs_didr_did(const uint8_t* pk, uint8_t* out) {
    uint32_t w[8];
    for (int k = 0; k < 8; k++) w[k] = load_le32(pk + 4 * k);
    ByteWriter b; b.init(out);
    didr_put_did(b, w);
    b.finish();
}

// the identity's (map entry's, for a reasoner or skill) length counted by ByteCounter and by didr_entry_bytes / didr_identity_bytes
void hs_didr_entry_bytes(uint32_t kind, uint32_t h, uint32_t a, uint32_t j, const uint8_t* id, uint64_t len, uint64_t* counted, uint64_t* arith) {
    const uint32_t z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    ByteCounter c; c.init();
    if (kind == DIDR_AGENT) didr_identity(c, kind, h, a, j, z, z, id, len);
    else didr_entry(c, kind, h, a, j, z, z, id, len);
    *counted = c.n;
    const uint32_t pl = didr_path_len(kind, h, a, j), esc = (uint32_t)didr_esc_len(id, len);
    *arith = kind == DIDR_AGENT ? didr_identity_bytes(kind, pl, 0) : didr_entry_bytes(kind, pl, esc);
}

// The batch, as the kernels compute it.  Outputs: comp_off (n + 1), per id flags / rank, per component (n + m entries) seeds, paths (48
// each), dids (55 each), kept; with pks (component order) also the bodies: body_off (n + 1), body (the sizes pass's total) — the caller
// reads body_off[n] from a first call without pks.
int hs_didr_run(const uint8_t* master, const uint8_t* server, uint64_t server_len, const uint8_t* nodes, const uint64_t* node_off,
                const uint32_t* agent_index, const uint64_t* id_idx, const uint8_t* ids, const uint64_t* id_off, uint32_t n, const uint8_t* pks,
                uint64_t* comp_off, uint8_t* id_flags, uint32_t* id_rank, uint8_t* seeds, uint8_t* paths, uint8_t* dids, uint8_t* kept,
                uint8_t* body, uint64_t* body_off) {
    const uint64_t base = id_idx[0];
    const uint32_t m = (uint32_t)(id_idx[2 * (size_t)n] - base);
    const uint32_t h = didr_server_hash(server, server_len);
    std::vector<uint32_t> list(m + 1), rank(m + 1);
    std::vector<uint8_t> flags(m + 1);
    std::vector<uint64_t> esc(m + 1), nz(m + 1), before(m + 1), mapb(2 * (size_t)n), blen(n + 1);
    std::vector<uint32_t> mapc(2 * (size_t)n);
    for (uint32_t j = 0; j < m; j++) {                            // k_didr_ids
        const uint64_t r = base + j;
        const uint32_t L = didr_list_of(id_idx, n, r);
        list[j] = L;
        flags[j] = (uint8_t)didr_id_flags(ids, id_off, r, id_idx[L + 1]);
        esc[j] = flags[j] ? didr_esc_len(ids + id_off[r], id_off[r + 1] - id_off[r]) : 0;
    }
    nz[0] = 0;                                                    // the scan
    for (uint32_t j = 0; j < m; j++) nz[j + 1] = nz[j] + (flags[j] ? 1 : 0);
    for (uint32_t j = 0; j < m; j++) {                            // k_didr_ranks
        if (flags[j] != DIDR_F_NONEMPTY) continue;
        const uint32_t L = list[j], kind = (L & 1) ? DIDR_SKILL : DIDR_REASONER, a = agent_index[L >> 1];
        const DidrRank q = didr_rank(ids, id_off, flags.data(), esc.data(), nz.data(), base, base + j, id_idx[L], id_idx[L + 1], kind, h, a);
        rank[j] = q.rank; before[j] = q.before;
        if (q.rank + 1 == q.kept) {
            mapb[L] = q.before + didr_entry_bytes(kind, didr_path_len(kind, h, a, (uint32_t)(nz[j] - nz[id_idx[L] - base])), esc[j]) + q.rank;
            mapc[L] = q.kept;
        }
    }
    for (uint32_t j = 0; j < m; j++) { id_flags[j] = flags[j]; id_rank[j] = flags[j] == DIDR_F_NONEMPTY ? rank[j] : 0; }
    std::vector<uint64_t> agent_bytes(n);
    comp_off[0] = 0;
    body_off[0] = 0;
    for (uint32_t i = 0; i < n; i++) {                            // k_didr_sizes, then the scan
        comp_off[i + 1] = (uint64_t)i + 1 + nz[id_idx[2 * (size_t)i + 2] - base];
        ByteCounter c; c.init();
        didr_tail(c, server, server_len, nodes + node_off[i], node_off[i + 1] - node_off[i], mapc[2 * i], mapc[2 * i + 1]);
        agent_bytes[i] = didr_identity_bytes(DIDR_AGENT, didr_path_len(DIDR_AGENT, h, agent_index[i], 0), 0);
        body_off[i + 1] = body_off[i] + didr_layout(agent_bytes[i], mapb[2 * i], mapb[2 * i + 1]).tail + c.n;
    }
    uint32_t ms[8];
    for (int k = 0; k < 8; k++) ms[k] = bswap32(load_le32(master + 4 * k));
    for (uint64_t t = 0; t < (uint64_t)n + m; t++) {              // k_didr_derive and k_didr_emit
        const DidrSlot sl = didr_slot(id_idx, list.data(), flags.data(), nz.data(), n, m, t);
        const uint32_t i = sl.i, kind = sl.kind, jx = sl.j;
        const uint64_t c = sl.c, r = sl.r;
        const bool comp = sl.comp, kp = comp && (kind == DIDR_AGENT || flags[t - n] == DIDR_F_NONEMPTY);
        uint8_t* slot = paths + 48 * c;
        if (!comp) {
            memset(seeds + 32 * c, 0, 32); memset(slot, 0, 48); memset(dids + 55 * c, 0, 55); kept[c] = 0;
            continue;
        }
        const uint32_t a = agent_index[i];
        alignas(16) uint8_t tmp[48];
        { ByteWriter w; w.init(tmp); didr_put_path(w, kind, h, a, jx); for (uint32_t k = didr_path_len(kind, h, a, jx); k < 48; k++) w.put(0); w.finish(); }
        memcpy(slot, tmp, 48);
        uint32_t seed[8];
        didr_derive(ms, tmp, didr_path_len(kind, h, a, jx), seed);
        for (int k = 0; k < 8; k++) store_le32(seeds + 32 * c + 4 * k, seed[k]);
        kept[c] = kp ? 1 : 0;
        if (!pks) continue;
        uint32_t pk[8];
        for (int k = 0; k < 8; k++) pk[k] = load_le32(pks + 32 * c + 4 * k);
        { ByteWriter w; w.init(dids + 55 * c); didr_put_did(w, pk); w.finish(); }
        if (!kp) continue;
        const DidrLayout Lo = didr_layout(agent_bytes[i], mapb[2 * i], mapb[2 * i + 1]);
        uint8_t* b = body + body_off[i];
        if (kind == DIDR_AGENT) { ByteWriter w; w.init(b + Lo.agent); didr_identity(w, kind, h, a, 0, pk, seed, nullptr, 0); w.finish(); continue; }
        const uint64_t jj = t - n;
        const uint64_t at = (kind == DIDR_REASONER ? Lo.rmap : Lo.smap) + before[jj] + rank[jj];
        ByteWriter w; w.init(b + at - (rank[jj] ? 1 : 0));
        if (rank[jj]) w.put(',');
        didr_entry(w, kind, h, a, jx, pk, seed, ids + id_off[r], id_off[r + 1] - id_off[r]);
        w.finish();
    }
    if (!pks) return 0;
    for (uint32_t i = 0; i < n; i++) {                            // k_didr_frame
        const uint64_t rb = mapb[2 * i], sb = mapb[2 * i + 1];
        const DidrLayout Lo = didr_layout(agent_bytes[i], rb, sb);
        uint8_t* b = body + body_off[i];
        { ByteWriter w; w.init(b); vci_put_text(w, DIDR_L_HEAD); w.finish(); }
        { ByteWriter w; w.init(b + Lo.agent + agent_bytes[i]); vci_put_text(w, DIDR_L_RMAP); w.finish(); }
        { ByteWriter w; w.init(b + Lo.rmap + rb); vci_put_text(w, DIDR_L_SMAP); w.finish(); }
        ByteWriter w; w.init(b + Lo.tail);
        didr_tail(w, server, server_len, nodes + node_off[i], node_off[i + 1] - node_off[i], mapc[2 * i], mapc[2 * i + 1]);
        w.finish();
    }
    return 0;
}

}  // extern "C"
