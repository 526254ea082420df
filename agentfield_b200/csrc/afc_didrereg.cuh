// Known agents re-registered on the device (afc_did_reregister_batch, include/afcrypto.h): what RegisterAgent
// (internal/services/did_service.go:129-183) returns for an agent the registry already holds, and what it changes there.
//
//   didrr_reg_flags    PerformDifferentialAnalysis (:757-800) for one registered component: GONE when no non-empty id of the request's list
//                      of the same kind equals its key (setDifference(existing, new), extractReasonerIDs dropping empty ids), DUP when another
//                      component of its list has the same key (a Go map cannot hold that: the request is refused)
//   didrr_id_flags     the same for one request id: NEW when no registered key of its list equals it (setDifference(new, existing) keeps
//                      duplicates), SHADOWED when a later id of the list is equal (the map keeps that occurrence)
//   didrr_stored       buildExistingIdentityPackage (:940-986) for one component: the stored did, "" for the private JWK, the stored
//                      public_key_jwk (a json.RawMessage turned into a Go string, so escaped as stored), the stored path, the component
//                      type and the stored function_name (omitempty)
//   didrr_message      the three messages: unchanged (:167-175), removals only (:1039-1044), partial (PartialRegisterAgent :1231-1235)
//
// New components (PartialRegisterAgent :1049-1236) use afc_didreg.cuh's didr_entry, with the path generateReasonerPath / generateSkillPath
// (:870-937) build: m/44'/<h>'/<a>'/<0|1>'/<j>' where j is the size of the agent's map of that kind after the removals and before any
// addition.  So every new component of one kind in one request gets the same path, key and DID, and that DID can be a surviving
// component's (a defect of the reference, reproduced).
//
// Shared by the kernels of k_didrereg.cu and the CPU build of the same logic in tests/hostsim.
#pragma once
#include "afc_didreg.cuh"

namespace afc {

enum : uint8_t { DIDRR_UNCHANGED = 0, DIDRR_REMOVED = 1, DIDRR_PARTIAL = 2, DIDRR_INVALID = 3 };     // AFC_DIDRR_*
enum : uint8_t { DIDRR_GONE = 1, DIDRR_NEW = 2 };                                                   // AFC_DIDRR_GONE / AFC_DIDRR_NEW
enum : uint8_t { DIDRR_R_GONE = 1, DIDRR_R_DUP = 2 };                                               // a registered component, internal
enum : uint8_t { DIDRR_I_NONEMPTY = 1, DIDRR_I_SHADOWED = 2, DIDRR_I_NEW = 4 };                     // a request id, internal
enum { DIDRR_COLS = 5, DIDRR_AGENT_COLS = 3 };          // key, did, public_key_jwk, derivation_path, function_name; did, public_key_jwk, path

#define DIDRR_L_STORED "\",\"private_key_jwk\":\"\",\"public_key_jwk\":\""
#define DIDRR_L_PATH "\",\"derivation_path\":\""
#define DIDRR_L_MSG "\"},\"message\":\""
#define DIDRR_L_BODY_END "\"}"
#define DIDRR_M_SAME "No changes detected, registration skipped"
#define DIDRR_M_REMOVED "Registration updated: removed "
#define DIDRR_M_REMOVED_R " reasoners, "
#define DIDRR_M_REMOVED_S " skills"
#define DIDRR_M_PARTIAL "Partial registration successful: "
#define DIDRR_M_PARTIAL_R " new reasoners, "
#define DIDRR_M_PARTIAL_S " new skills"

// A stored identity's text but its four strings and the component type
constexpr uint64_t DIDRR_STORED_FIXED = DIDR_LEN(DIDR_L_DID) + DIDR_LEN(DIDRR_L_STORED) + DIDR_LEN(DIDRR_L_PATH) + DIDR_LEN(DIDR_L_TYPE) +
                                        DIDR_LEN(DIDR_L_END);
// Bounds of one request's body (afc_did_reregister_bound): the frame with the longest message and two 10-digit counts, and the agent's
// stored identity; per registered component its map entry with the longest type and a function_name; 6 bytes per escaped byte.  Per
// request id: afc_didreg.cuh's DIDR_PER_ID_FIXED and 12 bytes per id byte.
constexpr uint64_t DIDRR_REQ_FIXED = DIDR_LEN(DIDR_L_HEAD) + DIDR_LEN(DIDR_L_RMAP) + DIDR_LEN(DIDR_L_SMAP) + DIDR_LEN(DIDR_L_SERVER) +
                                     DIDR_LEN(DIDRR_L_MSG) + DIDR_LEN(DIDRR_M_PARTIAL) + DIDR_LEN(DIDRR_M_PARTIAL_R) + DIDR_LEN(DIDRR_M_PARTIAL_S) +
                                     20 + DIDR_LEN(DIDRR_L_BODY_END) + DIDRR_STORED_FIXED + 5;
constexpr uint64_t DIDRR_PER_REG_FIXED = 4 + DIDRR_STORED_FIXED + 8 + DIDR_LEN(DIDR_L_FN);

// ---- columns

struct DidrrStr { const uint8_t* p; uint64_t len; };
AFC_HD DidrrStr didrr_col(const uint8_t* cols, const uint64_t* col_off, uint64_t k) { DidrrStr s; s.p = cols + col_off[k]; s.len = col_off[k + 1] - col_off[k]; return s; }

// ---- the differential analysis

// Registered component g (absolute) of the list whose components are [rlo, rhi) and whose request ids are [ilo, ihi)
AFC_HD uint32_t didrr_reg_flags(const uint8_t* reg_cols, const uint64_t* reg_col_off, uint64_t g, uint64_t rlo, uint64_t rhi, const uint8_t* ids,
                                const uint64_t* id_off, uint64_t ilo, uint64_t ihi) {
    const DidrrStr key = didrr_col(reg_cols, reg_col_off, DIDRR_COLS * g);
    uint32_t f = DIDRR_R_GONE;
    for (uint64_t k = ilo; k < ihi; k++) {
        const uint64_t len = id_off[k + 1] - id_off[k];
        if (len && didr_eq(key.p, key.len, ids + id_off[k], len)) { f = 0; break; }
    }
    for (uint64_t k = rlo; k < rhi; k++) {
        if (k == g) continue;
        const DidrrStr o = didrr_col(reg_cols, reg_col_off, DIDRR_COLS * k);
        if (didr_eq(key.p, key.len, o.p, o.len)) { f |= DIDRR_R_DUP; break; }
    }
    return f;
}

// Request id r (absolute) of the list whose ids end before ihi and whose registered components are [rlo, rhi)
AFC_HD uint32_t didrr_id_flags(const uint8_t* ids, const uint64_t* id_off, uint64_t r, uint64_t ihi, const uint8_t* reg_cols,
                               const uint64_t* reg_col_off, uint64_t rlo, uint64_t rhi) {
    const uint8_t* s = ids + id_off[r];
    const uint64_t len = id_off[r + 1] - id_off[r];
    if (len == 0) return 0;
    for (uint64_t k = rlo; k < rhi; k++) {
        const DidrrStr o = didrr_col(reg_cols, reg_col_off, DIDRR_COLS * k);
        if (didr_eq(s, len, o.p, o.len)) return DIDRR_I_NONEMPTY;
    }
    for (uint64_t k = r + 1; k < ihi; k++)
        if (didr_eq(s, len, ids + id_off[k], id_off[k + 1] - id_off[k])) return DIDRR_I_NONEMPTY | DIDRR_I_NEW | DIDRR_I_SHADOWED;
    return DIDRR_I_NONEMPTY | DIDRR_I_NEW;
}

// ---- one stored identity

// json.Marshal(types.DIDIdentity) of buildExistingIdentityPackage.  c: did, public_key_jwk, derivation_path, function_name.
template <class Sink>
AFC_HD void didrr_stored(Sink& out, uint32_t kind, DidrrStr did, DidrrStr jwk, DidrrStr path, DidrrStr fn) {
    vci_put_text(out, DIDR_L_DID);
    go_json_escape(out, did.p, did.len);
    vci_put_text(out, DIDRR_L_STORED);
    go_json_escape(out, jwk.p, jwk.len);
    vci_put_text(out, DIDRR_L_PATH);
    go_json_escape(out, path.p, path.len);
    vci_put_text(out, DIDR_L_TYPE);
    vci_put_text(out, kind == DIDR_AGENT ? "agent" : kind == DIDR_REASONER ? "reasoner" : "skill");
    if (fn.len) {
        vci_put_text(out, DIDR_L_FN);
        go_json_escape(out, fn.p, fn.len);
    }
    vci_put_text(out, DIDR_L_END);
}
// A registered component's map entry: "key": identity
template <class Sink>
AFC_HD void didrr_stored_entry(Sink& out, uint32_t kind, const uint8_t* reg_cols, const uint64_t* reg_col_off, uint64_t g) {
    const uint64_t c = DIDRR_COLS * g;
    const DidrrStr key = didrr_col(reg_cols, reg_col_off, c);
    out.put('"');
    go_json_escape(out, key.p, key.len);
    out.put('"'); out.put(':');
    didrr_stored(out, kind, didrr_col(reg_cols, reg_col_off, c + 1), didrr_col(reg_cols, reg_col_off, c + 2), didrr_col(reg_cols, reg_col_off, c + 3),
                 didrr_col(reg_cols, reg_col_off, c + 4));
}
AFC_HD uint64_t didrr_stored_entry_bytes(uint32_t kind, const uint8_t* reg_cols, const uint64_t* reg_col_off, uint64_t g) {
    ByteCounter c; c.init();
    didrr_stored_entry(c, kind, reg_cols, reg_col_off, g);
    return c.n;
}
// The agent's identity from its three columns (did, public_key_jwk, derivation_path) starting at agent_col_off[3 i]
template <class Sink>
AFC_HD void didrr_agent(Sink& out, const uint8_t* agent_cols, const uint64_t* agent_col_off, uint64_t i) {
    const uint64_t c = DIDRR_AGENT_COLS * i;
    DidrrStr none; none.p = nullptr; none.len = 0;
    didrr_stored(out, DIDR_AGENT, didrr_col(agent_cols, agent_col_off, c), didrr_col(agent_cols, agent_col_off, c + 1),
                 didrr_col(agent_cols, agent_col_off, c + 2), none);
}
AFC_HD uint64_t didrr_agent_bytes(const uint8_t* agent_cols, const uint64_t* agent_col_off, uint64_t i) {
    ByteCounter c; c.init();
    didrr_agent(c, agent_cols, agent_col_off, i);
    return c.n;
}

// ---- ranks in the maps

// Registered component g among its list's survivors [lo, hi) (rflags, ebytes indexed by absolute index - base)
AFC_HD DidrRank didrr_reg_rank(const uint8_t* reg_cols, const uint64_t* reg_col_off, const uint8_t* rflags, const uint64_t* ebytes, uint64_t base,
                               uint64_t g, uint64_t lo, uint64_t hi) {
    DidrRank r; r.rank = 0; r.kept = 0; r.before = 0;
    const DidrrStr key = didrr_col(reg_cols, reg_col_off, DIDRR_COLS * g);
    for (uint64_t k = lo; k < hi; k++) {
        if (rflags[k - base] & DIDRR_R_GONE) continue;
        r.kept++;
        const DidrrStr o = didrr_col(reg_cols, reg_col_off, DIDRR_COLS * k);
        if (!didr_less(o.p, o.len, key.p, key.len)) continue;
        r.rank++;
        r.before += ebytes[k - base];
    }
    return r;
}
// The survivors of a list: its size after the removals (j of every new component of that kind)
AFC_HD uint32_t didrr_survivors(const uint8_t* rflags, uint64_t base, uint64_t lo, uint64_t hi) {
    uint32_t s = 0;
    for (uint64_t k = lo; k < hi; k++) s += (rflags[k - base] & DIDRR_R_GONE) ? 0 : 1;
    return s;
}
// Request id r among its list's kept new ids [lo, hi) (iflags, esc indexed by absolute index - base); plen: their common path's length
AFC_HD DidrRank didrr_id_rank(const uint8_t* ids, const uint64_t* id_off, const uint8_t* iflags, const uint64_t* esc, uint64_t base, uint64_t r,
                              uint64_t lo, uint64_t hi, uint32_t kind, uint32_t plen) {
    DidrRank q; q.rank = 0; q.kept = 0; q.before = 0;
    const uint8_t* s = ids + id_off[r];
    const uint64_t len = id_off[r + 1] - id_off[r];
    for (uint64_t k = lo; k < hi; k++) {
        if (iflags[k - base] != (DIDRR_I_NONEMPTY | DIDRR_I_NEW)) continue;
        q.kept++;
        if (!didr_less(ids + id_off[k], id_off[k + 1] - id_off[k], s, len)) continue;
        q.rank++;
        q.before += didr_entry_bytes(kind, plen, esc[k - base]);
    }
    return q;
}

// ---- one request's frame

// The request's state from its lists: dup (a registered list repeats a key), the distinct new ids and the removed components per kind
AFC_HD uint8_t didrr_state(bool dup, uint32_t new_r, uint32_t new_s, uint32_t gone_r, uint32_t gone_s) {
    if (dup) return DIDRR_INVALID;
    if (new_r || new_s) return DIDRR_PARTIAL;
    return (gone_r || gone_s) ? DIDRR_REMOVED : DIDRR_UNCHANGED;
}
// counts: new reasoners, new skills, removed reasoners, removed skills
template <class Sink>
AFC_HD void didrr_message(Sink& out, uint8_t state, const uint32_t counts[4]) {
    if (state == DIDRR_UNCHANGED) { vci_put_text(out, DIDRR_M_SAME); return; }
    const bool p = state == DIDRR_PARTIAL;
    vci_put_text(out, p ? DIDRR_M_PARTIAL : DIDRR_M_REMOVED);
    vci_put_int(out, (int64_t)counts[p ? 0 : 2]);
    vci_put_text(out, p ? DIDRR_M_PARTIAL_R : DIDRR_M_REMOVED_R);
    vci_put_int(out, (int64_t)counts[p ? 1 : 3]);
    vci_put_text(out, p ? DIDRR_M_PARTIAL_S : DIDRR_M_REMOVED_S);
}
// From the skill map's '}' to the end: the server id and the message
template <class Sink>
AFC_HD void didrr_tail(Sink& out, const uint8_t* server, uint64_t server_len, uint8_t state, const uint32_t counts[4]) {
    vci_put_text(out, DIDR_L_SERVER);
    go_json_escape(out, server, server_len);
    vci_put_text(out, DIDRR_L_MSG);
    didrr_message(out, state, counts);
    vci_put_text(out, DIDRR_L_BODY_END);
}

// ---- where things go

// The map bytes of request i's body: the new maps for a partial registration, the surviving ones otherwise
AFC_HD uint64_t didrr_map_bytes(const uint64_t* map_bytes, uint32_t n, uint8_t st, uint32_t i, uint32_t kind) {
    return map_bytes[(st == DIDRR_PARTIAL ? 2 * (size_t)n : 0) + 2 * (size_t)i + kind];
}

// The place of item t's entry in its body (after the comma that precedes it when it is not its map's first)
AFC_HD uint64_t didrr_at(const uint64_t* map_bytes, const uint64_t* agent_bytes, const uint32_t* rank, const uint64_t* before, uint32_t n, uint8_t st,
                         uint32_t i, uint32_t kind, uint64_t t) {
    const DidrLayout Lo = didr_layout(agent_bytes[i], didrr_map_bytes(map_bytes, n, st, i, 0), didrr_map_bytes(map_bytes, n, st, i, 1));
    return (kind == DIDR_REASONER ? Lo.rmap : Lo.smap) + before[t] + rank[t];
}

}  // namespace afc
