// Agent DIDs registered on the device (afc_did_register_batch, include/afcrypto.h): what handleNewRegistration
// (internal/services/did_service.go:186-365) derives and returns for one DIDRegistrationRequest.
//
//   didr_server_hash   hashAgentFieldServerID (:578-582): FNV-1a 32 of the server id, mod 2^31.
//   didr_put_path      the derivation paths m/44'/<h>'/<a>' (agent), .../0'/<j>' (reasoner j), .../1'/<j>' (skill j) (:222, :244, :290);
//                      j counts the non-empty ids before this one in its list: empty ids are skipped and take no index (:227-265, :273-311).
//   didr_derive        derivePrivateKey (:515-525): SHA-256(masterSeed || path), 43..76 bytes, one or two blocks.
//   didr_identity      types.DIDIdentity (pkg/types/did_types.go:114-121) as json.Marshal writes it: did:key:z + base64url(0xED 0x01 || pk)
//                      (generateDIDKey :528-536), the private and public JWK texts (:538-575: json.Marshal of a map, so keys sorted) as
//                      JSON strings, the path, the component type and, for reasoners and skills, function_name (omitempty).
//   didr_rank          the map[string]DIDIdentity of one list: a repeated id is derived (it takes an index) but the map keeps the last
//                      assignment, so earlier occurrences are shadowed; json.Marshal writes the kept keys in raw byte order.
//   didr_tail          the rest of json.Marshal(types.DIDRegistrationResponse) (did_types.go:106-111, 253-265): the server id and the message
//                      "Successfully registered agent %s with %d reasoners and %d skills", the counts being the maps' sizes.
//
// Secrets: the derived seed (the private JWK's "d") and everything computed from it.  didr_derive and the base64url below neither branch
// on nor index memory by secret bytes: base64url is computed arithmetically per character, as libsodium's sodium_bin2base64 does, with no
// alphabet table.
//
// Shared by the kernels of k_didreg.cu and the CPU build of the same logic in tests/hostsim.
#pragma once
#include "afc_vcissue.cuh"

namespace afc {

enum : uint32_t { DIDR_AGENT = 0, DIDR_REASONER = 1, DIDR_SKILL = 2 };
enum {
    DIDR_DID_CHARS = 55,     // did:key:z + 46 base64url characters
    DIDR_PATH_SLOT = 48,     // paths output: one NUL-padded slot per component (AFC_DID_PATH_SLOT)
    DIDR_PATH_MAX = 44,      // m/44'/<10 digits>'/<10 digits>'/0'/<10 digits>'
    DIDR_B64_32 = 43,        // base64url of 32 bytes, no padding
};
enum : uint8_t { DIDR_F_NONEMPTY = 1, DIDR_F_SHADOWED = 2 };

// The constant text.  The JWKs are JSON strings inside the identity, so their quotes are escaped.
#define DIDR_L_DID "{\"did\":\""
#define DIDR_L_PRIV "\",\"private_key_jwk\":\"{\\\"alg\\\":\\\"EdDSA\\\",\\\"crv\\\":\\\"Ed25519\\\",\\\"d\\\":\\\""
#define DIDR_L_PRIV_X "\\\",\\\"kty\\\":\\\"OKP\\\",\\\"use\\\":\\\"sig\\\",\\\"x\\\":\\\""
#define DIDR_L_PUB "\\\"}\",\"public_key_jwk\":\"{\\\"alg\\\":\\\"EdDSA\\\",\\\"crv\\\":\\\"Ed25519\\\",\\\"kty\\\":\\\"OKP\\\",\\\"use\\\":\\\"sig\\\",\\\"x\\\":\\\""
#define DIDR_L_PATH "\\\"}\",\"derivation_path\":\""
#define DIDR_L_TYPE "\",\"component_type\":\""
#define DIDR_L_FN "\",\"function_name\":\""
#define DIDR_L_END "\"}"
#define DIDR_L_HEAD "{\"success\":true,\"identity_package\":{\"agent_did\":"
#define DIDR_L_RMAP ",\"reasoner_dids\":{"
#define DIDR_L_SMAP "},\"skill_dids\":{"
#define DIDR_L_SERVER "},\"agentfield_server_id\":\""
#define DIDR_L_MSG "\"},\"message\":\"Successfully registered agent "
#define DIDR_L_WITH " with "
#define DIDR_L_REAS " reasoners and "
#define DIDR_L_SKILLS " skills\"}"
#define DIDR_LEN(lit) ((uint64_t)sizeof(lit) - 1)

// Every identity's text but the path, the type and function_name: did, both JWKs (three base64url keys)
constexpr uint64_t DIDR_ID_FIXED = DIDR_LEN(DIDR_L_DID) + DIDR_DID_CHARS + DIDR_LEN(DIDR_L_PRIV) + DIDR_B64_32 + DIDR_LEN(DIDR_L_PRIV_X) + DIDR_B64_32 +
                                   DIDR_LEN(DIDR_L_PUB) + DIDR_B64_32 + DIDR_LEN(DIDR_L_PATH) + DIDR_LEN(DIDR_L_TYPE) + DIDR_LEN(DIDR_L_END);
// The response around the identities and maps, but the escaped server and node ids and the two counts
constexpr uint64_t DIDR_FRAME_FIXED = DIDR_LEN(DIDR_L_HEAD) + DIDR_LEN(DIDR_L_RMAP) + DIDR_LEN(DIDR_L_SMAP) + DIDR_LEN(DIDR_L_SERVER) +
                                      DIDR_LEN(DIDR_L_MSG) + DIDR_LEN(DIDR_L_WITH) + DIDR_LEN(DIDR_L_REAS) + DIDR_LEN(DIDR_L_SKILLS);
// Bounds of one request's body (afc_did_register_bound): the frame with two 10-digit counts and the agent's identity with the longest
// agent path; per id its map entry ("key": identity, a comma) with the longest path and type, and 6 bytes per id byte for each of its two
// appearances (the key, function_name).  Node and server ids: 6 bytes per byte.
constexpr uint64_t DIDR_REQ_FIXED = DIDR_FRAME_FIXED + 20 + DIDR_ID_FIXED + 29 + 5;
constexpr uint64_t DIDR_PER_ID_FIXED = 4 + DIDR_ID_FIXED + DIDR_PATH_MAX + 8 + DIDR_LEN(DIDR_L_FN);

// ---- numbers and paths

AFC_HD uint32_t didr_fnv1a(const uint8_t* p, uint64_t n) {
    uint32_t h = 2166136261u;
    for (uint64_t k = 0; k < n; k++) h = (h ^ p[k]) * 16777619u;
    return h;
}
AFC_HD uint32_t didr_server_hash(const uint8_t* p, uint64_t n) { return didr_fnv1a(p, n) & 0x7fffffffu; }

AFC_HD uint32_t didr_digits(uint32_t v) {
    uint32_t d = 1;
    for (uint64_t p = 10; p <= v; p *= 10) d++;
    return d;
}
AFC_HD uint32_t didr_path_len(uint32_t kind, uint32_t h, uint32_t a, uint32_t j) {
    return 9 + didr_digits(h) + didr_digits(a) + (kind != DIDR_AGENT ? 5 + didr_digits(j) : 0);
}
template <class Sink>
AFC_HD void didr_put_path(Sink& out, uint32_t kind, uint32_t h, uint32_t a, uint32_t j) {
    out.put('m'); out.put('/'); out.put('4'); out.put('4'); out.put('\''); out.put('/');
    vci_put_int(out, (int64_t)h);
    out.put('\''); out.put('/');
    vci_put_int(out, (int64_t)a);
    out.put('\'');
    if (kind == DIDR_AGENT) return;
    out.put('/'); out.put(kind == DIDR_REASONER ? '0' : '1'); out.put('\''); out.put('/');
    vci_put_int(out, (int64_t)j);
    out.put('\'');
}

// ---- derivation

// SHA-256(master || path) as 8 little-endian words of the digest bytes (the seed the expansion kernels load).  master: the 32-byte
// master seed as big-endian words; slot: the path, NUL-padded to DIDR_PATH_SLOT bytes, 16-byte aligned; len: its length (<= 44).
AFC_HD void didr_derive(const uint32_t master[8], const uint8_t* slot, uint32_t len, uint32_t seed_le[8]) {
    uint32_t pw[12];
#pragma unroll
    for (int q = 0; q < 3; q++) {
        const word4 v = ld_u128(slot + 16 * q);
        pw[4 * q] = bswap32(v.x); pw[4 * q + 1] = bswap32(v.y); pw[4 * q + 2] = bswap32(v.z); pw[4 * q + 3] = bswap32(v.w);
    }
#pragma unroll
    for (uint32_t k = 0; k < 12; k++) pw[k] |= (k == (len >> 2)) ? 0x80u << (24 - 8 * (len & 3)) : 0u;     // the padding byte
    const uint32_t bits = (32 + len) * 8;
    uint32_t st[8], w[16];
    sha256_init(st);
#pragma unroll
    for (int k = 0; k < 8; k++) { w[k] = master[k]; w[8 + k] = pw[k]; }
    if (32 + len <= 55) {
        w[15] = bits;
        sha256_compress(st, w);
    } else {
        sha256_compress(st, w);
#pragma unroll
        for (int k = 0; k < 16; k++) w[k] = k < 4 ? pw[8 + k] : 0u;
        w[15] = bits;
        sha256_compress(st, w);
    }
#pragma unroll
    for (int k = 0; k < 8; k++) seed_le[k] = bswap32(st[k]);
}

// ---- base64url without a table

// The base64url character of a 6-bit value: masks from arithmetic alone, so nothing depends on x but the result
AFC_HD uint32_t didr_b64_char(uint32_t x) {
    const uint32_t lt26 = 0u - ((x - 26u) >> 31), lt52 = 0u - ((x - 52u) >> 31), lt62 = 0u - ((x - 62u) >> 31);
    const uint32_t eq62 = 0u - (((x ^ 62u) - 1u) >> 31), eq63 = 0u - (((x ^ 63u) - 1u) >> 31);
    return (lt26 & (x + 65u)) | (~lt26 & lt52 & (x + 71u)) | (~lt52 & lt62 & (x - 4u)) | (eq62 & 45u) | (eq63 & 95u);    // 'A', 'a' - 26, '0' - 52, '-', '_'
}
template <class Sink>
AFC_HD void didr_b64_group(Sink& out, uint32_t v, uint32_t chars) {     // v: three bytes, first in bits 16..23
    out.put(didr_b64_char((v >> 18) & 63));
    out.put(didr_b64_char((v >> 12) & 63));
    if (chars > 2) out.put(didr_b64_char((v >> 6) & 63));
    if (chars > 3) out.put(didr_b64_char(v & 63));
}
AFC_HD uint32_t didr_byte(const uint32_t w[8], uint32_t k) { return (w[k >> 2] >> (8 * (k & 3))) & 0xffu; }

// base64.RawURLEncoding of 32 bytes held as little-endian words: 43 characters
template <class Sink>
AFC_HD void didr_b64_32(Sink& out, const uint32_t w[8]) {
#pragma unroll
    for (uint32_t k = 0; k < 30; k += 3) didr_b64_group(out, didr_byte(w, k) << 16 | didr_byte(w, k + 1) << 8 | didr_byte(w, k + 2), 4);
    didr_b64_group(out, didr_byte(w, 30) << 16 | didr_byte(w, 31) << 8, 3);
}
// did:key:z + base64.RawURLEncoding(0xED 0x01 || pk): 55 characters
template <class Sink>
AFC_HD void didr_put_did(Sink& out, const uint32_t pk[8]) {
    vci_put_text(out, "did:key:z");
    didr_b64_group(out, 0xED0100u | didr_byte(pk, 0), 4);
#pragma unroll
    for (uint32_t k = 1; k < 31; k += 3) didr_b64_group(out, didr_byte(pk, k) << 16 | didr_byte(pk, k + 1) << 8 | didr_byte(pk, k + 2), 4);
    didr_b64_group(out, didr_byte(pk, 31) << 16, 2);
}

// ---- one identity

// json.Marshal(types.DIDIdentity).  id: the reasoner or skill id (function_name), unused for the agent.
template <class Sink>
AFC_HD void didr_identity(Sink& out, uint32_t kind, uint32_t h, uint32_t a, uint32_t j, const uint32_t pk[8], const uint32_t seed[8], const uint8_t* id,
                          uint64_t id_len) {
    vci_put_text(out, DIDR_L_DID);
    didr_put_did(out, pk);
    vci_put_text(out, DIDR_L_PRIV);
    didr_b64_32(out, seed);
    vci_put_text(out, DIDR_L_PRIV_X);
    didr_b64_32(out, pk);
    vci_put_text(out, DIDR_L_PUB);
    didr_b64_32(out, pk);
    vci_put_text(out, DIDR_L_PATH);
    didr_put_path(out, kind, h, a, j);
    vci_put_text(out, DIDR_L_TYPE);
    vci_put_text(out, kind == DIDR_AGENT ? "agent" : kind == DIDR_REASONER ? "reasoner" : "skill");
    if (kind != DIDR_AGENT) {
        vci_put_text(out, DIDR_L_FN);
        go_json_escape(out, id, id_len);
    }
    vci_put_text(out, DIDR_L_END);
}
// Its length from the escaped id's (esc) and the path's
AFC_HD uint64_t didr_identity_bytes(uint32_t kind, uint32_t path_len, uint64_t esc) {
    const uint64_t t = kind == DIDR_AGENT ? 5 : kind == DIDR_REASONER ? 8 : 5;
    return DIDR_ID_FIXED + path_len + t + (kind != DIDR_AGENT ? DIDR_LEN(DIDR_L_FN) + esc : 0);
}
// A map entry: "key": identity (the comma before every entry but the first is counted by the map)
template <class Sink>
AFC_HD void didr_entry(Sink& out, uint32_t kind, uint32_t h, uint32_t a, uint32_t j, const uint32_t pk[8], const uint32_t seed[8], const uint8_t* id,
                       uint64_t id_len) {
    out.put('"');
    go_json_escape(out, id, id_len);
    out.put('"'); out.put(':');
    didr_identity(out, kind, h, a, j, pk, seed, id, id_len);
}
AFC_HD uint64_t didr_entry_bytes(uint32_t kind, uint32_t path_len, uint64_t esc) { return esc + 3 + didr_identity_bytes(kind, path_len, esc); }

AFC_HD uint64_t didr_esc_len(const uint8_t* s, uint64_t len) {
    ByteCounter c; c.init();
    go_json_escape(c, s, len);
    return c.n;
}

// ---- one list of ids (a request's reasoners or its skills)

AFC_HD bool didr_eq(const uint8_t* a, uint64_t al, const uint8_t* b, uint64_t bl) {
    if (al != bl) return false;
    for (uint64_t k = 0; k < al; k++) if (a[k] != b[k]) return false;
    return true;
}
AFC_HD bool didr_less(const uint8_t* a, uint64_t al, const uint8_t* b, uint64_t bl) {     // Go's a < b on strings: raw bytes
    const uint64_t m = al < bl ? al : bl;
    for (uint64_t k = 0; k < m; k++) if (a[k] != b[k]) return a[k] < b[k];
    return al < bl;
}

// Id `me` (absolute index) of the list that ends before absolute index `hi`: DIDR_F_NONEMPTY, and DIDR_F_SHADOWED when a later id of the
// list is equal (the map keeps that one)
AFC_HD uint32_t didr_id_flags(const uint8_t* ids, const uint64_t* id_off, uint64_t me, uint64_t hi) {
    const uint8_t* s = ids + id_off[me];
    const uint64_t len = id_off[me + 1] - id_off[me];
    if (len == 0) return 0;
    for (uint64_t k = me + 1; k < hi; k++)
        if (didr_eq(s, len, ids + id_off[k], id_off[k + 1] - id_off[k])) return DIDR_F_NONEMPTY | DIDR_F_SHADOWED;
    return DIDR_F_NONEMPTY;
}

// Where a kept id's entry goes in its map: rank = kept ids with a smaller key, before = the bytes of their entries; kept = the map's size.
// List [lo, hi) in absolute indices; flags, esc and nz (the exclusive scan of the non-empty flags) are indexed by absolute index - base.
struct DidrRank { uint32_t rank, kept; uint64_t before; };
AFC_HD DidrRank didr_rank(const uint8_t* ids, const uint64_t* id_off, const uint8_t* flags, const uint64_t* esc, const uint64_t* nz, uint64_t base,
                          uint64_t me, uint64_t lo, uint64_t hi, uint32_t kind, uint32_t h, uint32_t a) {
    DidrRank r; r.rank = 0; r.kept = 0; r.before = 0;
    const uint8_t* s = ids + id_off[me];
    const uint64_t len = id_off[me + 1] - id_off[me];
    const uint64_t j0 = nz[lo - base];
    for (uint64_t k = lo; k < hi; k++) {
        if (flags[k - base] != DIDR_F_NONEMPTY) continue;
        r.kept++;
        if (!didr_less(ids + id_off[k], id_off[k + 1] - id_off[k], s, len)) continue;
        r.rank++;
        r.before += didr_entry_bytes(kind, didr_path_len(kind, h, a, (uint32_t)(nz[k - base] - j0)), esc[k - base]);
    }
    return r;
}

// ---- the batch's indices

// the list (0 .. 2n - 1) holding absolute id index r: the last L with id_idx[L] <= r
AFC_HD uint32_t didr_list_of(const uint64_t* id_idx, uint32_t n, uint64_t r) {
    uint32_t lo = 0, hi = 2 * n;
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (id_idx[mid] <= r) lo = mid; else hi = mid;
    }
    return lo;
}

// What slot t (an agent, or id t - n) is: its request, kind, index j in its list, component index c, and for an id its absolute index
struct DidrSlot { uint32_t i, kind, j; uint64_t c, r; bool comp; };
AFC_HD DidrSlot didr_slot(const uint64_t* id_idx, const uint32_t* list, const uint8_t* flags, const uint64_t* nz, uint32_t n,
                                              uint32_t m, uint64_t t) {
    DidrSlot s;
    const uint64_t base = id_idx[0];
    if (t < n) {
        s.i = (uint32_t)t; s.kind = DIDR_AGENT; s.j = 0; s.r = 0; s.comp = true;
        s.c = t + nz[id_idx[2 * t] - base];
        return s;
    }
    const uint64_t jj = t - n;
    const uint32_t L = list[jj];
    s.i = L >> 1; s.kind = (L & 1) ? DIDR_SKILL : DIDR_REASONER; s.r = base + jj;
    s.comp = flags[jj] != 0;
    s.j = (uint32_t)(nz[jj] - nz[id_idx[L] - base]);
    s.c = s.comp ? (uint64_t)s.i + 1 + nz[jj] : (uint64_t)n + nz[m] + (jj - nz[jj]);     // the tail: empty ids in order
    return s;
}

// ---- one request's frame

template <class Sink>
AFC_HD void didr_tail(Sink& out, const uint8_t* server, uint64_t server_len, const uint8_t* node, uint64_t node_len, uint32_t nr, uint32_t ns) {
    vci_put_text(out, DIDR_L_SERVER);
    go_json_escape(out, server, server_len);
    vci_put_text(out, DIDR_L_MSG);
    go_json_escape(out, node, node_len);
    vci_put_text(out, DIDR_L_WITH);
    vci_put_int(out, (int64_t)nr);
    vci_put_text(out, DIDR_L_REAS);
    vci_put_int(out, (int64_t)ns);
    vci_put_text(out, DIDR_L_SKILLS);
}

// Where the pieces of a body start, relative to it: the agent's identity, the reasoner map (after its '{'), the skill map, the tail (at
// the skill map's '}')
struct DidrLayout { uint64_t agent, rmap, smap, tail; };
AFC_HD DidrLayout didr_layout(uint64_t agent_bytes, uint64_t rbytes, uint64_t sbytes) {
    DidrLayout L;
    L.agent = DIDR_LEN(DIDR_L_HEAD);
    L.rmap = L.agent + agent_bytes + DIDR_LEN(DIDR_L_RMAP);
    L.smap = L.rmap + rbytes + DIDR_LEN(DIDR_L_SMAP);
    L.tail = L.smap + sbytes;
    return L;
}

}  // namespace afc
