// Execution credentials issued on the device (afc_vc_issue_execution_batch, include/afcrypto.h): what GenerateExecutionVC
// (internal/services/vc_service.go:138-239) computes and stores for one request, written per credential.
//
//   vci_hashdata_one   hashData(marshalDataOrNull(data))        vc_service.go:508-515, 1297-1306
//                      SHA-256 over  "  base64(data)  "  (null for a nil payload), base64url without padding (43 characters).
//                      The base64 text is generated from the payload 48 bytes at a time, straight into the message schedule; it
//                      never exists in memory.  The leading quote shifts every 64-character group by one byte across blocks.
//   vci_doc            createVCDocument + json.Marshal           vc_service.go:374-431, 436-439 (signing form), :201 (stored form)
//                      the constant text of types.VCDocument interleaved with the request's columns, Go-escaped (go_json_escape),
//                      the two digests, durationMs (a Go int) and the optional, truncated errorMessage (:153-160).
//   vci_proof_one      base64.RawURLEncoding of the signature   vc_service.go:465
//
// Shared by the kernels of k_vcissue.cu and the CPU build of the same logic in tests/hostsim.
#pragma once
#include "afc_json.cuh"
#include "afc_sha.cuh"

namespace afc {

enum {
    VCI_COLUMNS = 14,        // vc_id, caller_did, issuance_date, execution_id, workflow_id, session_id, caller_type, agent_node_did,
                             // target_did, function_name, timestamp, status, error_message, proof_created (AFC_ISSUE_COLUMNS)
    VCI_COL_VC_ID = 0, VCI_COL_CALLER_DID = 1, VCI_COL_ERROR = 12, VCI_COL_PROOF_CREATED = 13,
    VCI_HASH_CHARS = 43,     // base64url(SHA-256) without padding
    VCI_PV_CHARS = 86,       // base64url(64-byte signature) without padding
    VCI_ERR_MAX = 500,       // vc_service.go:153-160: longer messages are cut to 500 bytes + "...[truncated]"
};

// What follows each literal of the program
enum : uint8_t {
    VCI_V_NONE = 0x80, VCI_V_HASH_IN, VCI_V_HASH_OUT, VCI_V_DURATION, VCI_V_ERROR, VCI_V_PROOF_VALUE,
    // values below 0x80 are column indices (escaped as Go strings)
};

// The constant text and column map of json.Marshal(types.VCDocument), staged once per block in shared memory.  Pieces
// [0, VCI_COMMON) are the signing and the stored document's common prefix up to "proof":; piece VCI_SIGN_TAIL is the zero-valued
// proof the reference signs over; pieces (VCI_SIGN_TAIL, VCI_PIECES) are the stored proof.  Every literal starts on a word of
// the pool, so it is copied four bytes at a time.
enum { VCI_COMMON = 21, VCI_SIGN_TAIL = 21, VCI_PIECES = 26, VCI_POOL_WORDS = 216 };
struct VciProgram {
    uint32_t pool[VCI_POOL_WORDS];
    uint16_t lit_off[VCI_PIECES], lit_len[VCI_PIECES];
    uint8_t val[VCI_PIECES];
};

// Builds the program (host code); returns the bytes of literal text (0 if the pool is too small, which would be a bug)
static inline uint32_t vci_program_build(VciProgram* P) {
    static const struct { const char* lit; uint8_t val; } pieces[VCI_PIECES] = {
        {"{\"@context\":[\"https://www.w3.org/2018/credentials/v1\",\"https://agentfield.example.com/contexts/execution/v1\"],"
         "\"type\":[\"VerifiableCredential\",\"AgentFieldExecutionCredential\"],\"id\":\"urn:agentfield:vc:", 0},
        {"\",\"issuer\":\"", 1},
        {"\",\"issuanceDate\":\"", 2},
        {"\",\"credentialSubject\":{\"executionId\":\"", 3},
        {"\",\"workflowId\":\"", 4},
        {"\",\"sessionId\":\"", 5},
        {"\",\"caller\":{\"did\":\"", 1},
        {"\",\"type\":\"", 6},
        {"\",\"agentNodeDid\":\"", 7},
        {"\"},\"target\":{\"did\":\"", 8},
        {"\",\"agentNodeDid\":\"", 7},
        {"\",\"functionName\":\"", 9},
        {"\"},\"execution\":{\"inputHash\":\"", VCI_V_HASH_IN},
        {"\",\"outputHash\":\"", VCI_V_HASH_OUT},
        {"\",\"timestamp\":\"", 10},
        {"\",\"durationMs\":", VCI_V_DURATION},
        {",\"status\":\"", 11},
        {"\"", VCI_V_ERROR},
        {"},\"audit\":{\"inputDataHash\":\"", VCI_V_HASH_IN},
        {"\",\"outputDataHash\":\"", VCI_V_HASH_OUT},
        {"\",\"metadata\":{\"agentfield_version\":\"1.0.0\",\"vc_version\":\"1.0\"}}},\"proof\":", VCI_V_NONE},
        {"{\"type\":\"\",\"created\":\"\",\"verificationMethod\":\"\",\"proofPurpose\":\"\",\"proofValue\":\"\"}}", VCI_V_NONE},
        {"{\"type\":\"Ed25519Signature2020\",\"created\":\"", 13},
        {"\",\"verificationMethod\":\"", 1},
        {"#key-1\",\"proofPurpose\":\"assertionMethod\",\"proofValue\":\"", VCI_V_PROOF_VALUE},
        {"\"}}", VCI_V_NONE},
    };
    memset(P, 0, sizeof *P);
    uint8_t* pool = (uint8_t*)P->pool;
    uint32_t at = 0, text = 0;
    for (int k = 0; k < VCI_PIECES; k++) {
        const uint32_t len = (uint32_t)strlen(pieces[k].lit);
        if (at + len > sizeof P->pool) return 0;
        memcpy(pool + at, pieces[k].lit, len);
        P->lit_off[k] = (uint16_t)at; P->lit_len[k] = (uint16_t)len; P->val[k] = pieces[k].val;
        at = (at + len + 3) & ~3u;
        text += len;
    }
    return text;
}

// One request's columns and numbers.  coff: its VCI_COLUMNS + 1 absolute offsets into cols; hashes: its 2 x 43 characters (input,
// output), nullptr without HashSensitiveData (both hashes are then "").
struct VciItem {
    const uint8_t* cols;
    const uint64_t* coff;
    const uint8_t* hashes;
    int64_t duration;
};

template <class Sink>
AFC_HD void vci_put_lit(Sink& out, const uint32_t* pool, uint32_t off, uint32_t len) {
    const uint32_t* t = pool + (off >> 2);
    uint32_t k = 0;
    for (; k + 4 <= len; k += 4) out.put4(t[k >> 2]);
    for (; k < len; k++) out.put((t[k >> 2] >> (8 * (k & 3))) & 0xffu);
}

template <class Sink>
AFC_HD void vci_put_text(Sink& out, const char* s) { for (; *s; ++s) out.put((uint8_t)*s); }

// Go's strconv.AppendInt for an int64: no local array, digits from the most significant
template <class Sink>
AFC_HD void vci_put_int(Sink& out, int64_t v) {
    uint64_t u = (uint64_t)v;
    if (v < 0) { out.put('-'); u = 0 - u; }
    uint64_t p = 1;
    while (u / p >= 10) p *= 10;                  // u <= 2^63 < 10^19: p stays <= 10^18
    for (; p; p /= 10) out.put('0' + (uint32_t)((u / p) % 10));
}

template <class Sink>
AFC_HD void vci_value(Sink& out, uint32_t v, const VciItem& it) {
    if (v < VCI_COLUMNS) { go_json_escape(out, it.cols + it.coff[v], it.coff[v + 1] - it.coff[v]); return; }
    switch (v) {
    case VCI_V_HASH_IN:
    case VCI_V_HASH_OUT:
        if (it.hashes) json_copy_raw(out, it.hashes + (v == VCI_V_HASH_OUT ? VCI_HASH_CHARS : 0), VCI_HASH_CHARS);
        break;
    case VCI_V_DURATION: vci_put_int(out, it.duration); break;
    case VCI_V_ERROR: {                            // omitempty; msg[:500] + "...[truncated]" past 500 bytes (a cut rune stays invalid bytes)
        const uint64_t len = it.coff[VCI_COL_ERROR + 1] - it.coff[VCI_COL_ERROR];
        if (len == 0) break;
        vci_put_text(out, ",\"errorMessage\":\"");
        go_json_escape(out, it.cols + it.coff[VCI_COL_ERROR], len > VCI_ERR_MAX ? (uint64_t)VCI_ERR_MAX : len);
        if (len > VCI_ERR_MAX) vci_put_text(out, "...[truncated]");
        out.put('"');
        break;
    }
    case VCI_V_PROOF_VALUE:                        // placeholder: vci_proof_one writes the characters once the signature exists
        for (uint32_t k = 0; k < VCI_PV_CHARS / 4; k++) out.put4(0x41414141u);
        out.put('A'); out.put('A');
        break;
    default: break;
    }
}

template <class Sink>
AFC_HD void vci_pieces(Sink& out, const VciProgram& P, uint32_t k0, uint32_t k1, const VciItem& it) {
    for (uint32_t k = k0; k < k1; k++) {
        vci_put_lit(out, P.pool, P.lit_off[k], P.lit_len[k]);
        vci_value(out, P.val[k], it);
    }
}

// Both lengths of one credential: the signing message and the stored document
AFC_HD void vci_doc_sizes(const VciProgram& P, const VciItem& it, uint64_t* msg_len, uint64_t* doc_len) {
    ByteCounter c; c.init();
    vci_pieces(c, P, 0, VCI_COMMON, it);
    *msg_len = c.n + P.lit_len[VCI_SIGN_TAIL];
    vci_pieces(c, P, VCI_SIGN_TAIL + 1, VCI_PIECES, it);
    *doc_len = c.n;
}

// Two sinks fed the same bytes: the common prefix goes to the signing message and to the stored document in one walk
struct TeeWriter {
    ByteWriter a, b;
    AFC_HDM void put(uint32_t x) { a.put(x); b.put(x); }
    AFC_HDM void put4(uint32_t x) { a.put4(x); b.put4(x); }
};

// Writes the signing message at msg and the stored document (proofValue still a placeholder) at doc
AFC_HD void vci_doc_fill(const VciProgram& P, const VciItem& it, uint8_t* msg, uint8_t* doc) {
    TeeWriter t; t.a.init(msg); t.b.init(doc);
    vci_pieces(t, P, 0, VCI_COMMON, it);
    vci_pieces(t.a, P, VCI_SIGN_TAIL, VCI_SIGN_TAIL + 1, it);
    t.a.finish();
    vci_pieces(t.b, P, VCI_SIGN_TAIL + 1, VCI_PIECES, it);
    t.b.finish();
}

// ---- base64 four characters at a time: x = four 6-bit values, one per byte (big-endian), mapped with byte-wise compares
AFC_HD uint32_t b64_chars4(uint32_t x, bool url) {
    const uint32_t L = 0x01010101u;
    const uint32_t m25 = ((x + 0x66666666u) >> 7) & L, m51 = ((x + 0x4c4c4c4cu) >> 7) & L;
    const uint32_t m61 = ((x + 0x42424242u) >> 7) & L, m62 = ((x + 0x41414141u) >> 7) & L;
    // std: 62 -> '+', 63 -> '/';  url: 62 -> '-', 63 -> '_'   (every byte of every intermediate stays in 0..255)
    return url ? x + 0x41414141u + 6 * m25 + 49 * m62 - 75 * m51 - 13 * m61
               : x + 0x41414141u + 6 * m25 + 3 * m62 - 75 * m51 - 15 * m61;
}
// 24 bits -> 4 characters, the first in the most significant byte
AFC_HD uint32_t b64_word(uint32_t v, bool url) {
    const uint32_t x = ((v >> 18) & 63u) << 24 | ((v >> 12) & 63u) << 16 | ((v >> 6) & 63u) << 8 | (v & 63u);
    return b64_chars4(x, url);
}
// bits [24 t, 24 t + 24) of the big-endian bit string held in W[] (t a compile-time constant at every call site)
AFC_HD uint32_t triple_at(const uint32_t* W, int nw, int t) {
    const int q = (24 * t) >> 5, s = (24 * t) & 31;
    const uint64_t pair = ((uint64_t)W[q] << 32) | (q + 1 < nw ? W[q + 1] : 0u);
    return (uint32_t)(pair >> (40 - s)) & 0xffffffu;
}

// 48 payload bytes (12 big-endian words) -> 64 base64 characters (16 big-endian words)
AFC_HD void vci_b64_group(uint32_t C[16], const uint32_t W[12]) {
#pragma unroll
    for (int t = 0; t < 16; t++) C[t] = b64_word(triple_at(W, 12, t), false);
}

// SHA-256 of  "  StdEncoding(p[0..len))  "  or of  null; st: the digest words
AFC_HD void vci_hashdata_digest(uint32_t st[8], const uint8_t* p, uint64_t len, bool nil) {
    sha256_init(st);
    uint32_t w[16];
    if (nil) {
#pragma unroll
        for (int i = 0; i < 16; i++) w[i] = 0;
        w[0] = 0x6e756c6cu; w[1] = 0x80000000u; w[15] = 32;
        sha256_compress(st, w);
        return;
    }
    const uint64_t nfull = len / 48, bits = 8 * (2 + 4 * ((len + 2) / 3));
    uint32_t carry = '"';                          // the byte that ends the previous block's characters
    const bool al = (((uintptr_t)p) & 15) == 0;
    MsgReader rd; rd.init(p, al ? 0 : 48 * nfull);
    for (uint64_t b = 0; b < nfull; b++) {
        uint32_t W[12], C[16];
        if (al) {
#pragma unroll
            for (int q = 0; q < 3; q++) {
                const word4 v = ld_u128(p + 48 * b + 16 * q);
                W[4 * q] = bswap32(v.x); W[4 * q + 1] = bswap32(v.y); W[4 * q + 2] = bswap32(v.z); W[4 * q + 3] = bswap32(v.w);
            }
        } else {
#pragma unroll
            for (int q = 0; q < 12; q++) W[q] = bswap32(rd.next());
        }
        vci_b64_group(C, W);
        w[0] = (carry << 24) | (C[0] >> 8);
#pragma unroll
        for (int j = 1; j < 16; j++) w[j] = (C[j - 1] << 24) | (C[j] >> 8);
        carry = C[15] & 0xffu;
        sha256_compress(st, w);
    }
    // the last r < 48 bytes: T = ceil(r / 3) character words, '=' padding, the closing quote, 0x80, the length
    const uint32_t r = (uint32_t)(len - 48 * nfull), T = (r + 2) / 3;
    uint32_t W[12], D[17];
    {
        MsgReader tr; tr.init(p + 48 * nfull, r);
#pragma unroll
        for (int q = 0; q < 12; q++) {
            const uint32_t x = tr.next();
            const uint32_t k = r > 4u * q ? r - 4u * q : 0u;
            W[q] = bswap32(k >= 4 ? x : (x & ((1u << (8 * k)) - 1u)));
        }
    }
    const uint32_t pad = r % 3 == 1 ? 0x3d3du : r % 3 == 2 ? 0x3du : 0u;
    const uint32_t keep = r % 3 == 1 ? 0xffff0000u : r % 3 == 2 ? 0xffffff00u : 0xffffffffu;
#pragma unroll
    for (int t = 0; t < 17; t++) {
        uint32_t c = t < 16 ? b64_word(triple_at(W, 12, t), false) : 0u;
        if ((uint32_t)t + 1 == T) c = (c & keep) | pad;
        D[t] = (uint32_t)t < T ? c : (uint32_t)t == T ? 0x22800000u : 0u;
    }
    w[0] = (carry << 24) | (D[0] >> 8);
#pragma unroll
    for (int j = 1; j < 16; j++) w[j] = (D[j - 1] << 24) | (D[j] >> 8);
    if (T <= 13) {
        w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits;
        sha256_compress(st, w);
        return;
    }
    sha256_compress(st, w);
    w[0] = (D[15] << 24) | (D[16] >> 8);
#pragma unroll
    for (int j = 1; j < 14; j++) w[j] = 0;
    w[14] = (uint32_t)(bits >> 32); w[15] = (uint32_t)bits;
    sha256_compress(st, w);
}

// A big-endian word of 4 characters to 4 bytes at an arbitrary address
AFC_HD void vci_store_chars(uint8_t* o, uint32_t c, uint32_t n) {
    for (uint32_t k = 0; k < n; k++) o[k] = (uint8_t)(c >> (24 - 8 * k));
}

// hashData of one payload: 43 base64url characters at out
AFC_HD void vci_hashdata_one(const uint8_t* p, uint64_t len, bool nil, uint8_t* out) {
    uint32_t st[8];
    vci_hashdata_digest(st, p, len, nil);
#pragma unroll
    for (int t = 0; t < 10; t++) vci_store_chars(out + 4 * t, b64_word(triple_at(st, 8, t), true), 4);
    vci_store_chars(out + 40, b64_word((st[7] & 0xffffu) << 8, true), 3);
}

// base64url of a 64-byte signature (16 little-endian-loaded words): 86 characters, written to each of the two outputs
AFC_HD void vci_proof_one(const uint32_t sig_le[16], uint8_t* out_a, uint8_t* out_b) {
    uint32_t W[16];
#pragma unroll
    for (int i = 0; i < 16; i++) W[i] = bswap32(sig_le[i]);
#pragma unroll
    for (int t = 0; t < 21; t++) {
        const uint32_t c = b64_word(triple_at(W, 16, t), true);
        vci_store_chars(out_a + 4 * t, c, 4);
        vci_store_chars(out_b + 4 * t, c, 4);
    }
    const uint32_t c = b64_word((W[15] & 0xffu) << 16, true);
    vci_store_chars(out_a + 84, c, 2);
    vci_store_chars(out_b + 84, c, 2);
}

}  // namespace afc
