// SHA-256 / SHA-512 / HMAC-SHA256 per-message device routines (FIPS 180-4, RFC 2104).
//
// Replaces, per message, what the reference reaches through Go's crypto/sha256, crypto/sha512 and
// crypto/hmac:  vc_service.go:513 (hashData), did_service.go:517 (derivePrivateKey),
// payload_store.go:69 (payload digest), webhook_dispatcher.go:470-474 (generateWebhookSignature), and
// the SHA-512 passes inside ed25519.Sign / ed25519.Verify (vc_service.go:463,504).
//
// sm_90a notes: 32-bit rotates are single funnel shifts (SHF.R.W), Ch/Maj/xor3 are single LOP3s; the
// round constants live in __constant__ memory and, with the rounds fully unrolled, become immediate
// constant-bank operands (c[bank][off]) — no load instructions, no shared-memory traffic.
#pragma once
#include "afc_common.cuh"

#if !defined(AFC_HOSTSIM)
#define AFC_CONST_DECL static __device__ __constant__
#endif
#include "afc_consts.inc"

namespace afc {

// ---------------------------------------------------------------------------------- SHA-256
AFC_HD uint32_t ch32(uint32_t x, uint32_t y, uint32_t z) { return (x & y) ^ (~x & z); }
AFC_HD uint32_t maj32(uint32_t x, uint32_t y, uint32_t z) { return (x & y) ^ (x & z) ^ (y & z); }

// Out-of-line on the device: HMAC alone has five compression call sites; inlining each (~1.6k instructions) would
// put >100 KB of SASS in one kernel and stall every warp on instruction fetch.
#if defined(AFC_HOSTSIM)
#define AFC_OUTLINE static inline
#else
#define AFC_OUTLINE static __device__ __noinline__
#endif

// ALU-pipe relief: the SHA-256 kernels are bound by the ALU pipe (shifts, LOP3, IADD3) while the FMA pipe
// idles.  A two-input add written as a * ONE + b with ONE read from the constant bank is emitted as an IMAD and executes on
// the FMA pipe instead (the compiler cannot fold a __constant__ operand).  AFC_SHA_IMAD_ADDS selects how many adds move.
#ifndef AFC_SHA_IMAD_ADDS
#define AFC_SHA_IMAD_ADDS 1
#endif
#if defined(AFC_HOSTSIM)
#define AFC_FADD(a, b) ((a) + (b))
#else
static __device__ __constant__ uint32_t AFC_ONE = 1u;
#if AFC_SHA_IMAD_ADDS
#define AFC_FADD(a, b) ((a) * AFC_ONE + (b))
#else
#define AFC_FADD(a, b) ((a) + (b))
#endif
#endif

// One compression: st += F(st, w[0..15]).  Fully unrolled (round constants become constant-bank immediates, the
// schedule window stays in registers); ONE out-of-line copy per kernel, state and block passed in registers.
struct sha256_io { uint32_t st[8]; uint32_t w[16]; };
struct sha256_st { uint32_t st[8]; };
AFC_OUTLINE sha256_st sha256_compress_regs(sha256_io x) {
    uint32_t a = x.st[0], b = x.st[1], c = x.st[2], d = x.st[3], e = x.st[4], f = x.st[5], g = x.st[6], h = x.st[7];
#pragma unroll
    for (int i = 0; i < 64; i++) {
        if (i >= 16) {
            uint32_t w15 = x.w[(i - 15) & 15], w2 = x.w[(i - 2) & 15];
            uint32_t s0 = rotr32(w15, 7) ^ rotr32(w15, 18) ^ (w15 >> 3);
            uint32_t s1 = rotr32(w2, 17) ^ rotr32(w2, 19) ^ (w2 >> 10);
            x.w[i & 15] = AFC_FADD(AFC_FADD(x.w[i & 15], x.w[(i - 7) & 15]), s0 + s1);
        }
        uint32_t hk = AFC_FADD(AFC_FADD(h, x.w[i & 15]), AFC_K256[i]);           // off the critical path: FMA pipe
#if AFC_SHA_IMAD_ADDS >= 2
        uint32_t t1 = AFC_FADD(AFC_FADD(hk, rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25)), ch32(e, f, g));
        uint32_t t2 = AFC_FADD(rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22), maj32(a, b, c));
        h = g; g = f; f = e; e = AFC_FADD(d, t1); d = c; c = b; b = a; a = AFC_FADD(t1, t2);
#else
        uint32_t t1 = hk + (rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25)) + ch32(e, f, g);
        uint32_t t2 = (rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22)) + maj32(a, b, c);
        h = g; g = f; f = e; e = AFC_FADD(d, t1); d = c; c = b; b = a; a = t1 + t2;
#endif
    }
    sha256_st r;
    r.st[0] = x.st[0] + a; r.st[1] = x.st[1] + b; r.st[2] = x.st[2] + c; r.st[3] = x.st[3] + d;
    r.st[4] = x.st[4] + e; r.st[5] = x.st[5] + f; r.st[6] = x.st[6] + g; r.st[7] = x.st[7] + h;
    return r;
}
AFC_HD void sha256_compress(uint32_t* st, uint32_t* w) {
    sha256_io x;
#pragma unroll
    for (int i = 0; i < 8; i++) x.st[i] = st[i];
#pragma unroll
    for (int i = 0; i < 16; i++) x.w[i] = w[i];
    sha256_st r = sha256_compress_regs(x);
#pragma unroll
    for (int i = 0; i < 8; i++) st[i] = r.st[i];
}

AFC_HD void sha256_init(uint32_t st[8]) {
#pragma unroll
    for (int i = 0; i < 8; i++) st[i] = AFC_H256[i];
}

// Absorb `len` message bytes after `prior` bytes have already been compressed into st (prior % 64 == 0),
// then pad and finish.  st holds the digest words (big-endian order) on return.
// Whole 64-byte blocks of a 16-byte-aligned message take the lean path: four 128-bit loads + 16 byte swaps, no per-word
// bounds / padding logic (these kernels are ALU-bound: every instruction saved in block loading is throughput).
AFC_HD void sha256_finish_stream(uint32_t st[8], const uint8_t* msg, uint64_t len, uint64_t prior) {
    uint64_t total = prior + len;
    if ((((uintptr_t)msg) & 15) == 0) {
        uint64_t nfull = len >> 6;
        for (uint64_t blk = 0; blk < nfull; blk++) {
            uint32_t w[16];
#pragma unroll
            for (int q = 0; q < 4; q++) {
                word4 v = ld_u128(msg + 16 * q);
                w[4 * q] = bswap32(v.x); w[4 * q + 1] = bswap32(v.y); w[4 * q + 2] = bswap32(v.z); w[4 * q + 3] = bswap32(v.w);
            }
            sha256_compress(st, w);
            msg += 64;
        }
        len &= 63;
    }
    PadStream ps; ps.init(msg, len);
    uint64_t nblk = (len + 9 + 63) / 64;
    for (uint64_t blk = 0; blk < nblk; blk++) {
        uint32_t w[16];
#pragma unroll
        for (int i = 0; i < 16; i++) w[i] = ps.next_be();
        if (blk == nblk - 1) { w[14] = (uint32_t)((total * 8) >> 32); w[15] = (uint32_t)(total * 8); }
        sha256_compress(st, w);
    }
}

// Absorb whole blocks only (len % 64 == 0), no padding: the middle of a stream (FilePayloadStore.SaveFromReader feeds the hash
// 32 KiB at a time, payload_store.go:69-94,154).
AFC_HD void sha256_absorb_blocks(uint32_t st[8], const uint8_t* msg, uint64_t len) {
    uint64_t nfull = len >> 6;
    if ((((uintptr_t)msg) & 15) == 0) {
        for (uint64_t blk = 0; blk < nfull; blk++) {
            uint32_t w[16];
#pragma unroll
            for (int q = 0; q < 4; q++) {
                word4 v = ld_u128(msg + 16 * q);
                w[4 * q] = bswap32(v.x); w[4 * q + 1] = bswap32(v.y); w[4 * q + 2] = bswap32(v.z); w[4 * q + 3] = bswap32(v.w);
            }
            sha256_compress(st, w);
            msg += 64;
        }
        return;
    }
    PadStream ps; ps.init(msg, nfull << 6);
    for (uint64_t blk = 0; blk < nfull; blk++) {
        uint32_t w[16];
#pragma unroll
        for (int i = 0; i < 16; i++) w[i] = ps.next_be();
        sha256_compress(st, w);
    }
}
// Streaming state between calls, laid out exactly like Go's crypto/sha256 (*digest).MarshalBinary: "sha\x03" || h[0..7] big-endian ||
// 64-byte block buffer || total length big-endian = 108 bytes.  States handed across this boundary always sit on a block
// boundary (length % 64 == 0), so the buffer is all zeros; a Go caller can UnmarshalBinary such a state and continue, and back.
static constexpr int SHA256_STATE_BYTES = 108;
AFC_HD int sha256_state_load(uint32_t st[8], uint64_t* total, const uint8_t* s) {
    if (s[0] != 's' || s[1] != 'h' || s[2] != 'a' || s[3] != 3) return 0;
#pragma unroll
    for (int i = 0; i < 8; i++) st[i] = ((uint32_t)s[4 + 4 * i] << 24) | ((uint32_t)s[5 + 4 * i] << 16) | ((uint32_t)s[6 + 4 * i] << 8) | s[7 + 4 * i];
    uint64_t t = 0;
    for (int i = 0; i < 8; i++) t = (t << 8) | s[100 + i];
    *total = t;
    return (t & 63) == 0;
}
AFC_HD void sha256_state_store(uint8_t* s, const uint32_t st[8], uint64_t total) {
    s[0] = 's'; s[1] = 'h'; s[2] = 'a'; s[3] = 3;
#pragma unroll
    for (int i = 0; i < 8; i++) store_be32(s + 4 + 4 * i, st[i]);
    for (int i = 0; i < 64; i++) s[36 + i] = 0;
    for (int i = 0; i < 8; i++) s[100 + i] = (uint8_t)(total >> (56 - 8 * i));
}

AFC_HD void sha256_msg(uint32_t st[8], const uint8_t* msg, uint64_t len) {
    sha256_init(st);
    sha256_finish_stream(st, msg, len, 0);
}

// SHA-256 of a short in-register message of nwords*4 bytes (nwords <= 13 -> single block).
template <int NWORDS>
AFC_HD void sha256_words(uint32_t st[8], const uint32_t* be_words) {
    static_assert(NWORDS <= 13, "single block only");
    uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = (i < NWORDS) ? be_words[i] : 0u;
    w[NWORDS] = 0x80000000u;
    w[15] = NWORDS * 32;
    sha256_init(st);
    sha256_compress(st, w);
}

// RFC 6962 interior node: SHA-256(0x01 || left || right), 65 bytes -> 2 blocks.  l, r: big-endian words.
AFC_HD void sha256_merkle_node(uint32_t out[8], const uint32_t l[8], const uint32_t r[8]) {
    uint32_t w[16];
    w[0] = 0x01000000u | (l[0] >> 8);
#pragma unroll
    for (int i = 1; i < 8; i++) w[i] = (l[i - 1] << 24) | (l[i] >> 8);
    w[8] = (l[7] << 24) | (r[0] >> 8);
#pragma unroll
    for (int i = 1; i < 8; i++) w[8 + i] = (r[i - 1] << 24) | (r[i] >> 8);
    sha256_init(out);
    sha256_compress(out, w);
    w[0] = (r[7] << 24) | 0x00800000u;
#pragma unroll
    for (int i = 1; i < 15; i++) w[i] = 0;
    w[15] = 65 * 8;
    sha256_compress(out, w);
}

// RFC 6962 leaf: SHA-256(0x00 || leaf).  One prefix byte, then the message stream — handled by
// feeding the stream shifted by one byte.
AFC_HD void sha256_merkle_leaf(uint32_t st[8], const uint8_t* leaf, uint64_t len) {
    PadStream ps; ps.init(leaf, len);
    uint64_t total = len + 1;
    uint64_t nblk = (total + 9 + 63) / 64;
    uint32_t carry = 0;                 // the 0x00 domain-separation byte, in the top 8 bits position
    sha256_init(st);
    for (uint64_t blk = 0; blk < nblk; blk++) {
        uint32_t w[16];
#pragma unroll
        for (int i = 0; i < 16; i++) {
            uint32_t x = ps.next_be();
            w[i] = (carry << 24) | (x >> 8);
            carry = x & 0xffu;
        }
        if (blk == nblk - 1) { w[14] = (uint32_t)((total * 8) >> 32); w[15] = (uint32_t)(total * 8); }
        sha256_compress(st, w);
    }
}

// HMAC-SHA256 (RFC 2104) exactly as Go's hmac.New(sha256.New, key): keys longer than the 64-byte block
// are hashed first; shorter keys are zero-padded.
AFC_HD void hmac_sha256_msg(uint32_t out[8], const uint8_t* key, uint32_t klen, const uint8_t* msg, uint64_t len) {
    uint32_t k0[16];
    if (klen > 64) {
        uint32_t kd[8];
        sha256_msg(kd, key, klen);
#pragma unroll
        for (int i = 0; i < 16; i++) k0[i] = (i < 8) ? kd[i] : 0u;
    } else {
        MsgReader rd; rd.init(key, klen);
        uint32_t rem = klen;            // zero padding only: no 0x80 marker
#pragma unroll
        for (int i = 0; i < 16; i++) {
            uint32_t w = 0;
            if (rem >= 4) { w = rd.next(); rem -= 4; }
            else if (rem) { w = rd.next() & ((1u << (8 * rem)) - 1u); rem = 0; }
            k0[i] = bswap32(w);
        }
    }
    uint32_t st[8], w[16];
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = k0[i] ^ 0x36363636u;
    sha256_init(st);
    sha256_compress(st, w);
    sha256_finish_stream(st, msg, len, 64);
    // outer: H(opad-block || inner digest)
    uint32_t inner[8];
#pragma unroll
    for (int i = 0; i < 8; i++) inner[i] = st[i];
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = k0[i] ^ 0x5c5c5c5cu;
    sha256_init(out);
    sha256_compress(out, w);
#pragma unroll
    for (int i = 0; i < 8; i++) w[i] = inner[i];
    w[8] = 0x80000000u;
#pragma unroll
    for (int i = 9; i < 15; i++) w[i] = 0;
    w[15] = (64 + 32) * 8;
    sha256_compress(out, w);
}

AFC_HD void store_digest256(uint8_t* out, const uint32_t st[8]) {
#if AFC_DEVICE_CODE
    if ((((uintptr_t)out) & 15) == 0) {
        uint4 a = make_uint4(bswap32(st[0]), bswap32(st[1]), bswap32(st[2]), bswap32(st[3]));
        uint4 b = make_uint4(bswap32(st[4]), bswap32(st[5]), bswap32(st[6]), bswap32(st[7]));
        ((uint4*)out)[0] = a; ((uint4*)out)[1] = b;
        return;
    }
#endif
#pragma unroll
    for (int i = 0; i < 8; i++) store_be32(out + 4 * i, st[i]);
}

// ---------------------------------------------------------------------------------- SHA-512
// (Moving the 64-bit adds to the FMA pipe the way AFC_FADD does for SHA-256 does not work here: ptxas splits
// mad.wide.u32 d, a, ONE, c64 into IMAD.WIDE + IADD3 + IMAD.X, so the ALU pipe keeps its add and the FMA pipe gains two.
// Rotates as multiplications by 2^(32-n) from the constant bank — two IMAD + two IMAD.HI per 64-bit rotate instead of two SHF —
// do leave the ALU pipe, but cost more than they free: each further rotate moved made k_ed_hram + verify slower.)
AFC_HD void sha512_round(uint64_t& a, uint64_t& b, uint64_t& c, uint64_t& d, uint64_t& e, uint64_t& f, uint64_t& g, uint64_t& h,
                         uint64_t kw) {
    const uint64_t t1 = h + (rotr64(e, 14) ^ rotr64(e, 18) ^ rotr64(e, 41)) + ((e & f) ^ (~e & g)) + kw;
    const uint64_t t2 = (rotr64(a, 28) ^ rotr64(a, 34) ^ rotr64(a, 39)) + ((a & b) ^ (a & c) ^ (b & c));
    h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
}

// One compression: returns st + F(st, w[0..15]).  State and block are passed by value in registers: through pointers both live in
// local memory, and as ONE 192-byte aggregate the calling convention passes them on the stack.  The first 16 rounds, which need no
// schedule, are peeled; the other 64 stay a rolled loop of 16 so that the ONE out-of-line copy per kernel stays small in the
// instruction cache.
struct sha512_st { uint64_t st[8]; };
struct sha512_blk { uint64_t w[16]; };
AFC_OUTLINE sha512_st sha512_compress_regs(sha512_st x, sha512_blk blk) {
    uint64_t a = x.st[0], b = x.st[1], c = x.st[2], d = x.st[3], e = x.st[4], f = x.st[5], g = x.st[6], h = x.st[7];
    uint64_t w[16];
#pragma unroll
    for (int j = 0; j < 16; j++) {
        w[j] = blk.w[j];
        sha512_round(a, b, c, d, e, f, g, h, AFC_K512[j] + w[j]);
    }
#pragma unroll 1
    for (int r = 16; r < 80; r += 16) {
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const uint64_t w15 = w[(j + 1) & 15], w2 = w[(j + 14) & 15];
            const uint64_t s0 = rotr64(w15, 1) ^ rotr64(w15, 8) ^ (w15 >> 7);
            const uint64_t s1 = rotr64(w2, 19) ^ rotr64(w2, 61) ^ (w2 >> 6);
            w[j] = w[j] + s0 + w[(j + 9) & 15] + s1;
            sha512_round(a, b, c, d, e, f, g, h, AFC_K512[r + j] + w[j]);
        }
    }
    sha512_st o;
    o.st[0] = x.st[0] + a; o.st[1] = x.st[1] + b; o.st[2] = x.st[2] + c; o.st[3] = x.st[3] + d;
    o.st[4] = x.st[4] + e; o.st[5] = x.st[5] + f; o.st[6] = x.st[6] + g; o.st[7] = x.st[7] + h;
    return o;
}
// 128 message bytes from 16-byte-aligned p as big-endian words
AFC_HD void sha512_load_block(uint64_t w[16], const uint8_t* p) {
#pragma unroll
    for (int q = 0; q < 8; q++) {
        const word4 v = ld_u128(p + 16 * q);
        w[2 * q] = ((uint64_t)bswap32(v.x) << 32) | bswap32(v.y);
        w[2 * q + 1] = ((uint64_t)bswap32(v.z) << 32) | bswap32(v.w);
    }
}

// The last len < 128 bytes of a message at 16-byte-aligned p, followed by 0x80 and zeros, as big-endian words.  Only 16-byte
// loads that hold at least one message byte are issued; the bytes they bring from past the end are masked off.  The caller adds
// the bit length: into w[15] when len < 112, otherwise into a block of its own.
AFC_HD void sha512_tail_block(uint64_t w[16], const uint8_t* p, uint32_t len) {
#pragma unroll
    for (int q = 0; q < 8; q++) {
        word4 v = {0u, 0u, 0u, 0u};
        if (16u * q < len) v = ld_u128(p + 16 * q);
        w[2 * q] = ((uint64_t)bswap32(v.x) << 32) | bswap32(v.y);
        w[2 * q + 1] = ((uint64_t)bswap32(v.z) << 32) | bswap32(v.w);
    }
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const int rem = (int)len - 8 * i;                      // message bytes in word i, if in 0..7
        if (rem <= 0) w[i] = rem == 0 ? 0x8000000000000000ull : 0ull;
        else if (rem < 8) w[i] = (w[i] & (~0ull << (64 - 8 * rem))) | (0x80ull << (56 - 8 * rem));
    }
}

// Bytes k..k+3 (k % 4 == 0) of msg followed by 0x80 and zeros, as a big-endian word.  Stateless, so nothing but (msg, len)
// stays live across a compression; only 4-byte loads that hold at least one message byte are issued.
AFC_HD uint32_t sha512_padded_word(const uint8_t* msg, uint64_t len, int64_t k) {
    const int64_t r = (int64_t)len - k;                // message bytes from k on
    if (r < 0) return 0u;
    if (r == 0) return 0x80000000u;
    const uintptr_t a = (uintptr_t)msg + (uint64_t)k;
    const uint32_t* p = (const uint32_t*)(a & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)(a & 3) * 8;
    const uint32_t lo = ld_u32(p), hi = (sh && (uintptr_t)(p + 1) < a + (uint64_t)r) ? ld_u32(p + 1) : 0u;
    const uint32_t v = bswap32(funnel_r(lo, hi, sh));
    return r >= 4 ? v : (v & (0xffffffffu << (32 - 8 * r))) | (0x80000000u >> (8 * r));
}

// SHA-512( prefix (PW 32-bit words, given as LITTLE-endian-loaded words of the byte string) || msg ).
// PW must be a multiple of 4 and <= 24.  Digest returned as 64 bytes little-endian-loaded into 16 u32 (i.e. the
// digest byte string viewed as LE words — the form the scalar reduction wants).
template <int PW>
AFC_HD void sha512_prefixed(uint32_t digest_le[16], const uint32_t* prefix_le, const uint8_t* msg, uint64_t len) {
    static_assert(PW % 4 == 0 && PW <= 24, "prefix must be whole 16-byte groups and leave room in block 0");
    sha512_st x;
    sha512_blk blk;
#pragma unroll
    for (int i = 0; i < 8; i++) x.st[i] = AFC_H512[i];
    const uint64_t total = (uint64_t)PW * 4 + len;
    constexpr int M0 = 128 - 4 * PW;                   // message bytes that share block 0 with the prefix
    if ((((uintptr_t)msg) & 15) == 0 && len >= (uint64_t)M0) {
        // lean path: block 0 = prefix || msg[0:M0], then whole 128-byte blocks, then the padded tail, all with 128-bit loads
#pragma unroll
        for (int i = 0; i < PW / 2; i++) blk.w[i] = ((uint64_t)bswap32(prefix_le[2 * i]) << 32) | bswap32(prefix_le[2 * i + 1]);
#pragma unroll
        for (int q = 0; q < M0 / 16; q++) {
            const word4 v = ld_u128(msg + 16 * q);
            blk.w[PW / 2 + 2 * q] = ((uint64_t)bswap32(v.x) << 32) | bswap32(v.y);
            blk.w[PW / 2 + 2 * q + 1] = ((uint64_t)bswap32(v.z) << 32) | bswap32(v.w);
        }
        x = sha512_compress_regs(x, blk);
        msg += M0; len -= M0;
        const uint64_t nfull = len >> 7;
        for (uint64_t i = 0; i < nfull; i++) {
            sha512_load_block(blk.w, msg);
            x = sha512_compress_regs(x, blk);
            msg += 128;
        }
        const uint32_t tail = (uint32_t)(len & 127);
        sha512_tail_block(blk.w, msg, tail);
        if (tail < 112) blk.w[15] = total * 8;
        x = sha512_compress_regs(x, blk);
        if (tail >= 112) {
#pragma unroll
            for (int i = 0; i < 15; i++) blk.w[i] = 0;
            blk.w[15] = total * 8;
            x = sha512_compress_regs(x, blk);
        }
    } else {
        // general path (unaligned or short messages): word by word, padded in registers
        const uint32_t nblk = (uint32_t)((total + 17 + 127) / 128);
#pragma unroll
        for (int i = 0; i < 16; i++) {
            if (2 * i < PW) blk.w[i] = ((uint64_t)bswap32(prefix_le[2 * i]) << 32) | bswap32(prefix_le[2 * i + 1]);
            else blk.w[i] = ((uint64_t)sha512_padded_word(msg, len, 8 * i - 4 * PW) << 32) | sha512_padded_word(msg, len, 8 * i + 4 - 4 * PW);
        }
        for (uint32_t bi = 0; bi < nblk; bi++) {
            if (bi > 0) {
                const int64_t k0 = 128 * (int64_t)bi - 4 * PW;
#pragma unroll
                for (int i = 0; i < 16; i++)
                    blk.w[i] = ((uint64_t)sha512_padded_word(msg, len, k0 + 8 * i) << 32) | sha512_padded_word(msg, len, k0 + 8 * i + 4);
            }
            if (bi == nblk - 1) { blk.w[14] = 0; blk.w[15] = total * 8; }
            x = sha512_compress_regs(x, blk);
        }
    }
#pragma unroll
    for (int i = 0; i < 8; i++) {
        digest_le[2 * i] = bswap32((uint32_t)(x.st[i] >> 32));
        digest_le[2 * i + 1] = bswap32((uint32_t)x.st[i]);
    }
}

}  // namespace afc
