// afcrypto-b200 — common device/host macros.
//
// Every per-credential routine (hash one message, verify one signature, ...) is written as a plain
// inline function marked AFC_HD so that the SAME source is (a) inlined into the sm_90a kernels and
// (b) compilable by g++ alone (-DAFC_HOSTSIM) into tests/hostsim — a CPU build of the kernel logic
// used ONLY by the no-GPU unit tests to check the arithmetic before spending GPU time.  The product
// library (libafcrypto.so) never contains or calls a CPU implementation: see afcrypto.cu.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#if defined(AFC_HOSTSIM)
#define AFC_HD static inline
#define AFC_HDM inline
#define AFC_HHD static inline
#define AFC_DEVICE_CODE 0
#else
#include <cuda_runtime.h>
#define AFC_HD __device__ __forceinline__
#define AFC_HDM __device__ __forceinline__
#define AFC_HHD __host__ __device__ __forceinline__     // also called by the launch code on the host (table geometry)
#if defined(__CUDA_ARCH__)
#define AFC_DEVICE_CODE 1
#else
#define AFC_DEVICE_CODE 0
#endif
#endif

namespace afc {

AFC_HD uint32_t rotr32(uint32_t x, int n) {
#if AFC_DEVICE_CODE
    return __funnelshift_r(x, x, n);            // one SHF.R.W
#else
    return (x >> n) | (x << ((32 - n) & 31));
#endif
}
// n is a compile-time constant at every call site.  On the device a 64-bit rotate is exactly two funnel shifts over the
// register pair; written as shifts and an OR, nvcc lowers it to three shifts plus LOP3 merges (SHA-512: 76 instead of
// ~45 instructions per round).
AFC_HD uint64_t rotr64(uint64_t x, int n) {
#if AFC_DEVICE_CODE
    const uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    uint32_t rl, rh;
    if (n == 32) { rl = hi; rh = lo; }
    else if (n < 32) { rl = __funnelshift_r(lo, hi, n); rh = __funnelshift_r(hi, lo, n); }
    else { rl = __funnelshift_r(hi, lo, n - 32); rh = __funnelshift_r(lo, hi, n - 32); }
    return ((uint64_t)rh << 32) | rl;
#else
    return (x >> n) | (x << ((64 - n) & 63));
#endif
}

AFC_HD uint32_t bswap32(uint32_t x) {
#if AFC_DEVICE_CODE
    return __byte_perm(x, 0, 0x0123);           // one PRMT
#else
    return (x >> 24) | ((x >> 8) & 0xff00u) | ((x << 8) & 0xff0000u) | (x << 24);
#endif
}
// bytes [sh/8 .. sh/8+4) of the 8-byte little-endian pair (lo, hi); sh in {0,8,16,24}
AFC_HD uint32_t funnel_r(uint32_t lo, uint32_t hi, uint32_t sh) {
#if AFC_DEVICE_CODE
    return __funnelshift_r(lo, hi, sh);
#else
    return sh ? (lo >> sh) | (hi << (32 - sh)) : lo;
#endif
}
AFC_HD uint32_t ld_u32(const uint32_t* p) {
#if AFC_DEVICE_CODE
    return __ldg(p);                            // read-only path (LDG.E.CONSTANT)
#else
    return *p;
#endif
}

// Sequential reader of an arbitrarily aligned byte string in global memory, 4 bytes at a time, using
// only 4-byte-aligned loads that contain at least one byte of the string (never reads a word lying
// wholly outside [p, p+len)).
struct MsgReader {
    const uint32_t* w;      // next aligned word to fetch
    const uint32_t* wend;   // first aligned word wholly past the end
    uint32_t cur, sh;
    AFC_HDM void init(const uint8_t* p, uint64_t len) {
        uintptr_t a = (uintptr_t)p;
        w = (const uint32_t*)(a & ~(uintptr_t)3);
        wend = (const uint32_t*)((a + len + 3) & ~(uintptr_t)3);
        sh = (uint32_t)(a & 3) * 8;
        cur = (w < wend) ? ld_u32(w) : 0u;
        ++w;
    }
    // next 4 bytes as a little-endian word (bytes past the end read as whatever shares the aligned word /
    // zero; the caller masks by the remaining length)
    AFC_HDM uint32_t next() {
        uint32_t nxt = (w < wend) ? ld_u32(w) : 0u;
        ++w;
        uint32_t r = funnel_r(cur, nxt, sh);
        cur = nxt;
        return r;
    }
};

// Merkle–Damgård padded stream: yields the message followed by 0x80, zeros; the caller patches the
// big-endian bit length into the tail of the final block.
struct PadStream {
    MsgReader rd;
    int64_t rem;        // message bytes not yet emitted
    bool padded;
    AFC_HDM void init(const uint8_t* p, uint64_t len) { rd.init(p, len); rem = (int64_t)len; padded = false; }
    // next 4 bytes, as a BIG-endian word (SHA message-schedule order)
    AFC_HDM uint32_t next_be() {
        uint32_t w;
        if (rem >= 4) {
            w = rd.next(); rem -= 4;
        } else if (!padded) {
            uint32_t r = (uint32_t)rem;
            w = r ? (rd.next() & ((1u << (8 * r)) - 1u)) : 0u;
            w |= 0x80u << (8 * r);
            rem = 0; padded = true;
        } else {
            w = 0;
        }
        return bswap32(w);
    }
};

// 128-bit read-only load of 16 message bytes (16-byte aligned): one LDG.E.128 instead of four LDG.E.32
struct word4 { uint32_t x, y, z, w; };
AFC_HD word4 ld_u128(const uint8_t* p) {
#if AFC_DEVICE_CODE
    uint4 v = __ldg((const uint4*)p);
    word4 r; r.x = v.x; r.y = v.y; r.z = v.z; r.w = v.w;
    return r;
#else
    word4 r;
    memcpy(&r, p, 16);
    return r;
#endif
}

#if AFC_DEVICE_CODE
// 32 read-only bytes (16-byte aligned) as two 128-bit loads (LDG.E.128.CONSTANT): sm_90 has no 256-bit global access.  Both
// halves fall in the same 32-byte sector, so a lane's gather still costs one sector.
AFC_HD void ldg_nc_32B(uint32_t* v, const uint32_t* p) {
    asm("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "l"(p));
    asm("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v[4]), "=r"(v[5]), "=r"(v[6]), "=r"(v[7]) : "l"(p + 4));
}
#endif

// The ends of a batch's offset arrays, which bound everything a call writes.  Span j writes out[2 j] = off[stride lo] and
// out[2 j + 1] = off[stride hi]: (lo, hi) = (0, n) when via < 0, else the two words span `via` (an earlier one) wrote, for an array indexed
// by those words.  A backwards (lo, hi) reads nothing and writes 0 for both words.  Run by one thread of k_offset_ends on the device
// arrays of a _dev call and on the host arrays by the afc_*_bound functions, so that both read the same words.
struct OffsetSpan { const uint64_t* off; uint32_t stride; int32_t via; };
AFC_HHD void offset_ends(const OffsetSpan* s, int k, uint32_t n, uint64_t* out) {
    for (int j = 0; j < k; j++) {
        const uint64_t lo = s[j].via < 0 ? 0 : out[2 * s[j].via], hi = s[j].via < 0 ? n : out[2 * s[j].via + 1];
        const bool ok = hi >= lo;
        out[2 * j] = ok ? s[j].off[s[j].stride * lo] : 0;
        out[2 * j + 1] = ok ? s[j].off[s[j].stride * hi] : 0;
    }
}

AFC_HD void store_be32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; }
AFC_HD uint32_t load_le32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
AFC_HD void store_le32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }

}  // namespace afc
