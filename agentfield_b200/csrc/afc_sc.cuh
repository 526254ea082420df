// Scalars modulo the group order L = 2^252 + 27742317777372353535851937790883648493 (RFC 8032 §5.1).
//
// Replaces edwards25519.Scalar.{SetUniformBytes, SetCanonicalBytes, MultiplyAdd} as used by Go's
// ed25519.Sign / ed25519.Verify (reference call sites vc_service.go:463,504).  Barrett reduction with
// 32-bit limbs (HAC 14.42, b = 2^32, k = 8, mu = floor(2^512 / L)); a few hundred integer ops per
// credential — negligible next to the curve arithmetic, so written in portable C.
#pragma once
#include "afc_sha.cuh"   // brings in afc_consts.inc (AFC_L_32, AFC_MU_32)

namespace afc {

AFC_HD int sc_geq(const uint32_t* a, const uint32_t* b, int n) {
    // a >= b, branch-free over n limbs
    int64_t bw = 0;
#pragma unroll
    for (int i = 0; i < 9; i++) {
        if (i < n) { bw += (int64_t)a[i] - b[i]; bw >>= 32; }
    }
    return bw == 0;
}

// out[8] = x[16] mod L
AFC_HD void sc_reduce512(uint32_t* out, const uint32_t* x) {
    uint32_t q2[18];
#pragma unroll
    for (int i = 0; i < 18; i++) q2[i] = 0;
#pragma unroll
    for (int i = 0; i < 9; i++) {                   // q2 = (x >> 224) * mu
        uint64_t c = 0;
#pragma unroll
        for (int j = 0; j < 9; j++) { c += (uint64_t)x[7 + i] * AFC_MU_32[j] + q2[i + j]; q2[i + j] = (uint32_t)c; c >>= 32; }
        q2[i + 9] = (uint32_t)c;
    }
    uint32_t r2[9];                                 // r2 = (q2 >> 288) * L mod 2^288
#pragma unroll
    for (int i = 0; i < 9; i++) r2[i] = 0;
#pragma unroll
    for (int i = 0; i < 9; i++) {
        uint64_t c = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            if (i + j < 9) { c += (uint64_t)q2[9 + i] * AFC_L_32[j] + r2[i + j]; r2[i + j] = (uint32_t)c; c >>= 32; }
        }
        if (i == 0) r2[8] += (uint32_t)c;
    }
    uint32_t r[9], l9[9];
    int64_t bw = 0;
#pragma unroll
    for (int i = 0; i < 9; i++) { bw += (int64_t)x[i] - r2[i]; r[i] = (uint32_t)bw; bw >>= 32; }
#pragma unroll
    for (int i = 0; i < 9; i++) l9[i] = (i < 8) ? AFC_L_32[i] : 0u;
#pragma unroll
    for (int k = 0; k < 2; k++) {                   // at most two corrective subtractions (HAC 14.42)
        uint32_t m = 0u - (uint32_t)sc_geq(r, l9, 9);
        bw = 0;
#pragma unroll
        for (int i = 0; i < 9; i++) { bw += (int64_t)r[i] - (l9[i] & m); r[i] = (uint32_t)bw; bw >>= 32; }
    }
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = r[i];
}

// out = x mod L for a 256-bit x
AFC_HD void sc_reduce256(uint32_t* out, const uint32_t* x) {
    uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = (i < 8) ? x[i] : 0u;
    sc_reduce512(out, w);
}

// out = (a*b + c) mod L
AFC_HD void sc_muladd(uint32_t* out, const uint32_t* a, const uint32_t* b, const uint32_t* c) {
    uint32_t x[16];
#pragma unroll
    for (int i = 0; i < 16; i++) x[i] = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        uint64_t cy = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) { cy += (uint64_t)a[i] * b[j] + x[i + j]; x[i + j] = (uint32_t)cy; cy >>= 32; }
        x[i + 8] = (uint32_t)cy;
    }
    uint64_t cy = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) { cy += (uint64_t)x[i] + ((i < 8) ? c[i] : 0u); x[i] = (uint32_t)cy; cy >>= 32; }
    sc_reduce512(out, x);
}

AFC_HD int sc_is_canonical(const uint32_t* s) { return !sc_geq(s, AFC_L_32, 8); }

// Signed radix-16 recoding of s < 2^254: t = s + 0x88..8; digit_i = nibble_i(t) - 8 in [-8, 7].
AFC_HD void sc_recode16(uint32_t* t, const uint32_t* s) {
    uint64_t c = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) { c += (uint64_t)s[i] + 0x88888888u; t[i] = (uint32_t)c; c >>= 32; }
}
AFC_HD int sc_digit16(const uint32_t* t, int i) { return (int)((t[i >> 3] >> ((i & 7) * 4)) & 15u) - 8; }

// Signed radix-256 recoding of s < 2^254: t = s + 0x80..80; digit_i = byte_i(t) - 128 in [-128, 127].
AFC_HD void sc_recode256(uint32_t* t, const uint32_t* s) {
    uint64_t c = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) { c += (uint64_t)s[i] + 0x80808080u; t[i] = (uint32_t)c; c >>= 32; }
}
AFC_HD int sc_digit256(const uint32_t* t, int i) { return (int)((t[i >> 2] >> ((i & 3) * 8)) & 255u) - 128; }

// Signed radix-65536 recoding of s < 2^254: t = s + 0x8000..8000; digit_i = half_i(t) - 32768 in [-32768, 32767].
AFC_HD void sc_recode65536(uint32_t* t, const uint32_t* s) {
    uint64_t c = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) { c += (uint64_t)s[i] + 0x80008000u; t[i] = (uint32_t)c; c >>= 32; }
}
AFC_HD int sc_digit65536(const uint32_t* t, int i) { return (int)((t[i >> 1] >> ((i & 1) * 16)) & 65535u) - 32768; }

// Signed radix-2^w recoding of s < L for any w in 16..22 (the verify-only fixed-base table): rows = ceil(254 / w);
// t = s + C with C = 2^(w-1) (1 + 2^w + ... + 2^(w (rows-2))); digit_i = field_i(t) - 2^(w-1) in [-2^(w-1), 2^(w-1)) for
// i < rows - 1; the top digit is everything above, t >> (w (rows-1)), with no offset: s < L < 2^253 bounds it by 2^(w-1)
// (it is 0 or 1 when w (rows-1) = 252).  At w = 16 the digits are those of sc_recode65536.
AFC_HHD int sc_wide_rows(int w) { return (254 + w - 1) / w; }
AFC_HHD void sc_wide_offset(uint32_t* c, int w) {
    for (int i = 0; i < 8; i++) c[i] = 0;
    for (int i = 0; i + 1 < sc_wide_rows(w); i++) { const int b = w * i + w - 1; c[b >> 5] |= 1u << (b & 31); }
}
AFC_HHD void sc_recode_wide(uint32_t* t, const uint32_t* s, const uint32_t* offset) {
    uint64_t c = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) { c += (uint64_t)s[i] + offset[i]; t[i] = (uint32_t)c; c >>= 32; }
}
AFC_HHD int sc_digit_wide(const uint32_t* t, int i, int w, int rows) {
    const int p = w * i, lo = p >> 5;
    const uint64_t v = (uint64_t)t[lo] | (lo < 7 ? (uint64_t)t[lo + 1] << 32 : 0ull);
    const uint32_t f = (uint32_t)(v >> (p & 31));
    return i + 1 == rows ? (int)f : (int)(f & ((1u << w) - 1u)) - (1 << (w - 1));
}

}  // namespace afc
