// float64 from decimal text and back, the way encoding/json does it for a value decoded into interface{} (afc_jsonval.cuh).
//
//   fl_parse   strconv.ParseFloat(s, 64) of a JSON number token  -?(0|[1-9]\d*)(\.\d+)?([eE][+-]?\d+)?  (the caller has checked the
//              syntax), correctly rounded:
//                exact path     at most 19 significant digits, mantissa <= 2^53 and |exponent| <= 22: one IEEE multiply or divide
//                Eisel-Lemire   the 19-digit mantissa times a 128-bit power of ten (Lemire, "Number Parsing at a Gigabyte per
//                               Second", Software: Practice and Experience 51(8), 2021); more than 19 digits are truncated to 19 and
//                               the value is accepted only if mantissa and mantissa + 1 round to the same float64 (what strconv does)
//              Declines (returns false, the caller's AFC_WEBHOOK_HOST): an Eisel-Lemire give-up (the product cannot decide the
//              rounding), a subnormal result, underflow to zero and overflow.  Zero mantissas give +-0 exactly.
//   fl_put     encoding/json floatEncoder: strconv's shortest digits that round-trip, the closest of them (Schubfach: Giulietti, "The
//              Schubfach way to render doubles", 2020), 'f' form, 'e' form when |x| < 1e-6 or |x| >= 1e21, e-0X cleaned to e-X; -0 is
//              written as -0.  Only finite, non-subnormal values reach it (fl_parse declines the rest).
//
// The power tables (afc_float.inc, tools/gen_constants.py --float) are indexed by a value that differs from thread to thread, so
// they are read from global memory through the read-only path, not from __constant__ (which serialises divergent reads).
#pragma once
#include "afc_common.cuh"

namespace afc {

#if AFC_DEVICE_CODE || defined(__CUDACC__)
#define AFC_CONST_DECL static __device__ const
#else
#define AFC_CONST_DECL static const
#endif
#include "afc_float.inc"
#undef AFC_CONST_DECL

AFC_HD uint64_t fl_tab(const uint64_t* t, int i) {
#if AFC_DEVICE_CODE
    return __ldg((const unsigned long long*)t + i);
#else
    return t[i];
#endif
}
AFC_HD uint64_t fl_mulhi(uint64_t a, uint64_t b) {
#if AFC_DEVICE_CODE
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}
AFC_HD uint32_t fl_clz64(uint64_t x) {          // x != 0
#if AFC_DEVICE_CODE
    return (uint32_t)__clzll((long long)x);
#else
    return (uint32_t)__builtin_clzll(x);
#endif
}
AFC_HD double fl_from_bits(uint64_t b) {
#if AFC_DEVICE_CODE
    return __longlong_as_double((long long)b);
#else
    double d; memcpy(&d, &b, 8); return d;
#endif
}
AFC_HD double fl_u64_to_double(uint64_t x) {     // round to nearest, ties to even
#if AFC_DEVICE_CODE
    return __ull2double_rn((unsigned long long)x);
#else
    return (double)x;
#endif
}
AFC_HD uint64_t fl_to_bits(double d) {
#if AFC_DEVICE_CODE
    return (uint64_t)__double_as_longlong(d);
#else
    uint64_t b; memcpy(&b, &d, 8); return b;
#endif
}

// Eisel-Lemire for man * 10^e10 (man != 0, at most 19 digits): the float64 bits without sign, or false where it cannot decide, the
// result is subnormal or zero, or it overflows
AFC_HD bool fl_eisel_lemire(uint64_t man, int e10, uint64_t* bits) {
    if (e10 < AFC_EL_MIN || e10 > AFC_EL_MAX) return false;
    const int idx = 2 * (e10 - AFC_EL_MIN);
    const uint64_t thi = fl_tab(AFC_POW10_EL, idx), tlo = fl_tab(AFC_POW10_EL, idx + 1);
    const uint32_t clz = fl_clz64(man);
    man <<= clz;
    // biased exponent of the result if the product's top bit is set: floor(e10 log2 10) + 64 + 1023 - clz
    int64_t exp2 = (int64_t)((e10 * 217706) >> 16) + 64 + 1023 - (int64_t)clz;
    uint64_t hi = fl_mulhi(man, thi), lo = man * thi;
    // the table is rounded down, so the exact product lies in [hi:lo, hi:lo + man); widen with the low word when the 9 bits below
    // the 55 kept ones are all ones and the low word could carry
    if ((hi & 0x1ff) == 0x1ff && lo + man < man) {
        const uint64_t yhi = fl_mulhi(man, tlo), ylo = man * tlo;
        uint64_t mhi = hi, mlo = lo + yhi;
        if (mlo < lo) ++mhi;
        if ((mhi & 0x1ff) == 0x1ff && mlo + 1 == 0 && ylo + man < man) return false;
        hi = mhi; lo = mlo;
    }
    const uint64_t msb = hi >> 63;
    uint64_t m = hi >> (msb + 9);                 // 54 bits
    exp2 -= (int64_t)(1 ^ msb);
    if (lo == 0 && (hi & 0x1ff) == 0 && (m & 3) == 1) return false;   // exactly halfway as far as the product can tell
    m += m & 1;                                   // round half to even, then drop the extra bit
    m >>= 1;
    if (m >> 53) { m >>= 1; ++exp2; }
    if (exp2 <= 0 || exp2 >= 0x7ff) return false; // subnormal / zero, or infinite
    *bits = ((uint64_t)exp2 << 52) | (m & ((1ull << 52) - 1));
    return true;
}

// strconv.ParseFloat(d[0..len), 64) for a token the JSON grammar accepts; false = declined (see the header comment)
AFC_HD bool fl_parse(const uint8_t* d, uint32_t len, uint64_t* out_bits) {
    uint32_t p = 0;
    const bool neg = d[0] == '-';
    if (neg) ++p;
    // strconv readFloat: nd significant digits, the first nm (<= 19) of them in man, dp = digits before the point
    uint64_t man = 0;
    int nd = 0, nm = 0, dp = 0;
    bool trunc = false, dot = false;
    for (; p < len; ++p) {
        const uint32_t c = d[p];
        if (c == '.') { dot = true; dp = nd; continue; }
        if (c < '0' || c > '9') break;
        if (c == '0' && nd == 0) { --dp; continue; }          // leading zeros carry no digits
        ++nd;
        if (nm < 19) { man = man * 10 + (c - '0'); ++nm; }
        else if (c != '0') trunc = true;
    }
    if (!dot) dp = nd;
    int64_t ex = 0;
    if (p < len) {                                // [eE][+-]?\d+
        ++p;
        bool eneg = false;
        if (d[p] == '+' || d[p] == '-') { eneg = d[p] == '-'; ++p; }
        for (; p < len; ++p) if (ex < 100000) ex = ex * 10 + (d[p] - '0');
        if (eneg) ex = -ex;
    }
    const uint64_t sign = neg ? 1ull << 63 : 0;
    if (man == 0) { *out_bits = sign; return true; }                     // +-0 whatever the exponent
    const int64_t e10 = ex + dp - nm;             // value = man * 10^e10 (man possibly truncated)
    if (e10 < -400 || e10 > 400) return false;    // far out of range: underflow or overflow
    if (!trunc && man <= (1ull << 53) && e10 >= -22 && e10 <= 22 + 15) {     // exact: one rounding of two exact float64s
        double f = (double)man, p10 = 1.0;
        int x = (int)e10;
        if (x > 22) {                             // move the excess into the mantissa while it stays exact (< 10^15)
            for (int k = 0; k < x - 22; k++) p10 *= 10.0;
            f *= p10;
            x = 22;
            p10 = 1.0;
        }
        if (f <= 1e15) {
            for (int k = 0; k < (x < 0 ? -x : x); k++) p10 *= 10.0;
            *out_bits = fl_to_bits(x >= 0 ? f * p10 : f / p10) | sign;
            return true;
        }
    }
    // Values that are integers below 2^64, or integers below 2^64 over 2^k (the decimal exponent is -k and 5^k divides the mantissa):
    // one correctly rounded integer conversion, then an exact scaling.  These are the inputs Eisel-Lemire cannot decide against a
    // table rounded down (the product lands just below an exactly representable value), such as the 17-digit spelling of a float64
    // between 2^53 and 2^60 with a fractional part.
    if (!trunc && e10 >= -27 && e10 <= 19) {
        uint64_t p = 1;
        for (int k = 0; k < (e10 < 0 ? -e10 : e10); k++) p *= e10 < 0 ? 5 : 10;
        if (e10 >= 0 && fl_mulhi(man, p) == 0) { *out_bits = fl_to_bits(fl_u64_to_double(man * p)) | sign; return true; }
        if (e10 < 0 && man % p == 0) {
            *out_bits = fl_to_bits(fl_u64_to_double(man / p) * fl_from_bits((uint64_t)(1023 + e10) << 52)) | sign;
            return true;
        }
    }
    uint64_t b;
    if (!fl_eisel_lemire(man, (int)e10, &b)) return false;
    if (trunc) {                                  // the dropped digits lie strictly between man and man + 1
        uint64_t b1;
        if (!fl_eisel_lemire(man + 1, (int)e10, &b1) || b1 != b) return false;
    }
    *out_bits = b | sign;
    return true;
}

// ---- Schubfach: the shortest decimal f * 10^e that rounds to c * 2^q (c the 53-bit significand of a normal float64), the closest
// of them, ties to an even last digit
AFC_HD uint64_t fl_rop(uint64_t g1, uint64_t g0, uint64_t cp) {
    const uint64_t x1 = fl_mulhi(g0, cp);
    const uint64_t y0 = g1 * cp, y1 = fl_mulhi(g1, cp);
    const uint64_t z = (y0 >> 1) + x1;
    const uint64_t vbp = y1 + (z >> 63);
    const uint64_t M63 = (1ull << 63) - 1;
    return vbp | (((z & M63) + M63) >> 63);
}
AFC_HD void fl_shortest(uint64_t c, int q, uint64_t* f_out, int* e_out) {
    const uint64_t out = c & 1;
    const uint64_t cb = c << 2, cbr = cb + 2;
    uint64_t cbl;
    int k;
    if (c != (1ull << 52) || q == -1074) { cbl = cb - 2; k = (int)(((int64_t)q * 661971961083LL) >> 41); }
    else { cbl = cb - 1; k = (int)(((int64_t)q * 661971961083LL - 274743187321LL) >> 41); }
    const int h = q + (int)(((int64_t)(-k) * 913124641741LL) >> 38) + 2;
    const int idx = 2 * (-k - AFC_SF_MIN);
    const uint64_t g1 = fl_tab(AFC_POW10_SF, idx), g0 = fl_tab(AFC_POW10_SF, idx + 1);
    const uint64_t vb = fl_rop(g1, g0, cb << h), vbl = fl_rop(g1, g0, cbl << h), vbr = fl_rop(g1, g0, cbr << h);
    const uint64_t s = vb >> 2;
    if (s >= 100) {
        const uint64_t sp10 = s / 10 * 10, tp10 = sp10 + 10;
        const bool upin = vbl + out <= sp10 << 2, wpin = (tp10 << 2) + out <= vbr;
        if (upin != wpin) { *f_out = upin ? sp10 : tp10; *e_out = k; return; }
    }
    const uint64_t t = s + 1;
    const bool uin = vbl + out <= s << 2, win = (t << 2) + out <= vbr;
    if (uin != win) { *f_out = uin ? s : t; *e_out = k; return; }
    const int64_t cmp = (int64_t)(vb - ((s + t) << 1));
    *f_out = (cmp < 0 || (cmp == 0 && (s & 1) == 0)) ? s : t;
    *e_out = k;
}

// The float64 with these bits (finite; zero or normal) as encoding/json writes it
template <class Sink>
AFC_HD void fl_put(Sink& out, uint64_t bits) {
    if (bits >> 63) out.put('-');
    const uint64_t mag = bits & ~(1ull << 63);
    if (mag == 0) { out.put('0'); return; }
    const int be = (int)(mag >> 52);
    uint64_t f;
    int e;
    fl_shortest((mag & ((1ull << 52) - 1)) | (1ull << 52), be - 1075, &f, &e);
    while (f % 10 == 0) { f /= 10; ++e; }
    uint64_t p10 = 1;
    int nd = 1;
    while (f / p10 >= 10) { p10 *= 10; ++nd; }
    const int pt = nd + e;                        // value = 0.d1 d2 ... dn x 10^pt
    const double a = fl_from_bits(mag);
    if (a < 1e-6 || a >= 1e21) {                  // d1[.d2...dn]e(+|-)X
        out.put('0' + (uint32_t)(f / p10));
        if (nd > 1) {
            out.put('.');
            for (uint64_t q = p10 / 10; q; q /= 10) out.put('0' + (uint32_t)((f / q) % 10));
        }
        out.put('e');
        int x = pt - 1;
        out.put(x < 0 ? '-' : '+');
        if (x < 0) x = -x;
        if (x >= 100) out.put('0' + x / 100);
        if (x >= 10) out.put('0' + (x / 10) % 10);
        out.put('0' + x % 10);
        return;
    }
    if (pt <= 0) {                                // 0.000ddd
        out.put('0'); out.put('.');
        for (int z = 0; z < -pt; z++) out.put('0');
        for (uint64_t q = p10; q; q /= 10) out.put('0' + (uint32_t)((f / q) % 10));
        return;
    }
    int j = 0;                                    // ddd[.ddd] or ddd000
    for (uint64_t q = p10; q; q /= 10, ++j) {
        if (j == pt) out.put('.');
        out.put('0' + (uint32_t)((f / q) % 10));
    }
    for (; j < pt; j++) out.put('0');
}

}  // namespace afc
