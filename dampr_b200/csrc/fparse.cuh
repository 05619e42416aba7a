// fparse.cuh: parse_f64, a correctly rounded decimal -> double parser for host and device code.
//
// It gives the bits of Python's float(s) for every string it accepts, and returns false for every other string
// (the caller then lets Python decide). Accepted, ASCII only:
//   [ \t]* [+-]? (\d+ \.? \d* | \. \d+) ([eE] [+-]? \d+)? [ \t]*
// with at most 19 significant digits (leading zeros dropped, trailing zeros counted). Refused: inf / nan /
// infinity, underscores, any other whitespace, more than 19 significant digits, empty or malformed text.
// A huge exponent gives +-inf or a (signed) zero, as float() does.
//
// Two steps:
//   1. Clinger's fast path: mantissa w <= 2^53 and |q| <= 22, so w and 10^|q| are exact doubles and one
//      correctly rounded multiply or divide is the answer.
//   2. Eisel-Lemire (Lemire, "Number Parsing at a Gigabyte per Second", 2021): w normalised to 64 bits times a
//      truncated 128-bit 5^q (pow5.cuh, tools/gen_pow5.py) gives the top bits of w * 10^q; when the truncation
//      could change the rounding (the discarded bits are all ones) the function returns false.
#pragma once
#include <stdint.h>

#include "pow5.cuh"

#if defined(__CUDACC__)
#define DAMPR_FP_HD __host__ __device__ __forceinline__
#else
#define DAMPR_FP_HD inline
#endif

namespace fparse {

#if defined(__CUDACC__)
// global, not __constant__: the threads of a warp read different entries, which constant memory serialises
static __device__ const uint64_t kPow5Dev[] = {DAMPR_POW5_DATA};
#endif
static const uint64_t kPow5Host[] = {DAMPR_POW5_DATA};

DAMPR_FP_HD const uint64_t *pow5_table() {
#if defined(__CUDA_ARCH__)
    return kPow5Dev;
#else
    return kPow5Host;
#endif
}

DAMPR_FP_HD void mul_64x64(uint64_t a, uint64_t b, uint64_t &hi, uint64_t &lo) {
#if defined(__CUDA_ARCH__)
    lo = a * b;
    hi = __umul64hi(a, b);
#else
    const unsigned __int128 p = (unsigned __int128)a * b;
    lo = (uint64_t)p;
    hi = (uint64_t)(p >> 64);
#endif
}

DAMPR_FP_HD int clz64(uint64_t x) {
#if defined(__CUDA_ARCH__)
    return __clzll((long long)x);
#else
    return __builtin_clzll(x);
#endif
}

DAMPR_FP_HD double bits_to_f64(uint64_t b) {
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)b);
#else
    double d;
    __builtin_memcpy(&d, &b, 8);
    return d;
#endif
}

DAMPR_FP_HD double exact_pow10(int k) {   // 10^k for 0 <= k <= 22: exact doubles
    double r = 1.0;
    double b = 10.0;
    while (k) {   // the products stay exact: every partial power of ten up to 10^22 is a double
        if (k & 1) r *= b;
        b *= b;
        k >>= 1;
    }
    return r;
}

// w * 10^q (w != 0, at most 19 digits) as the bits of a positive double; false when undecided
DAMPR_FP_HD bool eisel_lemire(uint64_t w, int q, uint64_t &bits) {
    if (q < DAMPR_POW5_QMIN) {   // w * 10^q < 10^19 * 10^-343 is below half the smallest subnormal
        bits = 0;
        return true;
    }
    if (q > DAMPR_POW5_QMAX) {   // w * 10^q >= 10^309
        bits = 0x7FF0000000000000ULL;
        return true;
    }
    const int lz = clz64(w);
    w <<= lz;
    const uint64_t *t = pow5_table() + 2 * (q - DAMPR_POW5_QMIN);
    uint64_t hi, lo;
    mul_64x64(w, t[0], hi, lo);
    if ((hi & 0x1FFULL) == 0x1FFULL) {   // the 55 bits kept could still move: add the low word's product
        uint64_t h2, l2;
        mul_64x64(w, t[1], h2, l2);
        lo += h2;
        if (lo < h2) ++hi;
        if ((hi & 0x1FFULL) == 0x1FFULL && lo == ~0ULL) return false;   // the truncated table decides nothing
    }
    const int upper = (int)(hi >> 63);
    const int shift = upper + 9;   // keep 54 bits + the leading one: 53 for the mantissa, one to round with
    uint64_t m = hi >> shift;
    // binary exponent: floor(q * log2(10)) + 63, for |q| < 1700 (217706 / 2^16 ~ log2(10))
    int p2 = (int)(((217706LL * q) >> 16) + 63) + upper - lz + 1023;
    if (p2 <= 0) {   // subnormal
        if (-p2 + 1 >= 64) {
            bits = 0;
            return true;
        }
        m >>= -p2 + 1;
        m += m & 1;
        m >>= 1;
        // rounding up may reach the smallest normal number: then the exponent field is 1
        bits = m;   // m < 2^52: exponent field 0; m == 2^52: exponent field 1, mantissa 0 (the same bits)
        return true;
    }
    // an exact halfway case can only arise for small |q| (5^q fits the product exactly); it rounds to even
    if (lo <= 1 && q >= -4 && q <= 23 && (m & 3) == 1 && (m << shift) == hi) m &= ~1ULL;
    m += m & 1;
    m >>= 1;
    if (m >= (2ULL << 52)) {
        m = 1ULL << 52;
        ++p2;
    }
    m &= ~(1ULL << 52);
    if (p2 >= 0x7FF) {
        bits = 0x7FF0000000000000ULL;
        return true;
    }
    bits = ((uint64_t)p2 << 52) | m;
    return true;
}

DAMPR_FP_HD double fast_path(uint64_t w, int q) {
    const double d = (double)w;
#if defined(__CUDA_ARCH__)
    return q < 0 ? __ddiv_rn(d, exact_pow10(-q)) : __dmul_rn(d, exact_pow10(q));
#else
    return q < 0 ? d / exact_pow10(-q) : d * exact_pow10(q);
#endif
}

}  // namespace fparse

// Python's float() of p[0 .. len) into out; false for every string outside the grammar above (Python decides)
DAMPR_FP_HD bool parse_f64(const uint8_t *p, uint32_t len, double &out) {
    uint32_t i = 0, e = len;
    while (i < e && (p[i] == ' ' || p[i] == '\t')) ++i;
    while (e > i && (p[e - 1] == ' ' || p[e - 1] == '\t')) --e;
    bool neg = false;
    if (i < e && (p[i] == '+' || p[i] == '-')) {
        neg = p[i] == '-';
        ++i;
    }
    uint64_t w = 0;
    int nd = 0;        // significant digits taken into w
    int ndig = 0;      // digits of the mantissa seen
    int dexp = 0;      // decimal exponent correction: -(significant digits after the point)
    bool dot = false;
    for (; i < e; ++i) {
        const uint32_t c = p[i];
        if (c == '.') {
            if (dot) return false;
            dot = true;
            continue;
        }
        const uint32_t d = c - '0';
        if (d > 9) break;
        ++ndig;
        if (w == 0 && d == 0) {   // a leading zero: not significant
            if (dot) --dexp;
            continue;
        }
        if (++nd > 19) return false;
        w = w * 10 + d;
        if (dot) --dexp;
    }
    if (ndig == 0) return false;
    int q = dexp;
    if (i < e) {
        if (p[i] != 'e' && p[i] != 'E') return false;
        ++i;
        bool eneg = false;
        if (i < e && (p[i] == '+' || p[i] == '-')) {
            eneg = p[i] == '-';
            ++i;
        }
        if (i >= e) return false;
        int x = 0;
        for (; i < e; ++i) {
            const uint32_t d = (uint32_t)p[i] - '0';
            if (d > 9) return false;
            if (x < 100000) x = x * 10 + (int)d;   // beyond that only the sign of the result matters
        }
        q += eneg ? -x : x;
    }
    uint64_t bits;
    if (w == 0) {
        bits = 0;
    } else if (w <= (1ULL << 53) && q >= -22 && q <= 22) {
        out = fparse::fast_path(w, q);
        if (neg) out = -out;
        return true;
    } else if (!fparse::eisel_lemire(w, q, bits)) {
        return false;
    }
    if (neg) bits |= 0x8000000000000000ULL;
    out = fparse::bits_to_f64(bits);
    return true;
}
