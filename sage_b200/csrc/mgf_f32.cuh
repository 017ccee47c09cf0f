// Decimal text -> f32 as Rust's `str::parse::<f32>` (core dec2flt) defines it: the grammar, and the correctly rounded (half to even) value
// for any number of digits and any exponent. Host and device code: the host build is what tests can run without a GPU.
//
//   grammar    [+-]? ( inf | infinity | nan  (any case)  |  digits [. digits?]? | . digits ) ( [eE] [+-]? digits )?   and nothing else
//   value      1. Clinger's fast path: at most 19 significant digits, w <= 2^24 and |q| <= 10: one correctly rounded f32 mul or div.
//              2. Eisel-Lemire on the first 19 significant digits with mgf_pow5.cuh's 128-bit powers of five; with more digits, the result
//                 must agree for w and w + 1, else 3.
//              3. Exact decimal shifting (digits kept to MGF_DEC_DIGITS, a sticky flag for the rest; an f32 halfway point needs at most
//                 112 significant digits): multiply or divide by powers of two until the value is in [1/2, 1), then round 24 bits.
// NaN is 0x7FC00000 (0xFFC00000 with '-'); overflow gives +-inf and underflow +-0. The decimal exponent saturates at +-10^12, past which
// every input of fewer than 10^12 digits is inf or 0.
#pragma once
#include <stdint.h>

#ifndef __CUDACC__
#define __host__
#define __device__
#define __forceinline__ inline
#endif

#include "mgf_pow5.cuh"

namespace sb {

constexpr int MGF_DEC_DIGITS = 800;

__host__ __device__ __forceinline__ bool mgf_is_digit(uint8_t c) { return c >= '0' && c <= '9'; }
__host__ __device__ __forceinline__ uint8_t mgf_lower(uint8_t c) { return (c >= 'A' && c <= 'Z') ? (uint8_t)(c + 32) : c; }

__host__ __device__ __forceinline__ int mgf_clz64(uint64_t x) {
#ifdef __CUDA_ARCH__
    return __clzll((long long)x);
#else
    return __builtin_clzll(x);
#endif
}
__host__ __device__ __forceinline__ void mgf_mul128(uint64_t a, uint64_t b, uint64_t& lo, uint64_t& hi) {
#ifdef __CUDA_ARCH__
    lo = a * b;
    hi = __umul64hi(a, b);
#else
    const unsigned __int128 p = (unsigned __int128)a * b;
    lo = (uint64_t)p;
    hi = (uint64_t)(p >> 64);
#endif
}
__host__ __device__ __forceinline__ float mgf_from_bits(uint32_t u) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    __builtin_memcpy(&f, &u, 4);
    return f;
#endif
}

// The big decimal of step 3: value = 0.d[0] d[1] ... d[nd-1] x 10^dp, d[0] != 0, no trailing zeros; trunc: nonzero digits were dropped.
struct MgfDecimal {
    int nd, dp;
    bool trunc;
    uint8_t d[MGF_DEC_DIGITS + 24];
};

__host__ __device__ inline void mgf_dec_trim(MgfDecimal& D) {
    while (D.nd > 0 && D.d[D.nd - 1] == 0) D.nd--;
}

// D /= 2^k, 1 <= k <= 60
__host__ __device__ inline void mgf_dec_rshift(MgfDecimal& D, int k) {
    int r = 0, w = 0;
    uint64_t n = 0;
    while ((n >> k) == 0) {
        if (r < D.nd) {
            n = 10 * n + D.d[r++];
        } else if (n == 0) {
            D.nd = 0;
            return;
        } else {
            while ((n >> k) == 0) { n *= 10; r++; }
            break;
        }
    }
    D.dp -= r - 1;
    const uint64_t mask = (1ull << k) - 1;
    while (r < D.nd) {
        const uint8_t q = (uint8_t)(n >> k);
        n = 10 * (n & mask) + D.d[r++];
        D.d[w++] = q;
    }
    while (n > 0) {
        const uint8_t q = (uint8_t)(n >> k);
        n = 10 * (n & mask);
        if (w < MGF_DEC_DIGITS) D.d[w++] = q;
        else if (q > 0) D.trunc = true;
    }
    D.nd = w;
    mgf_dec_trim(D);
}

// D *= 2^k, 1 <= k <= 60: written right-aligned k/3 + 1 places further out (at least the digits the product gains), then moved down.
__host__ __device__ inline void mgf_dec_lshift(MgfDecimal& D, int k) {
    if (D.nd == 0) return;
    const int extra = k / 3 + 1;
    int rd = D.nd, wr = D.nd + extra;
    uint64_t n = 0;
    while (rd > 0) {
        rd--;
        wr--;
        n += (uint64_t)D.d[rd] << k;
        const uint64_t q = n / 10;
        D.d[wr] = (uint8_t)(n - 10 * q);
        n = q;
    }
    while (n > 0) {
        wr--;
        const uint64_t q = n / 10;
        D.d[wr] = (uint8_t)(n - 10 * q);
        n = q;
    }
    int len = D.nd + extra - wr;
    for (int i = 0; i < len; i++) D.d[i] = D.d[wr + i];
    D.dp += len - D.nd;
    if (len > MGF_DEC_DIGITS) {
        for (int i = MGF_DEC_DIGITS; i < len; i++)
            if (D.d[i]) D.trunc = true;
        len = MGF_DEC_DIGITS;
    }
    D.nd = len;
    mgf_dec_trim(D);
}

// The integer part of D rounded half to even (the sticky flag breaks a tie upwards); D < 10^19.
__host__ __device__ inline uint64_t mgf_dec_round(const MgfDecimal& D) {
    if (D.nd == 0 || D.dp < 0) return 0;
    uint64_t n = 0;
    for (int i = 0; i < D.dp; i++) n = 10 * n + (i < D.nd ? D.d[i] : 0);
    bool up = false;
    if (D.dp < D.nd) {
        up = D.d[D.dp] >= 5;
        if (D.d[D.dp] == 5 && D.dp + 1 == D.nd) up = D.trunc || (n & 1);
    }
    return n + (up ? 1 : 0);
}

__host__ __device__ inline int mgf_dec_shift_for(int n) {
    constexpr uint8_t P[19] = {0, 3, 6, 9, 13, 16, 19, 23, 26, 29, 33, 36, 39, 43, 46, 49, 53, 56, 59};   // floor(log2(10^n))
    return n < 19 ? P[n] : 60;
}

// Step 3 on D (nonzero): the f32 bits without the sign.
__host__ __device__ inline uint32_t mgf_dec_to_f32(MgfDecimal& D) {
    constexpr int MIN_EXP = -127, MANT = 23;
    if (D.dp < -50) return 0;
    if (D.dp > 40) return 0x7F800000u;
    int e2 = 0;
    while (D.dp > 0) {
        const int s = mgf_dec_shift_for(D.dp);
        mgf_dec_rshift(D, s);
        e2 += s;
    }
    while (D.dp <= 0) {
        int s;
        if (D.dp == 0) {
            if (D.d[0] >= 5) break;
            s = D.d[0] < 2 ? 2 : 1;
        } else {
            s = mgf_dec_shift_for(-D.dp);
        }
        mgf_dec_lshift(D, s);
        e2 -= s;
    }
    e2 -= 1;   // D in [1/2, 1): value = 2D x 2^e2, 2D in [1, 2)
    while (MIN_EXP + 1 > e2) {
        int n = MIN_EXP + 1 - e2;
        if (n > 60) n = 60;
        mgf_dec_rshift(D, n);
        e2 += n;
    }
    if (e2 - MIN_EXP >= 0xFF) return 0x7F800000u;
    mgf_dec_lshift(D, MANT + 1);
    uint64_t m = mgf_dec_round(D);
    if (m >= (1ull << (MANT + 1))) {
        mgf_dec_rshift(D, 1);
        e2 += 1;
        m = mgf_dec_round(D);
        if (e2 - MIN_EXP >= 0xFF) return 0x7F800000u;
    }
    int p2 = e2 - MIN_EXP;
    if (m < (1ull << MANT)) p2 -= 1;
    return ((uint32_t)p2 << MANT) | (uint32_t)(m & ((1ull << MANT) - 1));
}

// Step 2: w x 10^q (w != 0) as biased exponent << 23 | mantissa, or -1 when the 128-bit product cannot decide.
__host__ __device__ inline int64_t mgf_lemire(int64_t q, uint64_t w) {
    constexpr int MANT = 23, MIN_EXP = -127;
    if (q < MGF_POW5_MIN) return 0;
    if (q > MGF_POW5_MAX) return 0x7F800000;
    const int lz = mgf_clz64(w);
    w <<= lz;
    const uint64_t* p5 = mgf_pow5((int)q);
    uint64_t lo, hi;
    mgf_mul128(w, p5[0], lo, hi);
    const uint64_t mask = ~0ull >> (MANT + 3);
    if ((hi & mask) == mask) {
        uint64_t lo2, hi2;
        mgf_mul128(w, p5[1], lo2, hi2);
        lo += hi2;
        if (hi2 > lo) hi++;
    }
    if (lo == ~0ull && !(q >= -27 && q <= 55)) return -1;
    const int upper = (int)(hi >> 63);
    uint64_t m = hi >> (upper + 64 - MANT - 3);
    int p2 = (int)(((152170 + 65536) * q) >> 16) + 63 + upper - lz - MIN_EXP;
    if (p2 <= 0) {
        if (-p2 + 1 >= 64) return 0;
        m >>= -p2 + 1;
        m += m & 1;
        m >>= 1;
        p2 = m >= (1ull << MANT) ? 1 : 0;
        return ((int64_t)p2 << MANT) | (int64_t)(m & ((1ull << MANT) - 1));
    }
    if (lo <= 1 && q >= -17 && q <= 10 && (m & 3) == 1 && (m << (upper + 64 - MANT - 3)) == hi) m &= ~1ull;
    m += m & 1;
    m >>= 1;
    if (m >= (2ull << MANT)) {
        m = 1ull << MANT;
        p2++;
    }
    if (p2 >= 0xFF) return 0x7F800000;
    return ((int64_t)p2 << MANT) | (int64_t)(m & ((1ull << MANT) - 1));
}

// Parses s[0, n). Returns false (and leaves *out) when the token is not in the grammar.
__host__ __device__ inline bool mgf_parse_f32(const uint8_t* s, uint64_t n, float* out) {
    if (n == 0) return false;
    const bool neg = s[0] == '-';
    if (s[0] == '-' || s[0] == '+') { s++; n--; }
    if (n == 0) return false;
    const uint32_t sign = neg ? 0x80000000u : 0u;
    if (!mgf_is_digit(s[0]) && s[0] != '.') {
        const char* words[3] = {"nan", "inf", "infinity"};
        const uint32_t bits[3] = {0x7FC00000u, 0x7F800000u, 0x7F800000u};
        for (int k = 0; k < 3; k++) {
            uint64_t len = 0;
            while (words[k][len]) len++;
            if (len != n) continue;
            bool eq = true;
            for (uint64_t i = 0; i < n; i++) eq = eq && mgf_lower(s[i]) == (uint8_t)words[k][i];
            if (eq) { *out = mgf_from_bits(bits[k] | sign); return true; }
        }
        return false;
    }
    uint64_t i = 0;
    const uint64_t i0 = i;
    while (i < n && mgf_is_digit(s[i])) i++;
    const uint64_t i1 = i;
    uint64_t f0 = i1, f1 = i1;
    if (i < n && s[i] == '.') {
        i++;
        f0 = i;
        while (i < n && mgf_is_digit(s[i])) i++;
        f1 = i;
    }
    if (i1 - i0 + f1 - f0 == 0) return false;
    int64_t ex = 0;
    if (i < n && (s[i] == 'e' || s[i] == 'E')) {
        i++;
        bool eneg = false;
        if (i < n && (s[i] == '-' || s[i] == '+')) { eneg = s[i] == '-'; i++; }
        if (i == n || !mgf_is_digit(s[i])) return false;
        while (i < n && mgf_is_digit(s[i])) {
            if (ex < 1000000000000ll) ex = 10 * ex + (s[i] - '0');
            i++;
        }
        if (eneg) ex = -ex;
    }
    if (i != n) return false;
    // significant digits: the first (e0: the power of ten of the first nonzero digit), up to 19 of them in w, and whether more follow
    const uint64_t nint = i1 - i0, nall = nint + (f1 - f0);
    auto dig = [&](uint64_t k) -> uint8_t { return (uint8_t)(k < nint ? s[i0 + k] - '0' : s[f0 + k - nint] - '0'); };
    uint64_t k = 0;
    while (k < nall && dig(k) == 0) k++;
    if (k == nall) { *out = mgf_from_bits(sign); return true; }
    const int64_t e0 = (int64_t)nint - 1 - (int64_t)k;   // the place of digit k
    uint64_t w = 0;
    int taken = 0;
    uint64_t kk = k;
    for (; kk < nall && taken < 19; kk++, taken++) w = 10 * w + dig(kk);
    bool many = false;
    for (uint64_t j = kk; j < nall && !many; j++) many = dig(j) != 0;
    const int64_t q = e0 - (taken - 1) + ex;
    if (!many && w <= (1ull << 24) && q >= -10 && q <= 10) {
        const float P[11] = {1e0f, 1e1f, 1e2f, 1e3f, 1e4f, 1e5f, 1e6f, 1e7f, 1e8f, 1e9f, 1e10f};
        const float fw = (float)w;
#ifdef __CUDA_ARCH__
        const float v = q >= 0 ? __fmul_rn(fw, P[q]) : __fdiv_rn(fw, P[-q]);
        *out = __uint_as_float(__float_as_uint(v) | sign);
#else
        volatile float a = fw, b = P[q >= 0 ? q : -q];
        float v = q >= 0 ? a * b : a / b;
        uint32_t u;
        __builtin_memcpy(&u, &v, 4);
        *out = mgf_from_bits(u | sign);
#endif
        return true;
    }
    int64_t r = mgf_lemire(q, w);
    if (r >= 0 && many && r != mgf_lemire(q, w + 1)) r = -1;
    if (r < 0) {
        MgfDecimal D;
        D.nd = 0;
        D.trunc = false;
        for (uint64_t j = k; j < nall; j++) {
            const uint8_t d = dig(j);
            if (D.nd < MGF_DEC_DIGITS) D.d[D.nd++] = d;
            else if (d) D.trunc = true;
        }
        mgf_dec_trim(D);
        const int64_t dp = e0 + 1 + ex;
        D.dp = dp < -1000 ? -1000 : dp > 1000 ? 1000 : (int)dp;
        r = mgf_dec_to_f32(D);
    }
    *out = mgf_from_bits((uint32_t)r | sign);
    return true;
}

}  // namespace sb
