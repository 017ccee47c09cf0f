// glibc_math.cuh — glibc's double-precision exp(), log1p() and log10(), reproduced operation by operation.
//
// Why: rescoring (linear_discriminant.rs, kde.rs) evaluates Rust's f64::exp in every KDE kernel term, f64::ln_1p in seven LDA features and
// f64::log10 on every posterior error probability. Those are the platform libm's functions. The discriminant scores are sorted and thresholded
// (qvalue.rs), so the device evaluates the same algorithms with the same rounding sequence as glibc 2.39, in the same manner as glibc_log.cuh:
//
//   exp    sysdeps/ieee754/dbl-64/e_exp.c (ARM optimized-routines), tables in glibc_exp_data.cuh (generated from libm.so.6).
//            FMA == true:  `__exp_fma`, which x86-64 glibc's ifunc picks on every CPU with FMA + AVX2. The fusion pattern is transcribed from the
//                          disassembly of Ubuntu GLIBC 2.39's libm.so.6 (+0x79b60) and noted next to each operation.
//            FMA == false: e_exp.c as written, without contraction.
//   log1p  sysdeps/ieee754/dbl-64/s_log1p.c (fdlibm, glibc's reorganised polynomial). x86-64 glibc 2.39 ships an FMA build of it too
//          (`__log1p_fma`, libm.so.6 +0x7aff0), transcribed the same way; FMA == false is the C source as written.
//   log10  sysdeps/ieee754/dbl-64/e_log10.c: a scaling step around glibc's log(). It has no FMA build of its own (libm.so.6 +0x2b6e0: plain
//          mulsd / addsd) but calls the ifunc'd log, so variant FMA pairs it with glibc_log<FMA>.
//
// The host (sage_b200.cu: sage_b200_host_math_variant) evaluates both variants on the CPU, compares them with the host libm bit for bit and
// selects the one that matches. tests/test_ml_oracle.py checks the host evaluation against libm on millions of inputs per function, and
// tests/test_gpu_fdr.py the device evaluation.
#pragma once
#include "glibc_exp_data.cuh"
#include "glibc_log.cuh"

namespace sb { namespace gmath {
using glog::g_add; using glog::g_sub; using glog::g_mul; using glog::g_fma; using glog::g_bits; using glog::g_dbl;

#if defined(__CUDA_ARCH__)
SB_HD double g_div(double a, double b) { return __ddiv_rn(a, b); }
SB_HD uint64_t e_tab(int i) { return gexp::TAB[i]; }
#else
SB_HD double g_div(double a, double b) { volatile double r = a / b; return r; }
SB_HD uint64_t e_tab(int i) { return gexp::H_TAB[i]; }
#endif

// e_exp.c: specialcase() for |x| in [512, 1024), where the scale 2^(k/N) would leave the normal range.
template <bool FMA>
SB_HD double exp_special(double tmp, uint64_t sbits, uint64_t ki) {
    if ((ki & 0x80000000ull) == 0) {                      // k > 0
        sbits -= 1009ull << 52;
        const double scale = g_dbl(sbits);
        const double y = FMA ? g_fma(scale, tmp, scale) : g_add(scale, g_mul(scale, tmp));   // fused in __exp_fma (+0x79d1a)
        return g_mul(0x1p1009, y);
    }
    sbits += 1022ull << 52;                               // k < 0: careful rounding into the subnormal range (not fused in either build)
    const double scale = g_dbl(sbits);
    const double st = g_mul(scale, tmp);
    double y = g_add(scale, st);
    if (y < 1.0) {
        double lo = g_add(g_sub(scale, y), st);
        const double hi = g_add(1.0, y);
        lo = g_add(g_add(g_sub(1.0, hi), y), lo);
        y = g_sub(g_add(hi, lo), 1.0);
        if (y == 0.0) y = 0.0;                            // no -0.0
    }
    return g_mul(0x1p-1022, y);
}

template <bool FMA>
SB_HD double glibc_exp(double x) {
    uint32_t abstop = (uint32_t)(g_bits(x) >> 52) & 0x7ff;
    if (abstop - 0x3c9u >= 0x408u - 0x3c9u) {            // |x| < 2^-54 or |x| >= 512 or not finite
        if (abstop - 0x3c9u >= 0x80000000u) return g_add(1.0, x);
        if (abstop >= 0x409u) {
            if (g_bits(x) == 0xfff0000000000000ull) return 0.0;
            if (abstop >= 0x7ffu) return g_add(1.0, x);
            return (g_bits(x) >> 63) ? 0.0 : g_dbl(0x7ff0000000000000ull);   // __math_uflow / __math_oflow
        }
        abstop = 0;                                       // large |x|: specialcase below
    }
    double kd, r;
    if (FMA) {
        kd = g_fma(x, gexp::INVLN2N, gexp::SHIFT);        // InvLn2N * x + Shift (fused)
    } else {
        kd = g_add(g_mul(gexp::INVLN2N, x), gexp::SHIFT);
    }
    const uint64_t ki = g_bits(kd);
    kd = g_sub(kd, gexp::SHIFT);
    if (FMA) {
        r = g_fma(kd, gexp::NEGLN2LON, g_fma(kd, gexp::NEGLN2HIN, x));   // x + kd*NegLn2hiN + kd*NegLn2loN, both products fused
    } else {
        r = g_add(g_add(x, g_mul(kd, gexp::NEGLN2HIN)), g_mul(kd, gexp::NEGLN2LON));
    }
    const int idx = 2 * (int)(ki % 128);
    const uint64_t top = ki << 45;
    const double tail = g_dbl(e_tab(idx));
    const uint64_t sbits = e_tab(idx + 1) + top;
    const double r2 = g_mul(r, r);
    double tmp;
    if (FMA) {
        const double p23 = g_fma(r, gexp::C3, gexp::C2);  // C2 + r*C3
        const double p45 = g_fma(r, gexp::C5, gexp::C4);  // C4 + r*C5
        const double a = g_fma(p23, r2, g_add(r, tail));  // tail + r + r2*(..)
        tmp = g_fma(g_mul(r2, r2), p45, a);               // + r2*r2*(..)
    } else {
        tmp = g_add(g_add(g_add(tail, r), g_mul(r2, g_add(gexp::C2, g_mul(r, gexp::C3)))), g_mul(g_mul(r2, r2), g_add(gexp::C4, g_mul(r, gexp::C5))));
    }
    if (abstop == 0) return exp_special<FMA>(tmp, sbits, ki);
    const double scale = g_dbl(sbits);
    return FMA ? g_fma(scale, tmp, scale) : g_add(scale, g_mul(scale, tmp));
}

// s_log1p.c. hx / hu are the high 32-bit words, as in the source.
template <bool FMA>
SB_HD double glibc_log1p(double x) {
    constexpr double ln2_hi = 0x1.62e42fee00000p-1, ln2_lo = 0x1.a39ef35793c76p-33;
    constexpr double Lp1 = 0x1.5555555555593p-1, Lp2 = 0x1.999999997fa04p-2, Lp3 = 0x1.2492494229359p-2, Lp4 = 0x1.c71c51d8e78afp-3,
                     Lp5 = 0x1.7466496cb03dep-3, Lp6 = 0x1.39a09d078c69fp-3, Lp7 = 0x1.2f112df3e5244p-3;
    const int32_t hx = (int32_t)(g_bits(x) >> 32), ax = hx & 0x7fffffff;
    int32_t k = 1, hu = 0;
    double f = 0.0, c = 0.0, u;
    if (hx < 0x3fda827a) {                                // x < 0.41422
        if (ax >= 0x3ff00000) {                           // x <= -1
            if (x == -1.0) return g_dbl(0xfff0000000000000ull);
            return g_dbl(0x7ff8000000000000ull);           // NaN (sign / payload not reproduced)
        }
        if (ax < 0x3e200000) {                            // |x| < 2^-29
            if (ax < 0x3c900000) return x;
            return FMA ? g_fma(-g_mul(x, x), 0.5, x) : g_sub(x, g_mul(g_mul(x, x), 0.5));   // fnmadd in __log1p_fma
        }
        if (hx > 0 || hx <= (int32_t)0xbfd2bec4) { k = 0; f = x; hu = 1; }   // -0.2929 < x < 0.41422
    } else if (hx >= 0x7ff00000) {
        return g_add(x, x);
    }
    if (k != 0) {
        if (hx < 0x43400000) {
            u = g_add(1.0, x);
            hu = (int32_t)(g_bits(u) >> 32);
            k = (hu >> 20) - 1023;
            c = k > 0 ? g_sub(1.0, g_sub(u, x)) : g_sub(x, g_sub(u, 1.0));
            c = g_div(c, u);
        } else {
            u = x;
            hu = (int32_t)(g_bits(u) >> 32);
            k = (hu >> 20) - 1023;
            c = 0.0;
        }
        hu &= 0x000fffff;
        const uint64_t lo = g_bits(u) & 0xffffffffull;
        if (hu < 0x6a09e) {
            u = g_dbl(((uint64_t)(uint32_t)(hu | 0x3ff00000) << 32) | lo);
        } else {
            k += 1;
            u = g_dbl(((uint64_t)(uint32_t)(hu | 0x3fe00000) << 32) | lo);
            hu = (0x00100000 - hu) >> 2;
        }
        f = g_sub(u, 1.0);
    }
    const double hfsq = g_mul(g_mul(0.5, f), f);
    const double kd = (double)k;
    if (hu == 0) {                                        // |f| < 2^-20
        if (f == 0.0) {
            if (k == 0) return 0.0;
            if (FMA) return g_fma(kd, ln2_hi, g_fma(kd, ln2_lo, c));
            c = g_add(c, g_mul(kd, ln2_lo));
            return g_add(g_mul(kd, ln2_hi), c);
        }
        const double R = g_mul(hfsq, FMA ? g_fma(-f, 0x1.5555555555555p-1, 1.0) : g_sub(1.0, g_mul(0x1.5555555555555p-1, f)));
        if (k == 0) return g_sub(f, R);
        if (FMA) return g_fma(kd, ln2_hi, -g_sub(g_sub(R, g_fma(kd, ln2_lo, c)), f));
        return g_sub(g_mul(kd, ln2_hi), g_sub(g_sub(R, g_add(g_mul(kd, ln2_lo), c)), f));
    }
    const double s = g_div(f, g_add(2.0, f));
    const double z = g_mul(s, s);
    const double z2 = g_mul(z, z), z4 = g_mul(z2, z2), z6 = g_mul(z4, z2);
    double R;
    if (FMA) {
        const double R2 = g_fma(z, Lp3, Lp2), R3 = g_fma(z, Lp5, Lp4), R4 = g_fma(z, Lp7, Lp6);
        R = g_fma(z, Lp1, g_mul(z2, R2));                 // R1 + z2*R2 with R1 = z*Lp1 fused
        R = g_fma(z4, R3, R);
        R = g_fma(z6, R4, R);
    } else {
        const double R1 = g_mul(z, Lp1), R2 = g_add(Lp2, g_mul(z, Lp3)), R3 = g_add(Lp4, g_mul(z, Lp5)), R4 = g_add(Lp6, g_mul(z, Lp7));
        R = g_add(g_add(g_add(R1, g_mul(z2, R2)), g_mul(z4, R3)), g_mul(z6, R4));
    }
    const double sr = g_mul(s, g_add(hfsq, R));
    if (k == 0) return g_sub(f, g_sub(hfsq, sr));
    if (FMA) return g_fma(kd, ln2_hi, -g_sub(g_sub(hfsq, g_add(g_fma(kd, ln2_lo, c), sr)), f));
    return g_sub(g_mul(kd, ln2_hi), g_sub(g_sub(hfsq, g_add(sr, g_add(g_mul(kd, ln2_lo), c))), f));
}

// e_log10.c around glibc's log().
template <bool FMA>
SB_HD double glibc_log10(double x) {
    constexpr double ivln10 = 0x1.bcb7b1526e50ep-2, log10_2hi = 0x1.34413509f6000p-2, log10_2lo = 0x1.9fef311f12b36p-42;
    int64_t hx = (int64_t)g_bits(x);
    int64_t k = -1023;
    if (hx < 0x0010000000000000ll) {                      // zero, subnormal or negative
        if ((hx & 0x7fffffffffffffffll) == 0) return g_dbl(0xfff0000000000000ull);
        if (hx < 0) return g_dbl(0x7ff8000000000000ull);
        k -= 54;
        hx = (int64_t)g_bits(g_mul(x, 0x1p54));
    }
    if ((uint64_t)hx > 0x7fefffffffffffffull) return g_add(x, x);
    k += hx >> 52;
    const int64_t i = (int64_t)((uint64_t)k >> 63);
    const double y = (double)(k + i);
    const double xs = g_dbl(((uint64_t)hx & 0x000fffffffffffffull) | ((uint64_t)(0x3ff - i) << 52));
    const double z = g_add(g_mul(glog::glibc_log<FMA>(xs), ivln10), g_mul(y, log10_2lo));
    return g_add(z, g_mul(y, log10_2hi));
}

// function: 0 exp, 1 log1p, 2 log10. variant: 0 the FMA builds, 1 the uncontracted ones (glibc_log.cuh numbering).
SB_HD double eval(int function, int variant, double x) {
    const bool fma = variant != 1;
    switch (function) {
        case 0: return fma ? glibc_exp<true>(x) : glibc_exp<false>(x);
        case 1: return fma ? glibc_log1p<true>(x) : glibc_log1p<false>(x);
        default: return fma ? glibc_log10<true>(x) : glibc_log10<false>(x);
    }
}

}}  // namespace sb::gmath
