// CPU check of sage_b200/csrc/glibc_math.cuh (compiled by tests/test_ml_oracle.py with g++): evaluates both variants of glibc's exp(), log1p()
// and log10() exactly as the device does and counts, per function, the inputs on which each variant differs from this host's libm.
#include "glibc_math.cuh"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>

static double bits(uint64_t u) { double x; memcpy(&x, &u, 8); return x; }

int main(int argc, char** argv) {
    std::mt19937_64 rng(2024);
    const long n = argc > 1 ? atol(argv[1]) : 1000000;
    long bad[3][2] = {{0, 0}, {0, 0}, {0, 0}}, tested[3] = {0, 0, 0};
    auto chk = [&](int f, double x) {
        volatile double vx = x;
        const double ref = f == 0 ? std::exp(vx) : f == 1 ? std::log1p(vx) : std::log10(vx);
        for (int v = 0; v < 2; v++) {
            const double got = sb::gmath::eval(f, v, x);
            if (memcmp(&got, &ref, 8) && !(got != got && ref != ref)) bad[f][v]++;
        }
        tested[f]++;
    };
    for (long i = 0; i < n; i++) {
        const uint64_t u = rng();
        const double unit = (double)(u >> 11) * 0x1p-53;
        double x;
        switch (i % 8) {
            case 0: x = bits(u); break;                                           // any bit pattern: every exponent, both signs, NaN, inf
            case 1: x = bits(u & 0x800fffffffffffffull); break;                   // subnormals of both signs
            case 2: x = -0.5 * std::ldexp(unit, (int)(u & 63) - 20) * std::ldexp(unit, (int)(u & 63) - 20); break;   // KDE arguments -0.5 u^2
            case 3: x = (unit - 0.5) * 1500.0; break;                             // exp's overflow / subnormal special cases
            case 4: x = (unit - 0.5) * 0x1p-20; break;                            // near 0 (log1p's small-|x| branches)
            case 5: x = unit * 2.0 - 1.0; break;                                  // (-1, 1): log1p's k == 0 range
            case 6: x = std::ldexp(unit, (int)((u >> 3) & 127) - 40); break;      // positive, many binades (features, PEPs)
            default: x = 1.0 + (unit - 0.5) * 0x1p-18; break;                     // near 1
        }
        for (int f = 0; f < 3; f++) chk(f, x);
    }
    const double sp[] = {0.0, -0.0, -1.0, 1.0, INFINITY, -INFINITY, NAN, 0x1p-1074, -0x1p-1074, 0x1.fffffffffffffp1023, 709.782712893384, 709.79, -745.1332191019411,
                         -745.14, -708.4, 512.0, -512.0, 1024.0, -1024.0, 0x1p-54, 0x1p-29, 0.41422, -0.2929, 1e300, 0x1p53, 0x1p54, 0.1, 10.0, 1e-308};
    for (double x : sp)
        for (int f = 0; f < 3; f++) chk(f, x);
    printf("n=%ld", tested[0]);
    const char* name[3] = {"exp", "log1p", "log10"};
    for (int f = 0; f < 3; f++) printf(" %s_variant0=%ld %s_variant1=%ld", name[f], bad[f][0], name[f], bad[f][1]);
    printf("\n");
    return 0;
}
