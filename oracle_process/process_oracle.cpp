// CPU oracle of SpectrumProcessor::process for spectra that are not MS2 (spectrum.rs:338-412), written from the Rust as plainly as it reads:
// (mz - PROTON) * 1.0 (MS1 with mobility: mz - PROTON), a stable sort by f32::total_cmp, and `intensities.iter().sum::<f32>()` as a left
// fold from +0.0. Compiled without FMA contraction or fast-math, so each operation is one x86-64 SSE instruction with its NaN rules
// (a NaN operand's payload comes through quieted; of two NaNs, the fold's accumulator wins). Level 2 is process_ms2 of oracle/sage_oracle.cpp,
// composed in process_oracle.py.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <numeric>
#include <vector>

static const float PROTON = 1.0072764f;   // mass.rs:5

static int32_t total_cmp_key(float x) {
    int32_t b;
    memcpy(&b, &x, 4);
    return b ^ (int32_t)(((uint32_t)(b >> 31)) >> 1);
}

// One spectrum of np peaks of level `level`; mobility may be NULL. Writes np masses, intensities and (with_mobility) mobilities; returns the TIC.
extern "C" float po_process_other(const float* mz, const float* intensity, const float* mobility, uint64_t np, uint32_t level, float* out_mass,
                                  float* out_int, float* out_mob) {
    const bool with_mobility = level == 1 && mobility != nullptr;
    std::vector<float> mass(np);
    for (uint64_t i = 0; i < np; i++) mass[i] = with_mobility ? mz[i] - PROTON : (mz[i] - PROTON) * 1.0f;
    std::vector<uint64_t> order(np);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](uint64_t a, uint64_t b) { return total_cmp_key(mass[a]) < total_cmp_key(mass[b]); });
    for (uint64_t i = 0; i < np; i++) {
        out_mass[i] = mass[order[i]];
        out_int[i] = intensity[order[i]];
        if (with_mobility) out_mob[i] = mobility[order[i]];
    }
    float tic = 0.0f;
    for (uint64_t i = 0; i < np; i++) tic = tic + out_int[i];
    return tic;
}
