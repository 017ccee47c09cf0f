// SpectrumProcessor::process for spectra that are not MS2 (spectrum.rs:338-412): mass = mz - PROTON, a stable sort by mass.total_cmp that
// carries intensities (and, for MS1 with mobility, mobilities) with their peak, and the f32 left fold of the sorted intensities (the TIC).
// Every peak is kept. Level-2 spectra are k_process_ms2's (kernels.cuh); the host code of sage_b200_process_raw routes them.
//
//   k_raw_process       one CTA per spectrum: picks the size class from the input and handles the first two
//                         sorted    (mass non-decreasing in total_cmp order): one coalesced pass, no sort
//                         small     (unsorted, <= RAW_SMEM_PEAKS): a bitonic sort of (total_cmp key, input index) in shared memory
//                         large     (unsorted, more peaks): keys and input indices are written out as one segment of
//                                   cub::DeviceSegmentedSort::StableSortPairs, run by the host
//   k_raw_gather_large  one CTA per large spectrum: writes the sorted segment out, then the TIC
//   k_raw_compact_ms2   one CTA per level-2 spectrum: copies k_process_ms2's kept peaks to their compacted place
//
// Exactness (DESIGN.md §16): outputs carry the bits the reference computes on x86-64, NaNs included. Device f32 arithmetic returns the
// canonical NaN, so NaN results are formed explicitly: raw_mass() keeps a NaN m/z's sign and payload, quieted, as SSE's subss does; tic_add()
// keeps the accumulator's NaN when both operands are NaN (addss with the accumulator as destination), else the NaN operand quieted, and
// returns x86's default NaN 0xFFC00000 for inf + -inf. The fold starts at +0.0.
#pragma once
#include <stdint.h>

#include "device_common.cuh"   // PROTON, f32_key

namespace sb {

constexpr uint32_t RAW_SMEM_PEAKS = 4096;   // largest unsorted spectrum sorted in shared memory: 4096 * 12 B = 48 KB, the no-opt-in limit
constexpr int RAW_THREADS = 256;
constexpr uint32_t X86_DEFAULT_NAN = 0xFFC00000u;

__device__ __forceinline__ float raw_quiet(float x) { return __uint_as_float(__float_as_uint(x) | 0x00400000u); }

// (mz - PROTON) * 1.0 (spectrum.rs:381; MS1 with mobility omits the * 1.0, spectrum.rs:350: the same f32)
__device__ __forceinline__ float raw_mass(float mz) { return isnan(mz) ? raw_quiet(mz) : __fsub_rn(mz, PROTON); }

__device__ __forceinline__ float tic_add(float t, float x) {
    const float r = __fadd_rn(t, x);
    if (!isnan(r)) return r;
    if (isnan(t)) return t;              // already quiet: it came out of an earlier step
    if (isnan(x)) return raw_quiet(x);
    return __uint_as_float(X86_DEFAULT_NAN);
}

// total_cmp order as an unsigned key, and back (f32_key's bit flip keeps the sign bit, so it is its own inverse)
__device__ __forceinline__ uint32_t raw_ukey(float x) { return (uint32_t)f32_key(x) ^ 0x80000000u; }
__device__ __forceinline__ float raw_unkey(uint32_t u) { return __int_as_float(f32_key(__int_as_float((int)(u ^ 0x80000000u)))); }

// The TIC of n intensities, folded in order by all 32 lanes of one warp (each lane holds the same value). Each step's 32 loads are issued
// together, one step ahead of the fold, so the only dependent chain is the additions.
template <class Load>
__device__ __forceinline__ float raw_fold(uint32_t n, Load ld) {
    const uint32_t lane = threadIdx.x & 31;
    float t = 0.0f;
    float v = lane < n ? ld(lane) : 0.0f;
    for (uint32_t base = 0; base < n; base += 32) {
        const float next = base + 32 + lane < n ? ld(base + 32 + lane) : 0.0f;
        if (n - base >= 32) {
#pragma unroll
            for (int k = 0; k < 32; k++) t = tic_add(t, __shfl_sync(0xffffffffu, v, k));
        } else {
            for (uint32_t k = 0; k < n - base; k++) t = tic_add(t, __shfl_sync(0xffffffffu, v, k));
        }
        v = next;
    }
    return t;
}

struct RawArgs {
    uint32_t n;
    const uint64_t* in_off;     // [n + 1], relative to the uploaded peaks
    const float *mz, *intensity, *mobility;   // mobility: NULL = no spectrum of the batch has one
    const uint8_t* level;       // NULL = every spectrum is MS1
    const uint64_t* out_off;    // [n + 1] compacted
    float *out_mass, *out_int, *out_mob, *out_tic;   // out_mob: NaN where the spectrum has no mobilities; out_mob / out_tic may be NULL
    const uint32_t* large_slot; // [n] slot of a spectrum with more than RAW_SMEM_PEAKS peaks, NULL when there is none
    int *seg_begin, *seg_end;   // [slots] segments of the large sort (empty for a sorted spectrum)
    uint32_t *sort_key, *sort_val;   // [peaks] keys and input indices of the large unsorted spectra, at their input positions
};

__device__ __forceinline__ bool raw_has_mob(const RawArgs& a, uint32_t lev) { return a.mobility && lev == 1; }

__global__ void __launch_bounds__(RAW_THREADS) k_raw_process(RawArgs a) {
    extern __shared__ __align__(16) unsigned char raw_smem[];
    const uint32_t s = blockIdx.x, tid = threadIdx.x;
    const uint32_t lev = a.level ? a.level[s] : 1u;
    if (lev == 2) return;
    const uint64_t p0 = a.in_off[s], o0 = a.out_off[s];
    const uint32_t np = (uint32_t)(a.in_off[s + 1] - p0);
    const bool mob = raw_has_mob(a, lev);
    const float* mz = a.mz + p0;
    const float* in = a.intensity + p0;
    bool unsorted = false;
    for (uint32_t i = tid; i + 1 < np; i += RAW_THREADS) unsorted |= raw_ukey(raw_mass(mz[i])) > raw_ukey(raw_mass(mz[i + 1]));
    unsorted = __syncthreads_or(unsorted);
    if (!unsorted) {
        for (uint32_t i = tid; i < np; i += RAW_THREADS) {
            a.out_mass[o0 + i] = raw_mass(mz[i]);
            a.out_int[o0 + i] = in[i];
            if (a.out_mob) a.out_mob[o0 + i] = mob ? a.mobility[p0 + i] : __uint_as_float(0x7FC00000u);
        }
        if (np > RAW_SMEM_PEAKS && tid == 0) a.seg_begin[a.large_slot[s]] = a.seg_end[a.large_slot[s]] = 0;
        if (tid < 32) {
            const float t = raw_fold(np, [&](uint32_t i) { return in[i]; });
            if (tid == 0 && a.out_tic) a.out_tic[s] = t;
        }
        return;
    }
    if (np > RAW_SMEM_PEAKS) {
        for (uint32_t i = tid; i < np; i += RAW_THREADS) { a.sort_key[p0 + i] = raw_ukey(raw_mass(mz[i])); a.sort_val[p0 + i] = i; }
        if (tid == 0) { a.seg_begin[a.large_slot[s]] = (int)p0; a.seg_end[a.large_slot[s]] = (int)(p0 + np); }
        return;
    }
    uint32_t n2 = 1;
    while (n2 < np) n2 <<= 1;
    uint64_t* keys = reinterpret_cast<uint64_t*>(raw_smem);   // [n2] (total_cmp key, input index): the index makes the sort stable
    float* sint = reinterpret_cast<float*>(keys + n2);          // [np] sorted intensities, for the fold
    for (uint32_t i = tid; i < n2; i += RAW_THREADS) keys[i] = i < np ? ((uint64_t)raw_ukey(raw_mass(mz[i])) << 32) | i : ~0ull;
    __syncthreads();
    for (uint32_t k = 2; k <= n2; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = tid; i < n2; i += RAW_THREADS) {
                const uint32_t l = i ^ j;
                if (l > i) {
                    const uint64_t x = keys[i], y = keys[l];
                    if ((x > y) == ((i & k) == 0)) { keys[i] = y; keys[l] = x; }
                }
            }
            __syncthreads();
        }
    }
    for (uint32_t i = tid; i < np; i += RAW_THREADS) {
        const uint64_t key = keys[i];
        const uint32_t src = (uint32_t)key;
        const float v = in[src];
        sint[i] = v;
        a.out_mass[o0 + i] = raw_unkey((uint32_t)(key >> 32));
        a.out_int[o0 + i] = v;
        if (a.out_mob) a.out_mob[o0 + i] = mob ? a.mobility[p0 + src] : __uint_as_float(0x7FC00000u);
    }
    __syncthreads();
    if (tid < 32) {
        const float t = raw_fold(np, [&](uint32_t i) { return sint[i]; });
        if (tid == 0 && a.out_tic) a.out_tic[s] = t;
    }
}

// After the segmented sort: sort_key / sort_val hold each large unsorted spectrum's keys and input indices in total_cmp order, stable.
__global__ void __launch_bounds__(RAW_THREADS) k_raw_gather_large(RawArgs a, const uint32_t* large_ids) {
    const uint32_t slot = blockIdx.x, tid = threadIdx.x;
    if (a.seg_end[slot] == a.seg_begin[slot]) return;   // sorted: k_raw_process wrote it
    const uint32_t s = large_ids[slot];
    const uint32_t lev = a.level ? a.level[s] : 1u;
    const uint64_t p0 = a.in_off[s], o0 = a.out_off[s];
    const uint32_t np = (uint32_t)(a.in_off[s + 1] - p0);
    const bool mob = raw_has_mob(a, lev);
    for (uint32_t i = tid; i < np; i += RAW_THREADS) {
        const uint32_t src = a.sort_val[p0 + i];
        a.out_mass[o0 + i] = raw_unkey(a.sort_key[p0 + i]);
        a.out_int[o0 + i] = a.intensity[p0 + src];
        if (a.out_mob) a.out_mob[o0 + i] = mob ? a.mobility[p0 + src] : __uint_as_float(0x7FC00000u);
    }
    __syncthreads();   // the fold reads what the whole CTA wrote (plain loads: the data was written by this kernel)
    if (tid < 32) {
        const float* oi = a.out_int + o0;
        const float t = raw_fold(np, [&](uint32_t i) { return oi[i]; });
        if (tid == 0 && a.out_tic) a.out_tic[s] = t;
    }
}

// k_process_ms2 ran on the level-2 spectra gathered contiguously (ms2_off): copy each one's kept peaks to its compacted place.
__global__ void __launch_bounds__(RAW_THREADS) k_raw_compact_ms2(uint32_t n2, const uint32_t* ms2_ids, const uint32_t* ms2_off, const uint32_t* ms2_cnt,
                                                                 const float* ms2_mass, const float* ms2_int, const float* ms2_tic, const uint64_t* out_off,
                                                                 float* out_mass, float* out_int, float* out_mob, float* out_tic) {
    const uint32_t j = blockIdx.x;
    if (j >= n2) return;
    const uint32_t s = ms2_ids[j], q0 = ms2_off[j], cnt = ms2_cnt[j];
    const uint64_t o0 = out_off[s];
    for (uint32_t i = threadIdx.x; i < cnt; i += RAW_THREADS) {
        out_mass[o0 + i] = ms2_mass[q0 + i];
        out_int[o0 + i] = ms2_int[q0 + i];
        if (out_mob) out_mob[o0 + i] = __uint_as_float(0x7FC00000u);
    }
    if (threadIdx.x == 0 && out_tic) out_tic[s] = ms2_tic[j];
}

// Gathers the level-2 spectra's raw peaks contiguously for k_process_ms2.
__global__ void __launch_bounds__(RAW_THREADS) k_raw_gather_ms2(uint32_t n2, const uint32_t* ms2_ids, const uint32_t* ms2_off, const uint64_t* in_off,
                                                                const float* mz, const float* intensity, float* ms2_mz, float* ms2_in) {
    const uint32_t j = blockIdx.x;
    if (j >= n2) return;
    const uint64_t p0 = in_off[ms2_ids[j]];
    const uint32_t q0 = ms2_off[j], np = ms2_off[j + 1] - q0;
    for (uint32_t i = threadIdx.x; i < np; i += RAW_THREADS) { ms2_mz[q0 + i] = mz[p0 + i]; ms2_in[q0 + i] = intensity[p0 + i]; }
}

// out_count[s] = peaks kept by spectrum s: every peak below level 2 and above, k_process_ms2's count at level 2. [n] is 0 for the scan.
__global__ void k_raw_counts(uint32_t n, const uint64_t* in_off, const uint8_t* level, const uint32_t* ms2_pos, const uint32_t* ms2_cnt, uint64_t* out_count) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s > n) return;
    out_count[s] = s == n ? 0 : level[s] == 2 ? ms2_cnt[ms2_pos[s]] : in_off[s + 1] - in_off[s];
}

}  // namespace sb
