// lfq.cuh — sm_90a kernels of label-free quantification (lfq.rs, isotopes.rs).
//
//   k_lfq_first_row / k_lfq_flag   the per-peptide "first kept row wins" of build_feature_map                 lfq.rs:100-131
//   k_lfq_isotopes                 peptide_isotopes(carbon, sulfur)                                              isotopes.rs:1-50
//   k_lfq_expand                   charge x isotope x {forward, decoy} PrecursorRange expansion                   lfq.rs:134-170
//   k_lfq_page_keys / k_lfq_gather the RT sort, 16384-entry pages, per-page mass_lo sort and min_rts            lfq.rs:172-184
//   k_lfq_trace<EMIT>              rt_slice + mass_lookup / mass_mobility_lookup + Grid::add_entry, one warp per MS1 spectrum
//                                  (count pass, then emit pass writing (cell, value) in the defined sequence order)   lfq.rs:239-287, 538-550, 648-686
//   k_lfq_fold                     each cell's run of the stably cell-sorted contributions, folded in order onto the stored f64
//   k_lfq_integrate                summarize_traces, find/apply_time_warps, scores, integrate: one CTA per touched grid   lfq.rs:347-610
//
// Every f32/f64 operation is a separately rounded IEEE operation in the reference's association order (the library builds with
// -fmad=false). The only libm function evaluated on the device is acos (CUDA's), see DESIGN.md §9.
#pragma once

#include "device_common.cuh"
#include "kernels.cuh"   // f32_ukey
#include "../../include/sage_b200.h"

namespace sb {

constexpr float LFQ_RT_TOL = 0.0050f;   // lfq.rs:15
constexpr int LFQ_K_WIDTH = 10;         // lfq.rs:17
constexpr int LFQ_GRID = 100;           // lfq.rs:21
constexpr int LFQ_ISO = 3;              // lfq.rs:23
constexpr uint32_t LFQ_PAGE = 16 * 1024;  // lfq.rs:176
constexpr int LFQ_SLACK = 75;           // lfq.rs:350
constexpr int LFQ_THREADS = 256;

// ------------------------------------------------------------------------------------------------ feature map build
__global__ void k_lfq_first_row(uint64_t n, const uint32_t* __restrict__ pep, const float* __restrict__ q, const int32_t* __restrict__ label, float q_max,
                                uint32_t* __restrict__ first_row) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && q[i] <= q_max && label[i] == 1) atomicMin(&first_row[pep[i]], (uint32_t)i);
}

__global__ void k_lfq_flag(uint64_t n, const uint32_t* __restrict__ first_row, uint8_t* __restrict__ flag) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flag[i] = first_row[i] != 0xFFFFFFFFu;
}

// isotopes.rs:2-10, the unrolled 4-term convolution
__device__ __forceinline__ void lfq_convolve4(const float* a, const float* b, float* c) {
    c[0] = a[0] * b[0];
    c[1] = a[0] * b[1] + a[1] * b[0];
    c[2] = a[0] * b[2] + a[1] * b[1] + a[2] * b[0];
    c[3] = a[0] * b[3] + a[1] * b[2] + a[2] * b[1] + a[3] * b[0];
}

// powi(x, k) for k = 0..3 as LLVM expands it (x, x*x, x*(x*x))
__device__ __forceinline__ float lfq_powi(float x, int k) {
    return k == 0 ? 1.0f : k == 1 ? x : k == 2 ? x * x : x * (x * x);
}

// peptide_isotopes (isotopes.rs:12-50). exp_c[c] = expf(-(c * 0.011f)), exp_s33[s] = expf(-(s * 0.0076f)), exp_s35[s] = expf(-(s * 0.044f)), all
// from the host libm.
__global__ void k_lfq_isotopes(uint32_t n, const uint16_t* __restrict__ carbon, const uint16_t* __restrict__ sulfur, const float* __restrict__ exp_c,
                               const float* __restrict__ exp_s33, const float* __restrict__ exp_s35, float* __restrict__ dist) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float fact[4] = {1.0f, 1.0f, 2.0f, 6.0f};
    const uint16_t cc = carbon[i], ss = sulfur[i];
    const float lc = (float)cc * 0.011f, l33 = (float)ss * 0.0076f, l35 = (float)ss * 0.044f;
    float c13[4], s33[4], s35[4], s[4], c[4];
    for (int k = 0; k < 4; k++) c13[k] = lfq_powi(lc, k) * exp_c[cc] / fact[k];
    for (int k = 0; k < 4; k++) s33[k] = lfq_powi(l33, k) * exp_s33[ss] / fact[k];
    s35[0] = 1.0f * exp_s35[ss];
    s35[1] = 0.0f;
    s35[2] = l35 * exp_s35[ss];
    s35[3] = 0.0f;
    lfq_convolve4(s33, s35, s);
    lfq_convolve4(c13, s, c);
    const float mx = fmaxf(fmaxf(c[0], c[1]), c[2]);
    for (int k = 0; k < 3; k++) dist[3 * i + k] = c[k] / mx;
}

// One thread per (slot, charge, isotope): the forward and the decoy range, at pre-sort position ((slot * n_charges + charge) * 3 + isotope) * 2 + decoy,
// i.e. ascending (PeptideIx, charge, isotope, forward before decoy).
__global__ void k_lfq_expand(uint32_t n_slots, uint32_t n_charges, uint32_t min_charge, float ppm, float mob_pct, const uint32_t* __restrict__ slot_pep,
                             const uint32_t* __restrict__ first_row, const float* __restrict__ aligned_rt, const float* __restrict__ calcmass,
                             const uint32_t* __restrict__ file_id, const float* __restrict__ ims, sage_b200_lfq_range* __restrict__ out,
                             uint32_t* __restrict__ rt_key, uint32_t* __restrict__ idx, uint32_t* __restrict__ slot_file) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_slots * n_charges * LFQ_ISO) return;
    const uint32_t iso = t % LFQ_ISO, ch = (t / LFQ_ISO) % n_charges, slot = t / (LFQ_ISO * n_charges);
    const uint32_t pep = slot_pep[slot], row = first_row[pep];
    const float rt = aligned_rt[row], mono = calcmass[row];
    if (ch == 0 && iso == 0) slot_file[slot] = file_id[row];
    float mob_lo, mob_hi;
    tol_bounds(Tol{1, -mob_pct, mob_pct}, ims[row], mob_lo, mob_hi);
    const uint32_t charge = min_charge + ch;
    const float mass = (mono + (float)iso * NEUTRON) / (float)charge;
    sage_b200_lfq_range r;
    r.rt = rt;
    tol_bounds(Tol{0, -ppm, ppm}, mass, r.mass_lo, r.mass_hi);
    r.mobility_lo = mob_lo;
    r.mobility_hi = mob_hi;
    r.peptide = pep;
    r.file_id = file_id[row];
    r.charge = (uint8_t)charge;
    r.isotope = (uint8_t)iso;
    r.decoy = 0;
    r._pad = 0;
    out[2 * t] = r;
    r.rt = fmaxf(rt - LFQ_RT_TOL * 2.0f, 0.0f);
    tol_bounds(Tol{0, -ppm, ppm}, mass + 11.06f, r.mass_lo, r.mass_hi);
    r.decoy = 1;
    out[2 * t + 1] = r;
    rt_key[2 * t] = f32_ukey(out[2 * t].rt);
    rt_key[2 * t + 1] = f32_ukey(r.rt);
    idx[2 * t] = 2 * t;
    idx[2 * t + 1] = 2 * t + 1;
}

// After the stable RT sort (perm = pre-sort indices in RT order): key (page, mass_lo) for the stable per-page mass sort, and min_rts.
__global__ void k_lfq_page_keys(uint32_t n, const uint32_t* __restrict__ perm, const sage_b200_lfq_range* __restrict__ pre, uint64_t* __restrict__ key,
                                float* __restrict__ min_rts) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const sage_b200_lfq_range& r = pre[perm[i]];
    key[i] = ((uint64_t)(i / LFQ_PAGE) << 32) | f32_ukey(r.mass_lo);
    if (i % LFQ_PAGE == 0) min_rts[i / LFQ_PAGE] = r.rt;
}

// Final layout, and the grid each range feeds: (slot, decoy) when charge states are combined, else (slot, charge, decoy).
__global__ void k_lfq_gather(uint32_t n, uint32_t n_charges, int combine, const uint32_t* __restrict__ perm, const sage_b200_lfq_range* __restrict__ pre,
                             sage_b200_lfq_range* __restrict__ ranges, uint32_t* __restrict__ grid_of) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t j = perm[i], decoy = j & 1, sc = j / (2 * LFQ_ISO);   // sc = slot * n_charges + charge
    ranges[i] = pre[j];
    grid_of[i] = (combine ? sc / n_charges : sc) * 2 + decoy;
}

// ------------------------------------------------------------------------------------------------ tracing
struct LfqTraceArgs {
    uint32_t n_spectra;
    const uint64_t* peak_off;   // n+1, relative to the chunk
    const float* masses;
    const float* intensities;
    const float* mobilities;    // nullptr: no mobility filter
    const uint32_t* file_id;
    const float* sst;
    const sage_b200_alignment* align;
    const sage_b200_lfq_range* ranges;
    const uint32_t* grid_of;
    uint32_t n_ranges, n_pages, n_files;
    const float* min_rts;
    uint64_t* counts;           // count pass: matches per peak
    const uint64_t* offsets;    // emit pass: exclusive scan of counts
    uint64_t* cell;             // emit pass: 2 per match
    double* value;
};

// FeatureMap::quantify's per-spectrum closure. One warp per spectrum, peaks lane-strided; each lane visits its peak's entries in the reference's
// order (page, then position in the page), so the emit pass writes contributions in (spectrum, peak, entry, lo/hi) order.
template <bool EMIT>
__global__ void __launch_bounds__(LFQ_THREADS) k_lfq_trace(LfqTraceArgs a) {
    const uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (s >= a.n_spectra) return;
    const sage_b200_alignment al = a.align[a.file_id[s]];
    const float rt = (a.sst[s] / al.max_rt) * al.slope + al.intercept;
    const float min_rt = rt - LFQ_RT_TOL, max_rt = rt + LFQ_RT_TOL;
    uint32_t page_lo, page_hi;
    {
        const int klo = f32_key(min_rt), khi = f32_key(max_rt);
        binary_search_slice(
            a.n_pages, [&](uint32_t i) { return f32_key(a.min_rts[i]) < klo; }, [&](uint32_t i) { return f32_key(a.min_rts[i]) <= khi; }, page_lo, page_hi);
    }
    const uint32_t file = a.file_id[s];
    const float rt_step = (LFQ_RT_TOL * 2.0f) / (float)LFQ_GRID;
    for (uint64_t p = a.peak_off[s] + lane; p < a.peak_off[s + 1]; p += 32) {
        const float mass = a.masses[p], inten = a.intensities[p];
        const bool has_mob = a.mobilities != nullptr;
        const float mob = has_mob ? a.mobilities[p] : 0.0f;
        uint64_t out = EMIT ? a.offsets[p] : 0;
        uint64_t cnt = 0;
        const int klo = f32_key(mass - 0.1f), khi = f32_key(mass + 0.1f);
        for (uint32_t page = page_lo; page < page_hi; page++) {
            const uint32_t left = page * LFQ_PAGE, right = min(left + LFQ_PAGE, a.n_ranges);
            const sage_b200_lfq_range* slice = a.ranges + left;
            uint32_t il, ir;
            binary_search_slice(
                right - left, [&](uint32_t i) { return f32_key(slice[i].mass_lo) < klo; }, [&](uint32_t i) { return f32_key(slice[i].mass_lo) <= khi; }, il,
                ir);
            for (uint32_t i = il; i < ir; i++) {
                const sage_b200_lfq_range r = slice[i];
                if (!(r.rt <= max_rt && r.rt >= min_rt && mass >= r.mass_lo && mass <= r.mass_hi)) continue;
                if (has_mob && !(r.mobility_hi >= mob && r.mobility_lo <= mob)) continue;
                if (!EMIT) { cnt++; continue; }
                // Grid::add_entry (lfq.rs:538-550); the grid was created by an entry with this rt (all ranges of one grid share it)
                const float rt_min = r.rt - LFQ_RT_TOL;
                const float x = floorf((rt - rt_min) / rt_step);
                uint32_t bin_lo = !(x > 0.0f) ? 0u : (x >= 4294967295.0f ? 0xFFFFFFFFu : (uint32_t)x);   // `as usize`: NaN / negative -> 0
                bin_lo = min(bin_lo, (uint32_t)(LFQ_GRID - 1));
                const uint32_t bin_hi = min(bin_lo + 1, (uint32_t)(LFQ_GRID - 1));
                const float bin_lo_rt = (float)bin_lo * rt_step + rt_min;
                const float interp = (rt - bin_lo_rt) / rt_step;
                const uint64_t row = ((uint64_t)a.grid_of[left + i] * a.n_files + file) * LFQ_ISO + r.isotope;
                a.cell[2 * out] = row * LFQ_GRID + bin_lo;
                a.value[2 * out] = (double)((1.0f - interp) * inten);
                a.cell[2 * out + 1] = row * LFQ_GRID + bin_hi;
                a.value[2 * out + 1] = (double)(interp * inten);
                out++;
            }
        }
        if (!EMIT) a.counts[p] = cnt;
    }
}

// Contributions sorted stably by cell: the first thread of each run folds the run, in order, onto the stored value.
__global__ void k_lfq_fold(uint64_t n, const uint64_t* __restrict__ cell, const double* __restrict__ value, double* __restrict__ grids,
                           uint8_t* __restrict__ touched, uint64_t cells_per_grid) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || (i > 0 && cell[i - 1] == cell[i])) return;
    const uint64_t c = cell[i];
    double acc = grids[c];
    for (uint64_t j = i; j < n && cell[j] == c; j++) acc = acc + value[j];
    grids[c] = acc;
    touched[c / cells_per_grid] = 1;
}

// ------------------------------------------------------------------------------------------------ integration
struct LfqIntegrateArgs {
    uint32_t n;                   // touched grids
    const uint32_t* grid_ids;     // ascending
    const double* grids;
    const float* slot_dist;       // 3 per slot
    const uint32_t* slot_file;    // reference_file_id
    const double* consts;         // gaussian_kernel(0.5, 10) [10], then (1 - |rt - 50| / 50).powf(0.33) for rt = 0..99 [100]
    uint32_t n_files, n_charges;
    int combine, peak_scoring, integration;
    double spectral_angle;
    uint8_t* present;
    uint32_t* rt;
    double* sa;
    double* score;
    double* areas;                // n * n_files
};

__host__ __device__ constexpr size_t lfq_integrate_smem(uint32_t n_files) {
    return sizeof(double) * (2 * (size_t)LFQ_GRID * n_files + (2 * LFQ_SLACK + 1) + 3 * LFQ_GRID) + sizeof(int) * (n_files + 4);
}

// convolve (lfq.rs:632-646) at one index, with the even 10-tap kernel's index arithmetic as written
__device__ __forceinline__ double lfq_convolve_at(const double* __restrict__ row, const double* __restrict__ k, int idx) {
    const int n = LFQ_K_WIDTH - LFQ_K_WIDTH / 2;
    const int ks = max(LFQ_K_WIDTH - (n + idx), 0), ws = max(idx - (n - 1), 0);
    const int len = min(LFQ_GRID - ws, LFQ_K_WIDTH - ks);
    double acc = 0.0;
    for (int t = 0; t < len; t++) acc = acc + row[ws + t] * k[ks + t];
    return acc;
}

__global__ void __launch_bounds__(LFQ_THREADS) k_lfq_integrate(LfqIntegrateArgs a) {
    extern __shared__ __align__(16) unsigned char lfq_smem[];
    const uint32_t F = a.n_files;
    double* sa = reinterpret_cast<double*>(lfq_smem);              // [F][100] spectral_angle
    double* dot = sa + (size_t)F * LFQ_GRID;                       // [F][100] dot_product
    double* wd = dot + (size_t)F * LFQ_GRID;                       // [151] dot of one file at every shift
    double* spectral = wd + (2 * LFQ_SLACK + 1);                   // [100]
    double* inten = spectral + LFQ_GRID;                           // [100]
    double* scores = inten + LFQ_GRID;                             // [100]
    int* warps = reinterpret_cast<int*>(scores + LFQ_GRID);        // [F]
    int* win = warps + F;                                          // present, best rt, left, right
    const uint32_t t = blockIdx.x;
    const uint32_t g = a.grid_ids[t];
    const uint32_t slot = a.combine ? g / 2 : g / 2 / a.n_charges;
    const double* grid = a.grids + (size_t)g * F * LFQ_ISO * LFQ_GRID;
    const double* kern = a.consts;
    float dist[LFQ_ISO];
    for (int i = 0; i < LFQ_ISO; i++) dist[i] = a.slot_dist[3 * slot + i];
    const double ss_dist = (double)sqrtf(dist[0] * dist[0] + dist[1] * dist[1] + dist[2] * dist[2]);
    const uint32_t ref = a.slot_file[slot];

    // summarize_traces (lfq.rs:558-610)
    for (uint32_t e = threadIdx.x; e < F * LFQ_GRID; e += blockDim.x) {
        const uint32_t f = e / LFQ_GRID, col = e % LFQ_GRID;
        double d = 0.0, ss = 0.0;
        for (int iso = 0; iso < LFQ_ISO; iso++) {
            const double c = lfq_convolve_at(grid + ((size_t)f * LFQ_ISO + iso) * LFQ_GRID, kern, (int)col);
            d = d + c * (double)dist[iso];
            ss = ss + c * c;
        }
        const double sim = ss > 0.0 ? d / (sqrt(ss) * ss_dist) : 0.0;
        sa[e] = 1.0 - 2.0 * acos(sim) / 3.141592653589793;
        dot[e] = d;
    }
    __syncthreads();

    // find_time_warps (lfq.rs:361-385): every warp is found on the unwarped dot products
    for (uint32_t f = 0; f < F; f++) {
        for (uint32_t o = threadIdx.x; o < 2 * LFQ_SLACK + 1; o += blockDim.x) {
            const int off = (int)o - LFQ_SLACK;
            const double* rr = dot + (size_t)ref * LFQ_GRID;
            const double* run = dot + (size_t)f * LFQ_GRID;
            double d = 0.0;
            for (int i = 0; i < LFQ_GRID; i++) {
                const int j = i + off;
                if (j >= 0 && j < LFQ_GRID) d = d + rr[i] * run[j];
            }
            wd[o] = d;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int best = 0;
            double bd = 0.0;
            for (int o = 0; o <= 2 * LFQ_SLACK; o++)
                if (wd[o] >= bd) { best = o - LFQ_SLACK; bd = wd[o]; }
            warps[f] = best;
        }
        __syncthreads();
    }

    // apply_time_warps (lfq.rs:388-400), one warp per file
    {
        const uint32_t w = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
        for (uint32_t f = w; f < F; f += nw) {
            double vs[4], vd[4];
            for (int k = 0; k < 4; k++) {
                const int i = (int)lane + 32 * k, j = i + warps[f];
                const bool ok = i < LFQ_GRID && j >= 0 && j < LFQ_GRID;
                vs[k] = ok ? sa[f * LFQ_GRID + j] : 0.0;
                vd[k] = ok ? dot[f * LFQ_GRID + j] : 0.0;
            }
            __syncwarp();
            for (int k = 0; k < 4; k++) {
                const int i = (int)lane + 32 * k;
                if (i < LFQ_GRID) { sa[f * LFQ_GRID + i] = vs[k]; dot[f * LFQ_GRID + i] = vd[k]; }
            }
        }
    }
    __syncthreads();

    // scores (lfq.rs:402-437)
    for (uint32_t col = threadIdx.x; col < LFQ_GRID; col += blockDim.x) {
        double summed = 1.0, weighted = 0.0;
        for (uint32_t f = 0; f < F; f++) {
            weighted = weighted + sa[f * LFQ_GRID + col] * dot[f * LFQ_GRID + col];
            summed = summed + dot[f * LFQ_GRID + col];
        }
        spectral[col] = weighted / summed;
        inten[col] = summed;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double mx = 0.0;
        for (int col = 0; col < LFQ_GRID; col++) mx = fmax(mx, inten[col]);
        const double* rtf = a.consts + LFQ_K_WIDTH;
        for (int col = 0; col < LFQ_GRID; col++) {
            const double s = spectral[col];
            double v;
            switch (a.peak_scoring) {
                case SAGE_B200_PEAK_RETENTION_TIME: v = rtf[col]; break;
                case SAGE_B200_PEAK_SPECTRAL_ANGLE: v = s; break;
                case SAGE_B200_PEAK_INTENSITY: v = sqrt(inten[col] / mx); break;
                default: v = s * (s * s) * rtf[col] * sqrt(inten[col] / mx); break;
            }
            scores[col] = v;
        }
        // integrate (lfq.rs:447-509)
        double best = 0.0;
        int brt = 0;
        for (int col = 0; col < LFQ_GRID; col++)
            if (scores[col] > best && spectral[col] >= a.spectral_angle) { best = scores[col]; brt = col; }
        int left = brt > 0 ? brt - 1 : 0, right = brt + 1;
        const double thr = best * 0.50;
        const int llim = brt > LFQ_GRID / 5 ? brt - LFQ_GRID / 5 : 0, rlim = min(LFQ_GRID - 1, brt + 20);
        while (left > llim && scores[left] >= thr && spectral[left] >= a.spectral_angle) left--;
        while (right < rlim && scores[right] >= thr && spectral[right] >= a.spectral_angle) right++;
        win[0] = best != 0.0;
        win[1] = brt;
        win[2] = left;
        win[3] = right;
        a.present[t] = best != 0.0;
        a.rt[t] = (uint32_t)brt;
        a.score[t] = best;
        a.sa[t] = spectral[brt];
    }
    __syncthreads();
    if (!win[0]) return;
    for (uint32_t f = threadIdx.x; f < F; f += blockDim.x) {
        double area;
        if (a.integration == SAGE_B200_INTEGRATE_SUM) {
            area = 0.0;
            for (int i = win[2]; i < win[3]; i++) area = area + dot[f * LFQ_GRID + i];
        } else {
            area = dot[f * LFQ_GRID + win[1]];
        }
        a.areas[(size_t)t * F + f] = area;
    }
}

}  // namespace sb
