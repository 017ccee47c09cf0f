// fdr.cuh — PSM rescoring on the device: Sage's linear_discriminant::score_psms (kde.rs, linear_discriminant.rs) and spectrum_q_value
// (qvalue.rs), as called by the runner's spectrum_fdr (runner.rs:280-291). Host orchestration: sage_b200.cu (sage_b200_spectrum_fdr).
//
// Exactness (DESIGN.md §10): every f64 value is the reference's, bit for bit, under these orders:
//   - sequential where the reference is sequential: Kde::new's mean and std (ml/mod.rs:24-32), the LDA class sums and scatter products
//     (linear_discriminant.rs:72-110) are single-thread folds in row order;
//   - Kde::pdf's rayon fold (kde.rs:38-48) is defined as chunks of KDE_CHUNK samples in sample order, each folded from 0.0, the chunk sums
//     added in chunk order starting from -0.0 (f64 Sum);
//   - exp / log1p / log10 are glibc's (glibc_math.cuh), log1pf glibc's (glibc_log.cuh); the library is built with -fmad=false so nothing else
//     is contracted.
#pragma once
#include <cuda_pipeline.h>
#include <stdint.h>

#include "glibc_math.cuh"
#include "../../include/sage_b200.h"

namespace sb {

constexpr int KDE_CHUNK = 4096;        // samples per fold chunk of Kde::pdf (the oracle uses the same constant)
constexpr int FDR_FEATURES = 20;       // linear_discriminant.rs:19
constexpr int LDA_TILE = 64;           // rows staged in shared memory per step of k_fdr_lda

// Rust's saturating `f64 as usize`: NaN and negatives -> 0, beyond the range -> usize::MAX.
__device__ __forceinline__ uint64_t sat_usize(double t) {
    if (!(t >= 0.0)) return 0;
    if (t >= 18446744073709551616.0) return ~0ull;
    return (uint64_t)t;
}

// kde.rs:148-168 Estimator::posterior_error
__device__ __forceinline__ double kde_posterior_error(const double* bins, uint64_t nb, double min_score, double step, double score) {
    const uint64_t last = nb == 0 ? 0 : nb - 1;
    uint64_t lo = sat_usize(floor((score - min_score) / step));
    lo = lo < last ? lo : last;
    const uint64_t hi = (lo + 1) < last ? lo + 1 : last;
    const double lower = bins[lo], upper = bins[hi];
    const double lo_score = (double)lo * step + min_score;
    const double linear = (score - lo_score) / step;
    return lower + (upper - lower) * linear;
}

// linear_discriminant.rs:140-152: the mass-error column and the decoy flags.
__global__ void k_fdr_mass(const sage_b200_feature* __restrict__ rows, uint64_t n, int tol_kind, double* __restrict__ mass_err,
                           uint8_t* __restrict__ decoy, uint8_t* __restrict__ target) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const sage_b200_feature& r = rows[i];
    mass_err[i] = tol_kind == SAGE_B200_TOL_PPM ? (double)r.delta_mass : (double)__fsub_rn(r.expmass, r.calcmass);
    decoy[i] = r.label == -1;
    target[i] = r.label != -1;
}

// ml/mod.rs:24-32 for one class per thread: mean (f64 Sum from -0.0, then / len) and std (fold from 0.0 of (x - mean)^2). Also the min / max
// of kde.rs:104-109 over all scores (f64::min / max ignore NaN; the result does not depend on the order).
__global__ void k_fdr_kde_moments(const double* __restrict__ d, uint64_t nd, const double* __restrict__ t, uint64_t nt, const double* __restrict__ all,
                                  uint64_t n, double* __restrict__ out /* [std_d, std_t, min, max] */) {
    const int tid = threadIdx.x;
    if (tid < 2) {
        const double* s = tid == 0 ? d : t;
        const uint64_t m = tid == 0 ? nd : nt;
        double sum = -0.0;
        for (uint64_t i = 0; i < m; i++) sum = sum + s[i];
        const double mean = sum / (double)m;
        double acc = 0.0;
        for (uint64_t i = 0; i < m; i++) {
            const double x = s[i] - mean;
            acc = acc + x * x;
        }
        out[tid] = sqrt(acc / (double)m);
    }
    __shared__ double smin[256], smax[256];
    double lo = 1.7976931348623157e308, hi = -1.7976931348623157e308;
    for (uint64_t i = tid; i < n; i += blockDim.x) {
        lo = fmin(lo, all[i]);
        hi = fmax(hi, all[i]);
    }
    smin[tid] = lo;
    smax[tid] = hi;
    __syncthreads();
    for (int w = blockDim.x / 2; w > 0; w >>= 1) {
        if (tid < w) {
            smin[tid] = fmin(smin[tid], smin[tid + w]);
            smax[tid] = fmax(smax[tid], smax[tid + w]);
        }
        __syncthreads();
    }
    if (tid == 0) {
        out[2] = smin[0];
        out[3] = smax[0];
    }
}

// kde.rs:34-48 for one class: partial[b * n_chunks + c] = the fold from 0.0 of exp(-0.5 * ((x_b - s_i) / h)^2) over chunk c's samples in order,
// x_b = b * step + min. Thread = bin; a warp's 32 bins read the same sample at once (broadcast).
template <bool FMA>
__global__ void k_fdr_kde_bins(const double* __restrict__ s, uint64_t m, uint32_t bins, uint32_t n_chunks, const double* __restrict__ moments,
                               double h, double* __restrict__ partial) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t c = blockIdx.y;
    if (b >= bins) return;
    const double step = (moments[3] - moments[2]) / (double)(bins - 1);
    const double x = (double)b * step + moments[2];
    const uint64_t i0 = (uint64_t)c * KDE_CHUNK, i1 = i0 + KDE_CHUNK < m ? i0 + KDE_CHUNK : m;
    double acc = 0.0;
    for (uint64_t i = i0; i < i1; i++) {
        const double u = (x - __ldg(s + i)) / h;
        acc = acc + gmath::glibc_exp<FMA>(-0.5 * (u * u));
    }
    partial[(uint64_t)b * n_chunks + c] = acc;
}

// kde.rs:112-129: the chunk sums of both classes in chunk order (f64 Sum, from -0.0), pdf = sum / constant, the PEP per bin, then (one thread)
// the monotone reverse running max.
__global__ void k_fdr_kde_pep(const double* __restrict__ part_d, uint32_t chunks_d, const double* __restrict__ part_t, uint32_t chunks_t, uint32_t bins,
                              double const_d, double const_t, double pi, int monotonic, double* __restrict__ out) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < bins) {
        double sd = -0.0, st = -0.0;
        for (uint32_t c = 0; c < chunks_d; c++) sd = sd + part_d[(uint64_t)b * chunks_d + c];
        for (uint32_t c = 0; c < chunks_t; c++) st = st + part_t[(uint64_t)b * chunks_t + c];
        const double decoy = (sd / const_d) * pi;
        const double target = (st / const_t) * (1.0 - pi);
        out[b] = decoy / (target + decoy);
    }
}
__global__ void k_fdr_kde_monotone(double* __restrict__ bins, uint32_t n) {
    double acc = bins[n - 1];
    for (uint32_t i = n; i-- > 0;) {
        acc = fmax(acc, bins[i]);   // f64::max: NaN operands are ignored
        bins[i] = acc;
    }
}

struct FdrColumns {
    const float *aligned_rt, *delta_rt, *delta_ims;   // NULL: the Feature defaults of scoring.rs:583-585
};

// linear_discriminant.rs:162-193: one feature row per PSM, row-major [n][20].
template <bool FMA>
__global__ void k_fdr_features(const sage_b200_feature* __restrict__ rows, uint64_t n, FdrColumns cols, const double* __restrict__ mass_err,
                               const double* __restrict__ mbins, uint32_t mnb, const double* __restrict__ mmoments, double* __restrict__ X) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const sage_b200_feature& r = rows[i];
    const double step = (mmoments[3] - mmoments[2]) / (double)(mnb - 1);
    double poisson = gmath::glibc_log1p<FMA>(-r.poisson);
    if (!isfinite(poisson)) poisson = 3.5;
    const float art = cols.aligned_rt ? cols.aligned_rt[i] : r.rt;
    const float drt = cols.delta_rt ? cols.delta_rt[i] : 0.999f, dims = cols.delta_ims ? cols.delta_ims[i] : 0.999f;
    auto clamp_sqrt = [](double v) {   // f64::clamp(0.001, 0.999) (NaN passes through), then sqrt
        if (v < 0.001) v = 0.001;
        if (v > 0.999) v = 0.999;
        return sqrt(v);
    };
    double* x = X + i * FDR_FEATURES;
    x[0] = (double)r.rank;
    x[1] = (double)r.charge;
    x[2] = gmath::glibc_log1p<FMA>(r.hyperscore);
    x[3] = gmath::glibc_log1p<FMA>(r.delta_next);
    x[4] = gmath::glibc_log1p<FMA>(r.delta_best);
    x[5] = kde_posterior_error(mbins, mnb, mmoments[2], step, mass_err[i]);
    x[6] = (double)r.isotope_error;
    x[7] = (double)r.average_ppm;
    x[8] = poisson;
    x[9] = gmath::glibc_log1p<FMA>((double)r.matched_intensity_pct);
    x[10] = (double)r.matched_peaks;
    x[11] = gmath::glibc_log1p<FMA>((double)r.longest_b);
    x[12] = gmath::glibc_log1p<FMA>((double)r.longest_y);
    x[13] = (double)r.longest_y / (double)r.peptide_len;
    x[14] = gmath::glibc_log1p<FMA>((double)r.peptide_len);
    x[15] = (double)r.missed_cleavages;
    x[16] = (double)art;
    x[17] = (double)r.ims;
    x[18] = clamp_sqrt((double)drt);
    x[19] = clamp_sqrt((double)dims);
}

// linear_discriminant.rs:72-110 for class blockIdx.x (0 decoy, 1 target): threads 0..19 fold the class sums in row order, then threads 0..209
// fold the distinct scatter products c_j * c_k (j <= k) in row order. Rows are staged through shared memory LDA_TILE at a time, double
// buffered: the asynchronous copy of the next tile is in flight while the current one is folded.
// out: [2][20] means, [2][20][20] scatter (both triangles), [2] counts.
__global__ void __launch_bounds__(256) k_fdr_lda(const double* __restrict__ X, const uint8_t* __restrict__ decoy, uint64_t n, double* __restrict__ means,
                                                 double* __restrict__ scatter, uint64_t* __restrict__ counts) {
    __shared__ __align__(16) double tile[2][LDA_TILE][FDR_FEATURES];
    __shared__ uint8_t cls[2][LDA_TILE];
    __shared__ double mu[FDR_FEATURES];
    const int c = blockIdx.x, tid = threadIdx.x;
    const uint8_t want = c == 0 ? 1 : 0;   // decoy flag of this class
    int pj = 0, pk = 0;
    if (tid < 210) {   // tid -> (j, k), j <= k, row-major over the upper triangle
        int t = tid;
        while (t >= FDR_FEATURES - pj) { t -= FDR_FEATURES - pj; pj++; }
        pk = pj + t;
    }
    auto stage = [&](int buf, uint64_t r0) {   // one commit group per call, empty past the end
        if (r0 < n) {
            const int nr = (int)(n - r0 < (uint64_t)LDA_TILE ? n - r0 : LDA_TILE);
            for (int e = tid; e < nr * FDR_FEATURES; e += blockDim.x) __pipeline_memcpy_async(&tile[buf][0][0] + e, X + r0 * FDR_FEATURES + e, 8);
            for (int e = tid; e < nr; e += blockDim.x) cls[buf][e] = decoy[r0 + e];
        }
        __pipeline_commit();
    };
    for (int pass = 0; pass < 2; pass++) {
        double acc = 0.0;
        uint64_t count = 0;
        stage(0, 0);
        int buf = 0;
        for (uint64_t r0 = 0; r0 < n; r0 += LDA_TILE, buf ^= 1) {
            const int nr = (int)(n - r0 < (uint64_t)LDA_TILE ? n - r0 : LDA_TILE);
            stage(buf ^ 1, r0 + LDA_TILE);
            __pipeline_wait_prior(1);   // this tile's group has landed; the next one may still be in flight
            __syncthreads();
            if (pass == 0) {
                if (tid < FDR_FEATURES) {
                    for (int r = 0; r < nr; r++)
                        if (cls[buf][r] == want) { acc = acc + tile[buf][r][tid]; count++; }
                }
            } else if (tid < 210) {
                const double mj = mu[pj], mk = mu[pk];
                for (int r = 0; r < nr; r++)
                    if (cls[buf][r] == want) acc = acc + (tile[buf][r][pj] - mj) * (tile[buf][r][pk] - mk);
            }
            __syncthreads();   // the next iteration stages into this buffer
        }
        __pipeline_wait_prior(0);
        if (pass == 0) {
            if (tid < FDR_FEATURES) {
                mu[tid] = acc / (double)count;
                means[c * FDR_FEATURES + tid] = mu[tid];
            }
            if (tid == 0) counts[c] = count;
            __syncthreads();
        } else if (tid < 210) {
            scatter[(c * FDR_FEATURES + pj) * FDR_FEATURES + pk] = acc;
            scatter[(c * FDR_FEATURES + pk) * FDR_FEATURES + pj] = acc;
        }
    }
}

// linear_discriminant.rs:209-228 and the discriminant's sort key: the dot product in order (f64 Sum from -0.0), `as f32`.
__global__ void k_fdr_project(const double* __restrict__ X, uint64_t n, const double* __restrict__ coef, double* __restrict__ disc, float* __restrict__ disc32) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double s = -0.0;
    for (int j = 0; j < FDR_FEATURES; j++) s = s + coef[j] * X[i * FDR_FEATURES + j];
    disc[i] = s;
    disc32[i] = (float)s;
}

template <bool FMA>
__global__ void k_fdr_pep(const double* __restrict__ disc, uint64_t n, const double* __restrict__ bins, uint32_t nb, const double* __restrict__ moments,
                          float* __restrict__ pep) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double step = (moments[3] - moments[2]) / (double)(nb - 1);
    float p = (float)gmath::glibc_log10<FMA>(kde_posterior_error(bins, nb, moments[2], step, disc[i]));
    if (isinf(p)) p = -324.0f;
    pep[i] = p;
}

// runner.rs:284-287: the heuristic discriminant when the LDA fails; posterior_error keeps the Feature default 1.0 (scoring.rs:577).
__global__ void k_fdr_fallback(const sage_b200_feature* __restrict__ rows, uint64_t n, float* __restrict__ disc32, float* __restrict__ pep) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    disc32[i] = __fadd_rn(glog::glibc_log1pf(-(float)rows[i].poisson), __fdiv_rn(rows[i].longest_y_pct, 3.0f));
    pep[i] = 1.0f;
}

// Sort key for `b.total_cmp(a)` (descending): ascending on the complement of f32 total order. The radix sort is stable and the values start
// as row indices, so ties keep ascending input row.
__global__ void k_fdr_sort_key(const float* __restrict__ disc32, uint64_t n, uint32_t* __restrict__ key, uint32_t* __restrict__ idx) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t u = __float_as_uint(disc32[i]);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    key[i] = ~u;
    idx[i] = (uint32_t)i;
}

__global__ void k_fdr_sorted_decoy(const sage_b200_feature* __restrict__ rows, const uint32_t* __restrict__ order, uint64_t n, uint32_t* __restrict__ is_decoy) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p < n) is_decoy[p] = rows[order[p]].label == -1;
}

// qvalue.rs:14-23 at sorted position p, stored reversed (rq[n-1-p]) for the suffix-min scan: decoy = 1 + decoys so far, target = the rest,
// both i32 cast to f32.
__global__ void k_fdr_q_raw(const uint32_t* __restrict__ decoys_incl, uint64_t n, float* __restrict__ rq) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const int32_t decoy = 1 + (int32_t)decoys_incl[p], target = (int32_t)(p + 1) - (int32_t)decoys_incl[p];
    rq[n - 1 - p] = __fdiv_rn((float)decoy, (float)target);
}

// qvalue.rs:26-34: q_min starts at 1.0; passing counts q <= 0.01.
__global__ void k_fdr_q_out(const float* __restrict__ rq_min, const uint32_t* __restrict__ order, uint64_t n, float* __restrict__ q_out,
                            unsigned long long* __restrict__ passing) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool pass = false;
    if (p < n) {
        const float q = fminf(1.0f, rq_min[n - 1 - p]);
        q_out[order[p]] = q;
        pass = q <= 0.01f;
    }
    const unsigned m = __ballot_sync(0xffffffffu, pass);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(passing, (unsigned long long)__popc(m));
}

template <bool FMA>
__global__ void k_device_math(int function, const double* x, uint64_t n, double* out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = gmath::eval(function, FMA ? 0 : 1, x[i]);
}

}  // namespace sb
