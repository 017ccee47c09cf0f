// rt.cuh — the runner's predict_rt stage on the device (runner.rs:513-531): the ascending poisson sort and interim spectrum q-values, then
// retention_alignment::global_alignment, retention_model::predict and mobility_model::predict, with regression.rs's LinearRegression::fit.
// Host orchestration: sage_b200.cu (sage_b200_predict_rt). The sort and the q-values reuse fdr.cuh.
//
// Exactness (DESIGN.md §11): every value is the reference's, bit for bit, under these orders:
//   - poisson ties: ascending input row (stable radix sort on the total-order key);
//   - the per-(peptide, file) minimum folds the training rows in poisson order with Rust's f64::min;
//   - matrix rows are in ascending PeptideIx, row means fold over files in ascending order, the per-file folds run sequentially in row order;
//   - LinearRegression::fit's fold/reduce is chunks of RT_CHUNK training rows in poisson order, each accumulator from 0.0, merged in chunk order
//     from 0.0; the SSE pass sums chunks from -0.0 and adds the chunk sums in order from -0.0; predict_peptide folds from +0.0;
//   - ln_1p is glibc's (glibc_math.cuh); the library is built with -fmad=false, so nothing is contracted.
#pragma once
#include <stdint.h>

#include "glibc_math.cuh"
#include "../../include/sage_b200.h"

namespace sb {

constexpr int RT_CHUNK = 1024;    // training rows per fold chunk of LinearRegression::fit (the oracle uses the same constant)
constexpr int RT_TILE = 32;       // rows embedded into shared memory at a time
constexpr int RT_FEATURES = 69;   // retention_model.rs:32  VALID_AA.len() * 3 + 3
constexpr int IMS_FEATURES = 100; // mobility_model.rs:75   VALID_AA.len() * 4 + 12
constexpr int N_VALID_AA = 22;

template <int MODEL> struct RtDims {
    static constexpr int D = MODEL == 0 ? RT_FEATURES : IMS_FEATURES;
    static constexpr int S = D | 1;                        // shared-memory row stride: odd, so a warp reading one column per row is conflict-free
    static constexpr int NCOV = D * (D + 1) / 2;           // distinct products cov[j][k], j <= k
    static constexpr int NACC = NCOV + D + 2;              // + X^T y, sum(y), sum(y^2)
};

// VALID_AA position of each letter A..Z (mass.rs:59-62). B, J, X and Z are not in VALID_AA: the zero-initialised map of
// retention_model.rs:64-67 sends them to column 0, A's.
__constant__ uint8_t c_aa_map[26] = {0, 0, 1, 2, 3, 4, 5, 6, 7, 0, 8, 9, 10, 11, 21, 12, 13, 14, 15, 16, 20, 17, 18, 0, 19, 0};

// mobility_model.rs:39-73: the group constants are letter offsets (b'L' - b'A', ...), but embed compares them with the VALID_AA position
// `idx`. Kept as written: "bulky" counts the residues at VALID_AA positions 11, 21, 8, 5 (N, O, K, G), and so on.
constexpr uint32_t rt_set(int a, int b = -1, int c = -1, int d = -1, int e = -1, int f = -1) {   // bit x set for each argument x >= 0
    return (a >= 0 ? 1u << a : 0u) | (b >= 0 ? 1u << b : 0u) | (c >= 0 ? 1u << c : 0u) | (d >= 0 ? 1u << d : 0u) | (e >= 0 ? 1u << e : 0u) |
           (f >= 0 ? 1u << f : 0u);
}
constexpr uint32_t RT_BULKY = rt_set('L' - 'A', 'V' - 'A', 'I' - 'A', 'F' - 'A', 'W' - 'A', 'Y' - 'A');
constexpr uint32_t RT_UC_POLAR = rt_set('S' - 'A', 'T' - 'A', 'N' - 'A', 'Q' - 'A');
constexpr uint32_t RT_POSITIVE = rt_set('R' - 'A', 'K' - 'A', 'H' - 'A');
constexpr uint32_t RT_NEGATIVE = rt_set('D' - 'A', 'E' - 'A');
constexpr uint32_t RT_TINY = rt_set('G' - 'A', 'A' - 'A', 'S' - 'A');
constexpr uint32_t RT_BRANCHED = rt_set('L' - 'A', 'I' - 'A', 'V' - 'A');

struct RtPeptides {
    const uint32_t* off;    // residue_offsets, n_peptides + 1
    const uint8_t* seq;     // residues, 'A'..'Z' (checked by the host)
    const float* mono;      // Peptide::monoisotopic
};

// Embeds rows list[r0 .. r0 + nr) (list == NULL: rows r0 ..) into emb[r * S + j], r < RT_TILE; ys[r] = the regression target (ycol[row], or
// the row's ims when ycol is NULL) when ys is given. Every thread of the block calls it. The counts are integers, so the shared-memory atomic
// adds give the same value in any order. retention_model.rs:42-59 (MODEL 0), mobility_model.rs:97-149 (MODEL 1).
template <int MODEL, bool FMA>
__device__ void rt_embed_tile(const RtPeptides P, const sage_b200_feature* __restrict__ rows, const uint32_t* __restrict__ list, uint64_t r0, int nr,
                              double* emb, double* ys, const float* __restrict__ ycol) {
    constexpr int S = RtDims<MODEL>::S;
    const int tid = threadIdx.x, nt = blockDim.x;
    __syncthreads();   // the previous tile has been read
    for (int e = tid; e < RT_TILE * S; e += nt) emb[e] = 0.0;
    if (ys && tid < nr) {
        const uint32_t row = list ? list[r0 + tid] : (uint32_t)(r0 + tid);
        ys[tid] = ycol ? (double)ycol[row] : (double)rows[row].ims;
    }
    __syncthreads();
    const int lane = tid & 31;
    for (int r = tid >> 5; r < nr; r += nt >> 5) {
        const uint32_t row = list ? list[r0 + r] : (uint32_t)(r0 + r);
        const uint32_t pep = rows[row].peptide_idx;
        const uint32_t a = P.off[pep], len = P.off[pep + 1] - a;
        const uint32_t cterm = len >= 3 ? len - 3 : 0;   // saturating_sub(3)
        double* e = emb + r * S;
        for (uint32_t p = lane; p < len; p += 32) {
            const int idx = c_aa_map[P.seq[a + p] - 'A'];
            atomicAdd(e + idx, 1.0);
            if (MODEL == 0) {
                if (p <= 1) atomicAdd(e + N_VALID_AA + idx, 1.0);                                  // N_TERMINAL
                else if (p == cterm || p == cterm + 1) atomicAdd(e + 2 * N_VALID_AA + idx, 1.0);    // C_TERMINAL: positions cterm, cterm + 1
            } else {
                if (p <= 1) atomicAdd(e + 2 * N_VALID_AA + idx, 1.0);                              // N_TERMINAL
                else if (p > cterm) atomicAdd(e + 3 * N_VALID_AA + idx, 1.0);                      // C_TERMINAL: every position past cterm
                const uint32_t bit = 1u << idx;
                if (RT_BULKY & bit) atomicAdd(e + 91, 1.0);       // NUM_BULKY
                if (RT_UC_POLAR & bit) atomicAdd(e + 90, 1.0);    // NUM_UC_POLAR
                if (RT_POSITIVE & bit) atomicAdd(e + 92, 1.0);    // NUM_POSITIVE
                if (RT_NEGATIVE & bit) atomicAdd(e + 93, 1.0);    // NUM_NEGATIVE
                if (RT_TINY & bit) atomicAdd(e + 89, 1.0);        // NUM_TINY
                if (RT_BRANCHED & bit) atomicAdd(e + 88, 1.0);    // NUM_BRANCHED
            }
        }
        if (lane == 0) {
            const double m = (double)P.mono[pep];
            if (MODEL == 0) {
                e[66] = (double)len;                        // PEPTIDE_LEN
                e[67] = gmath::glibc_log1p<FMA>(m);         // PEPTIDE_MASS: (monoisotopic as f64).ln_1p()
                e[68] = 1.0;                                // INTERCEPT
            } else {
                const double z = (double)(uint8_t)rows[row].charge;   // Feature::charge is a u8
                e[95] = z;                                  // PEPTIDE_CHARGE
                e[94] = 1.0 / z;                            // INV_PEPTIDE_CHARGE
                e[97] = (double)len;                        // PEPTIDE_LEN
                e[98] = m / 1000.0;                         // PEPTIDE_MASS
                e[96] = (m / z) / 1000.0;                   // PEPTIDE_MZ
                e[99] = 1.0;                                // INTERCEPT
            }
        }
    }
    __syncthreads();
    if (MODEL == 1) {   // PCT features: count / length
        for (int q = tid; q < nr * N_VALID_AA; q += nt) {
            const int r = q / N_VALID_AA, j = q % N_VALID_AA;
            emb[r * S + N_VALID_AA + j] = emb[r * S + j] / emb[r * S + 97];
        }
        __syncthreads();
    }
}

// regression.rs:38-51 over chunk blockIdx.x of the training list: thread = one distinct accumulator (cov[j][k] for j <= k, X^T y, sum y, sum y^2)
// of accumulator block blockIdx.y, folded from 0.0 over the chunk's rows in order. cov[k][j] is the same product in the same order, so the host
// mirrors it. partial[chunk][NACC]. Launched with 256 threads; __maxnreg__ (instead of __launch_bounds__, which left ptxas spilling at 40
// registers) lets the mobility model's embedding keep its state in registers.
template <int MODEL, bool FMA>
__global__ void __maxnreg__(64) k_rt_accumulate(const RtPeptides P, const sage_b200_feature* __restrict__ rows, const uint32_t* __restrict__ train,
                                                       uint64_t n_train, const float* __restrict__ ycol, double* __restrict__ partial) {
    using Dm = RtDims<MODEL>;
    constexpr int D = Dm::D, S = Dm::S;
    __shared__ double emb[RT_TILE * S];
    __shared__ double ys[RT_TILE];
    const int a = blockIdx.y * blockDim.x + threadIdx.x;
    int kind = 4, pj = 0, pk = 0;   // 0 cov, 1 X^T y, 2 sum y, 3 sum y^2, 4 idle
    if (a < Dm::NCOV) {
        int t = a;
        while (t >= D - pj) { t -= D - pj; pj++; }
        pk = pj + t;
        kind = 0;
    } else if (a < Dm::NCOV + D) {
        kind = 1;
        pj = a - Dm::NCOV;
    } else if (a < Dm::NACC) {
        kind = a == Dm::NCOV + D ? 2 : 3;
    }
    const uint64_t c0 = (uint64_t)blockIdx.x * RT_CHUNK, c1 = c0 + RT_CHUNK < n_train ? c0 + RT_CHUNK : n_train;
    double acc = 0.0;
    for (uint64_t r0 = c0; r0 < c1; r0 += RT_TILE) {
        const int nr = (int)(c1 - r0 < (uint64_t)RT_TILE ? c1 - r0 : RT_TILE);
        rt_embed_tile<MODEL, FMA>(P, rows, train, r0, nr, emb, ys, ycol);
        if (kind == 0) {
            for (int r = 0; r < nr; r++) acc = acc + emb[r * S + pj] * emb[r * S + pk];
        } else if (kind == 1) {
            for (int r = 0; r < nr; r++) acc = acc + emb[r * S + pj] * ys[r];
        } else if (kind == 2) {
            for (int r = 0; r < nr; r++) acc = acc + ys[r];
        } else if (kind == 3) {
            for (int r = 0; r < nr; r++) acc = acc + ys[r] * ys[r];
        }
    }
    if (kind != 4) partial[(uint64_t)blockIdx.x * Dm::NACC + a] = acc;
}

// Acc::merge under reduce(Acc::zero): ((0 + A_0) + A_1) + ... in chunk order, one thread per accumulator.
__global__ void k_rt_merge(const double* __restrict__ partial, uint64_t n_chunks, int nacc, double* __restrict__ out) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= nacc) return;
    double s = 0.0;
    for (uint64_t c = 0; c < n_chunks; c++) s = s + partial[c * nacc + a];
    out[a] = s;
}

// regression.rs:104-113 for chunk blockIdx.x (one warp): per row pred = X beta in order (f64 Sum, from -0.0), (pred - y)^2; the chunk's sum from
// -0.0 in row order. The host adds the chunk sums in chunk order from -0.0.
template <int MODEL, bool FMA>
__global__ void __launch_bounds__(32) k_rt_sse(const RtPeptides P, const sage_b200_feature* __restrict__ rows, const uint32_t* __restrict__ train,
                                               uint64_t n_train, const float* __restrict__ ycol, const double* __restrict__ beta, double* __restrict__ chunk_sse) {
    constexpr int D = RtDims<MODEL>::D, S = RtDims<MODEL>::S;
    __shared__ double emb[RT_TILE * S];
    __shared__ double ys[RT_TILE], sq[RT_TILE];
    const int lane = threadIdx.x;
    const uint64_t c0 = (uint64_t)blockIdx.x * RT_CHUNK, c1 = c0 + RT_CHUNK < n_train ? c0 + RT_CHUNK : n_train;
    double csum = -0.0;
    for (uint64_t r0 = c0; r0 < c1; r0 += RT_TILE) {
        const int nr = (int)(c1 - r0 < (uint64_t)RT_TILE ? c1 - r0 : RT_TILE);
        rt_embed_tile<MODEL, FMA>(P, rows, train, r0, nr, emb, ys, ycol);
        if (lane < nr) {
            double pred = -0.0;
            for (int j = 0; j < D; j++) pred = pred + emb[lane * S + j] * __ldg(beta + j);
            const double d = pred - ys[lane];
            sq[lane] = d * d;   // powi(2)
        }
        __syncwarp();
        if (lane == 0)
            for (int r = 0; r < nr; r++) csum = csum + sq[r];
        __syncwarp();
    }
    if (lane == 0) chunk_sse[blockIdx.x] = csum;
}

// retention_model.rs:14-25 / mobility_model.rs:14-32 for rows blockIdx.x * RT_TILE .. (one warp, one lane per row): predict_peptide folds
// x * beta from +0.0, then clamp(0, hi) (NaN passes) as f32, and |actual - bounded| in f32. actual: aligned_rt (MODEL 0) or ims (MODEL 1).
template <int MODEL, bool FMA>
__global__ void __launch_bounds__(32) k_rt_predict(const RtPeptides P, const sage_b200_feature* __restrict__ rows, uint64_t n, const double* __restrict__ beta,
                                                   const float* __restrict__ aligned_rt, float* __restrict__ predicted, float* __restrict__ delta) {
    constexpr int D = RtDims<MODEL>::D, S = RtDims<MODEL>::S;
    __shared__ double emb[RT_TILE * S];
    const int lane = threadIdx.x;
    const uint64_t r0 = (uint64_t)blockIdx.x * RT_TILE;
    const int nr = (int)(n - r0 < (uint64_t)RT_TILE ? n - r0 : RT_TILE);
    rt_embed_tile<MODEL, FMA>(P, rows, nullptr, r0, nr, emb, nullptr, nullptr);
    if (lane >= nr) return;
    double s = 0.0;
    for (int j = 0; j < D; j++) s = s + emb[lane * S + j] * __ldg(beta + j);
    const double hi = MODEL == 0 ? 1.0 : 2.0;
    if (s < 0.0) s = 0.0;
    if (s > hi) s = hi;
    const float bounded = __double2float_rn(s);
    const uint64_t row = r0 + lane;
    const float actual = MODEL == 0 ? aligned_rt[row] : rows[row].ims;
    predicted[row] = bounded;
    delta[row] = fabsf(__fsub_rn(actual, bounded));
}

// The Feature defaults when a model returns None (scoring.rs): predicted 0.0, delta 0.999.
__global__ void k_rt_defaults(uint64_t n, float* __restrict__ predicted, float* __restrict__ delta) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    predicted[i] = 0.0f;
    delta[i] = 0.999f;
}

// ------------------------------------------------------------------------------------------------ sort, training set, global_alignment
// Ascending key of `a.poisson.total_cmp(&b.poisson)`; the values start as row indices, so the stable radix sort breaks ties by ascending row.
__global__ void k_rt_poisson_key(const sage_b200_feature* __restrict__ rows, uint64_t n, uint64_t* __restrict__ key, uint32_t* __restrict__ idx) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t u = (uint64_t)__double_as_longlong(rows[i].poisson);
    key[i] = (u >> 63) ? ~u : (u | 0x8000000000000000ull);
    idx[i] = (uint32_t)i;
}

// The training filter of retention_alignment.rs:48 / retention_model.rs:71 / mobility_model.rs:161, at each sorted position.
__global__ void k_rt_train_flag(const sage_b200_feature* __restrict__ rows, const uint32_t* __restrict__ order, const float* __restrict__ q, uint64_t n,
                                uint8_t* __restrict__ flag) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const uint32_t r = order[p];
    flag[p] = rows[r].label == 1 && q[r] <= 0.01f;
}

// retention_alignment.rs:26-40: fetch_max of `rt.ceil() as u32` (Rust's saturating cast: NaN and negatives -> 0, beyond -> u32::MAX).
__global__ void k_rt_max_rt(const sage_b200_feature* __restrict__ rows, const uint32_t* __restrict__ file_id, uint64_t n, unsigned* __restrict__ max_rt) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float c = ceilf(rows[i].rt);
    const unsigned v = !(c >= 0.0f) ? 0u : (c >= 4294967296.0f ? 0xFFFFFFFFu : (unsigned)c);
    atomicMax(max_rt + file_id[i], v);
}

// (PeptideIx, file) key of each training row, for the stable sort that groups them without disturbing poisson order.
__global__ void k_rt_pf_key(const sage_b200_feature* __restrict__ rows, const uint32_t* __restrict__ file_id, const uint32_t* __restrict__ train,
                            uint64_t n_train, uint64_t* __restrict__ key) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_train) return;
    const uint32_t r = train[t];
    key[t] = ((uint64_t)rows[r].peptide_idx << 32) | file_id[r];
}

__global__ void k_rt_heads(const uint64_t* __restrict__ key, uint64_t n, uint8_t* __restrict__ flag) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) flag[t] = t == 0 || key[t] != key[t - 1];
}

// Rust's f64::min as the fold uses it: a NaN operand yields the other one; -0.0 is kept over +0.0.
__device__ __forceinline__ double rust_min(double a, double b) {
    if (isnan(a)) return b;
    if (isnan(b)) return a;
    if (b < a || (b == a && signbit(b))) return b;
    return a;
}

// retention_alignment.rs:44-57 for one (peptide, file) segment: the first rt as f64, then f64::min in poisson order. Also flags the first
// segment of each peptide.
__global__ void k_rt_seg_min(const sage_b200_feature* __restrict__ rows, const uint64_t* __restrict__ key, const uint32_t* __restrict__ val,
                             const uint32_t* __restrict__ seg_start, uint64_t n_seg, uint64_t n_train, double* __restrict__ seg_min,
                             uint8_t* __restrict__ pep_head) {
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_seg) return;
    const uint64_t t0 = seg_start[s], t1 = s + 1 < n_seg ? seg_start[s + 1] : n_train;
    double m = (double)rows[val[t0]].rt;
    for (uint64_t t = t0 + 1; t < t1; t++) m = rust_min(m, (double)rows[val[t]].rt);
    seg_min[s] = m;
    pep_head[s] = s == 0 || (key[t0] >> 32) != (key[seg_start[s - 1]] >> 32);
}

// retention_alignment.rs:62-80 for one peptide (segments in ascending file order): sum from 0.0 and len of rt / max_rt[file]; the row is kept
// when the mean is_normal().
__global__ void k_rt_row_mean(const uint64_t* __restrict__ key, const uint32_t* __restrict__ seg_start, const double* __restrict__ seg_min,
                              const uint32_t* __restrict__ prow_start, uint64_t n_pr, uint64_t n_seg, const unsigned* __restrict__ max_rt,
                              uint32_t* __restrict__ keep) {
    const uint64_t pr = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pr >= n_pr) return;
    const uint64_t s0 = prow_start[pr], s1 = pr + 1 < n_pr ? prow_start[pr + 1] : n_seg;
    double sum = 0.0, len = 0.0;
    for (uint64_t s = s0; s < s1; s++) {
        const uint32_t f = (uint32_t)key[seg_start[s]];
        sum = sum + seg_min[s] / (double)max_rt[f];
        len = len + 1.0;
    }
    const double mean = sum / len;
    keep[pr] = isfinite(mean) && fabs(mean) >= 2.2250738585072014e-308;
}

// One kept matrix row: mat[row][file] = rt / max_rt[file] (the rest stays NaN) and retention_alignment.rs:99-109's mean over the finite entries
// in file order.
__global__ void k_rt_fill(const uint64_t* __restrict__ key, const uint32_t* __restrict__ seg_start, const double* __restrict__ seg_min,
                          const uint32_t* __restrict__ prow_start, uint64_t n_pr, uint64_t n_seg, const unsigned* __restrict__ max_rt,
                          const uint32_t* __restrict__ keep, const uint32_t* __restrict__ mrow, uint64_t n_files, double* __restrict__ mat,
                          double* __restrict__ mean_rts) {
    const uint64_t pr = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pr >= n_pr || !keep[pr]) return;
    const uint64_t s0 = prow_start[pr], s1 = pr + 1 < n_pr ? prow_start[pr + 1] : n_seg, row = mrow[pr];
    uint64_t len = 0;
    double sum = 0.0;
    for (uint64_t s = s0; s < s1; s++) {
        const uint32_t f = (uint32_t)key[seg_start[s]];
        const double x = seg_min[s] / (double)max_rt[f];
        mat[row * n_files + f] = x;
        if (isfinite(x)) { len++; sum = sum + x; }
    }
    mean_rts[row] = sum / (double)len;
}

// retention_alignment.rs:112-158 for one file: the sequential folds over the matrix column in row order, slope and intercept (the intercept
// from the slope before its reset), the f32 casts.
__global__ void k_rt_align(const double* __restrict__ mat, const double* __restrict__ mean_rts, uint64_t n_rows, uint64_t n_files,
                           const unsigned* __restrict__ max_rt, sage_b200_alignment* __restrict__ out) {
    const uint64_t f = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_files) return;
    uint64_t len = 0;
    double dot = 0.0, sum_x = 0.0, sum_y = 0.0;
    for (uint64_t r = 0; r < n_rows; r++) {
        const double x = mat[r * n_files + f];
        if (!isfinite(x)) continue;
        const double y = mean_rts[r];
        len++;
        dot = dot + x * y;
        sum_x = sum_x + x;
        sum_y = sum_y + y;
    }
    const double x_mean = sum_x / (double)len, y_mean = sum_y / (double)len;
    const double ssxy = dot - (double)len * x_mean * y_mean;
    double sx2 = 1E-8;
    for (uint64_t r = 0; r < n_rows; r++) {
        const double x = mat[r * n_files + f];
        if (!isfinite(x)) continue;
        const double d = x - x_mean;
        sx2 = sx2 + d * d;
    }
    double slope = ssxy / sx2;
    double intercept = y_mean - slope * x_mean;
    if (!isfinite(slope)) slope = 1.0;
    if (!isfinite(intercept)) intercept = 0.0;
    out[f].max_rt = __double2float_rn((double)max_rt[f]);
    out[f].slope = __double2float_rn(slope);
    out[f].intercept = __double2float_rn(intercept);
}

// retention_alignment.rs:163-170: aligned_rt = (rt / max_rt) * slope + intercept in f32.
__global__ void k_rt_aligned(const sage_b200_feature* __restrict__ rows, const uint32_t* __restrict__ file_id, uint64_t n,
                             const sage_b200_alignment* __restrict__ al, float* __restrict__ aligned_rt) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const sage_b200_alignment a = al[file_id[i]];
    aligned_rt[i] = __fadd_rn(__fmul_rn(__fdiv_rn(rows[i].rt, a.max_rt), a.slope), a.intercept);
}

}  // namespace sb
