// picked.cuh — picked-peptide / picked-protein FDR and MS1 precursor q-values on the device: Sage's fdr.rs (Competition::assign_q_value,
// picked_peptide, picked_protein, picked_precursor). Host orchestration: sage_b200.cu (sage_b200_picked_fdr, sage_b200_picked_precursor).
//
// Exactness (DESIGN.md §12): every output is the reference's, bit for bit, under these definitions:
//   - competition entries are ordered by the first row that reaches them (an insertion-ordered map);
//   - f32::max is `v > acc ? v : acc` (NaN ignored, the earlier of two equal zeros kept); f32::min on q-values keeps -0.0 over +0.0 and
//     ignores NaN;
//   - the running PEP sum is a sequential f32 fold; the f32 target counter is min(count, 2^24);
//   - peptide keys are equal when their Display strings are, i.e. when the canonical tuples below are.
#pragma once
#include <stdint.h>

#include "fdr.cuh"

namespace sb {

constexpr float PICKED_F32_MIN = -3.40282347e+38f;   // f32::MIN, where Competition's scores start (fdr.rs:31-39)

// A referenced peptide's key material: its residues and modifications (compact CSR over the referenced peptides), nterm / cterm (NaN = None)
// and whether the interior is read reversed (generate_decoys && decoy: Peptide::reverse, peptide.rs:307-318).
struct PickedPeptides {
    const uint32_t* off;
    const uint8_t* seq;
    const float* mods;
    const float* nterm;
    const float* cterm;
    const uint8_t* reversed;
};

// Residue index j of the key of a peptide of length L: `sequence[1..n].reverse()` with n = L - 1 when reversed and n > 1.
__device__ __forceinline__ uint32_t picked_pos(uint32_t j, uint32_t L, bool rev) {
    const uint32_t n = L - 1;
    return (rev && L > 2 && j >= 1 && j < n) ? n - j : j;
}
// Canonical modification: what `m != 0.0` / `{:+}` can tell apart. Both zeros print nothing, every NaN prints "NaN".
__device__ __forceinline__ uint32_t picked_mod(float m) {
    if (m == 0.0f) return 0u;
    if (m != m) return 0x7FC00000u;
    return __float_as_uint(m);
}
// Canonical terminal: None (NaN) or the bits (Some(-0.0) prints "[-0]", so the sign of zero is kept). 64-bit so None differs from every f32.
__device__ __forceinline__ uint64_t picked_term(float t) { return t != t ? (1ull << 32) : (uint64_t)__float_as_uint(t); }

__device__ __forceinline__ uint64_t picked_mix(uint64_t h, uint64_t x) {
    h ^= x + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
    h *= 0xFF51AFD7ED558CCDull;
    return h ^ (h >> 31);
}

// One thread per referenced peptide: a 64-bit hash of the canonical key, truncated to `mask` (the collision hook narrows it).
__global__ void k_picked_hash(PickedPeptides P, uint32_t n, uint64_t mask, uint64_t* __restrict__ hash, uint32_t* __restrict__ idx) {
    const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n) return;
    const uint32_t o = P.off[u], L = P.off[u + 1] - o;
    const bool rev = P.reversed[u] != 0;
    uint64_t h = picked_mix(0x5A6E, picked_term(P.nterm[u]));
    h = picked_mix(h, L);
    for (uint32_t j = 0; j < L; j++) {
        const uint32_t s = o + picked_pos(j, L, rev);
        h = picked_mix(h, ((uint64_t)P.seq[s] << 32) | picked_mod(P.mods[s]));
    }
    h = picked_mix(h, picked_term(P.cterm ? P.cterm[u] : __int_as_float(0x7FC00000)));
    hash[u] = h & mask;
    idx[u] = u;
}

__device__ bool picked_key_equal(const PickedPeptides& P, uint32_t a, uint32_t b) {
    const uint32_t oa = P.off[a], La = P.off[a + 1] - oa, ob = P.off[b], Lb = P.off[b + 1] - ob;
    if (La != Lb || picked_term(P.nterm[a]) != picked_term(P.nterm[b])) return false;
    if (P.cterm && picked_term(P.cterm[a]) != picked_term(P.cterm[b])) return false;
    const bool ra = P.reversed[a] != 0, rb = P.reversed[b] != 0;
    for (uint32_t j = 0; j < La; j++) {
        const uint32_t sa = oa + picked_pos(j, La, ra), sb = ob + picked_pos(j, Lb, rb);
        if (P.seq[sa] != P.seq[sb] || picked_mod(P.mods[sa]) != picked_mod(P.mods[sb])) return false;
    }
    return true;
}

// Exact grouping after the sort by hash: the peptide at sorted position p joins the first position of its equal-hash run whose key is equal
// to its own. group[peptide] = that position, so equal keys share one id even when distinct keys share a hash.
__global__ void k_picked_group(PickedPeptides P, const uint64_t* __restrict__ hash_sorted, const uint32_t* __restrict__ u_sorted, uint32_t n,
                               uint32_t* __restrict__ group) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const uint64_t h = hash_sorted[p];
    const uint32_t u = u_sorted[p];
    uint32_t rep = p;
    for (uint32_t q = p; q-- > 0 && hash_sorted[q] == h;)
        if (picked_key_equal(P, u_sorted[q], u)) rep = q;
    group[u] = rep;
}

// Row i's key for the competition: the group of its peptide (peptide level) or its protein id (protein level; rows without exactly one
// protein take no part).
__global__ void k_picked_peptide_keys(const uint32_t* __restrict__ row_slot, const uint32_t* __restrict__ group, uint32_t n, uint32_t* __restrict__ key) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) key[i] = group[row_slot[i]];
}

// Heads of equal-key runs in the (key, row)-sorted list: the head's row is the first row that reaches the entry.
__global__ void k_picked_heads(const uint32_t* __restrict__ key_sorted, uint32_t n, uint32_t* __restrict__ head) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < n) head[p] = (p == 0 || key_sorted[p] != key_sorted[p - 1]) ? 1u : 0u;
}

// entry rank of every row: rank_of_group[group index at its sorted position], then the (rank << 1 | side) key of the fold sort.
__global__ void k_picked_row_rank(const uint32_t* __restrict__ row_sorted, const uint32_t* __restrict__ group_incl, const uint32_t* __restrict__ rank_of_group,
                                  const uint8_t* __restrict__ row_decoy, uint32_t n, uint32_t* __restrict__ rank, uint32_t* __restrict__ side_key,
                                  uint32_t* __restrict__ idx) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const uint32_t i = row_sorted[p];
    const uint32_t r = rank_of_group[group_incl[p] - 1];
    rank[i] = r;
    side_key[i] = (r << 1) | (row_decoy[i] ? 1u : 0u);
    idx[i] = i;
}

__global__ void k_picked_iota(uint32_t n, uint32_t* __restrict__ v) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = i;
}

// rank_of_group[g] = position of group g in ascending first-row order.
__global__ void k_picked_scatter_rank(const uint32_t* __restrict__ g_sorted, uint32_t n, uint32_t* __restrict__ rank_of_group) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n) rank_of_group[g_sorted[r]] = r;
}

// fdr.rs:125-144 / 160-177 for one (entry, side) segment of the (rank << 1 | side)-sorted rows, in row order: `score = score.max(feature)`,
// the side's ix set. Peptide level (pep != NULL): two distinct PeptideIx in one segment is the reference's panic; the first such pair is
// reported in clash[0..1] (clash[2] = 1).
__global__ void k_picked_fold(const uint32_t* __restrict__ key_sorted, const uint32_t* __restrict__ row_sorted, const uint32_t* __restrict__ seg_start,
                              uint32_t n_seg, uint32_t n, const float* __restrict__ score, const uint32_t* __restrict__ pep, float* __restrict__ side_score,
                              uint8_t* __restrict__ side_has, uint32_t* __restrict__ clash) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_seg) return;
    const uint32_t a = seg_start[s], b = s + 1 < n_seg ? seg_start[s + 1] : n;
    float acc = PICKED_F32_MIN;
    const uint32_t first = row_sorted[a];
    for (uint32_t p = a; p < b; p++) {
        const uint32_t i = row_sorted[p];
        const float v = score[i];
        acc = v > acc ? v : acc;
        if (pep && pep[i] != pep[first] && atomicCAS(clash + 2, 0u, 1u) == 0u) {
            clash[0] = pep[first];
            clash[1] = pep[i];
        }
    }
    const uint32_t k = key_sorted[a];   // rank << 1 | side
    side_score[k] = acc;
    side_has[k] = 1;
}

// fdr.rs:43-57 per entry: score() = forward.max(reverse), is_decoy() = reverse >= forward, as the KDE's sample; and the number of rows it gives.
__global__ void k_picked_entries(const float* __restrict__ side_score, const uint8_t* __restrict__ side_has, uint32_t n_entries, double* __restrict__ kde_score,
                                 uint8_t* __restrict__ kde_flags /* [decoy | target] */, uint32_t* __restrict__ n_rows) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_entries) return;
    const float f = side_has[2 * e] ? side_score[2 * e] : PICKED_F32_MIN, r = side_has[2 * e + 1] ? side_score[2 * e + 1] : PICKED_F32_MIN;
    kde_score[e] = (double)(r > f ? r : f);
    const bool dec = r >= f;
    kde_flags[e] = dec;
    kde_flags[n_entries + e] = !dec;
    n_rows[e] = (uint32_t)side_has[2 * e] + side_has[2 * e + 1];
}

// fdr.rs:69-85: the entry's forward row, then its reverse row, each where its ix is set. ix = rank * 2 + side (or rank * 2 when ix_has_side
// is false: picked_protein's ix without generate_decoys is the protein name alone). Also the sort key of the descending f32 total order.
__global__ void k_picked_rows(const float* __restrict__ side_score, const uint8_t* __restrict__ side_has, const uint32_t* __restrict__ row_off,
                              uint32_t n_entries, bool ix_has_side, float* __restrict__ q_score, uint8_t* __restrict__ q_decoy, uint32_t* __restrict__ q_ix,
                              uint32_t* __restrict__ q_key, uint32_t* __restrict__ q_idx) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_entries) return;
    uint32_t o = row_off[e];
    for (uint32_t side = 0; side < 2; side++) {
        if (!side_has[2 * e + side]) continue;
        const float s = side_score[2 * e + side];
        q_score[o] = s;
        q_decoy[o] = (uint8_t)side;
        q_ix[o] = 2 * e + (ix_has_side ? side : 0u);
        uint32_t u = __float_as_uint(s);
        u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
        q_key[o] = ~u;
        q_idx[o] = o;
        o++;
    }
}

// Per sorted row: pep = posterior_error(score as f64) as f32 (fdr.rs:92), or for picked_precursor 1.0 on decoy rows and 0.0 on target rows
// (bins == NULL: adding +0.0 leaves the sum as it is, so the one running sum is both of fdr.rs:257-263's counters); the target flag.
__global__ void k_picked_pep(const uint32_t* __restrict__ order, const float* __restrict__ score, const uint8_t* __restrict__ decoy, uint32_t n,
                             const double* __restrict__ bins, const double* __restrict__ moments, float* __restrict__ pep, uint32_t* __restrict__ is_target) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const uint32_t r = order[p];
    if (bins) {
        const double step = (moments[3] - moments[2]) / 999.0;
        pep[p] = (float)kde_posterior_error(bins, 1000, moments[2], step, (double)score[r]);
    } else {
        pep[p] = decoy[r] ? 1.0f : 0.0f;
    }
    is_target[p] = decoy[r] ? 0u : 1u;
}

// fdr.rs:89-99: `decoy += pep` from 1.0, one f32 addition after another. One thread; the next 32 values are loaded while the current 32 are
// added, so the loads stay off the dependent chain.
__global__ void __launch_bounds__(32) k_picked_running_sum(const float* __restrict__ pep, uint32_t n, float* __restrict__ sum) {
    if (threadIdx.x != 0) return;
    constexpr uint32_t B = 32;
    float cur[B], nxt[B];
    float acc = 1.0f;
    const uint32_t full = n / B * B;
    if (full) {
#pragma unroll
        for (uint32_t k = 0; k < B; k++) cur[k] = pep[k];
    }
    for (uint32_t b = 0; b < full; b += B) {
        if (b + B < full) {
#pragma unroll
            for (uint32_t k = 0; k < B; k++) nxt[k] = pep[b + B + k];
        }
#pragma unroll
        for (uint32_t k = 0; k < B; k++) {
            acc = __fadd_rn(acc, cur[k]);
            sum[b + k] = acc;
        }
#pragma unroll
        for (uint32_t k = 0; k < B; k++) cur[k] = nxt[k];
    }
    for (uint32_t p = full; p < n; p++) {
        acc = __fadd_rn(acc, pep[p]);
        sum[p] = acc;
    }
}

// q = decoy / target at sorted position p (target: f32 `+= 1.0` from 0, which stops at 2^24), stored reversed for the suffix-minimum scan.
__global__ void k_picked_q_raw(const float* __restrict__ sum, const uint32_t* __restrict__ targets_incl, uint32_t n, float* __restrict__ rq) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const uint32_t t = targets_incl[p] < (1u << 24) ? targets_incl[p] : (1u << 24);
    rq[n - 1 - p] = __fdiv_rn(sum[p], (float)t);
}

// f32::min as DESIGN.md §12 defines it: NaN ignored, -0.0 below +0.0. Associative and commutative, so a scan computes the sequential fold.
struct PickedMin {
    __device__ float operator()(float a, float b) const {
        if (a != a) return b;
        if (b != b) return a;
        if (a < b) return a;
        if (b < a) return b;
        return signbit(a) ? a : b;
    }
};

// fdr.rs:103-111: q_min from 1.0 over the rows from the back; `passing` counts target rows at q <= threshold. The winner of each ix is the
// latest sorted row that carries it (rayon's ordered collect into a map).
__global__ void k_picked_q_min(const float* __restrict__ rq_min, const uint8_t* __restrict__ decoy, const uint32_t* __restrict__ order,
                               const uint32_t* __restrict__ ix, uint32_t n, float threshold, float* __restrict__ q, uint32_t* __restrict__ win,
                               unsigned long long* __restrict__ passing) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    bool pass = false;
    if (p < n) {
        const float v = PickedMin()(1.0f, rq_min[n - 1 - p]);
        q[p] = v;
        const uint32_t r = order[p];
        pass = v <= threshold && !decoy[r];
        atomicMax(win + ix[r], p);
    }
    const unsigned m = __ballot_sync(0xffffffffu, pass);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(passing, (unsigned long long)__popc(m));
}

__global__ void k_picked_q_ix(const float* __restrict__ q, const uint32_t* __restrict__ order, const uint32_t* __restrict__ ix, const uint32_t* __restrict__ win,
                              uint32_t n, float* __restrict__ q_ix) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const uint32_t i = ix[order[p]];
    if (win[i] == p) q_ix[i] = q[p];
}

// fdr.rs:148-150 / 181-187: each competing row reads the q of its ix.
__global__ void k_picked_gather(const uint32_t* __restrict__ rank, const uint8_t* __restrict__ row_decoy, uint32_t n, bool ix_has_side,
                                const float* __restrict__ q_ix, float* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = q_ix[2 * rank[i] + (ix_has_side && row_decoy[i] ? 1u : 0u)];
}

// picked_precursor's rows (fdr.rs:245-253): score = peak.score as f32, in the caller's row order; ix = the row.
__global__ void k_picked_precursor_rows(const double* __restrict__ score, uint32_t n, float* __restrict__ q_score, uint32_t* __restrict__ q_ix,
                                        uint32_t* __restrict__ q_key, uint32_t* __restrict__ q_idx) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float s = (float)score[i];
    q_score[i] = s;
    q_ix[i] = i;
    uint32_t u = __float_as_uint(s);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    q_key[i] = ~u;
    q_idx[i] = i;
}

}  // namespace sb
