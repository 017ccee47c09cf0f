// prefilter.cuh — the database prefilter on the device: runner.rs:104-128 and 161-238 (prefilter_peptides) with database.rs:221-258
// (reorder_peptides) over a table of materialized rows. Host orchestration (the chunk loop, the automatic chunk size, the stage order):
// sage_b200.cu (sage_b200_prefilter_create). DESIGN.md §15 states the contract.
//
// Layout: a table is the digest's export layout held on the device (residue and protein-reference offsets per row, residues and
// modifications per residue, nterm / cterm / mono / decoy / missed / semi per row, protein ids per reference). The kept rows of every chunk
// are appended to one such table in chunk order; the merge sorts and merges its rows and writes the final table in the same layout.
#pragma once
#include <stdint.h>

#include "digest.cuh"   // dg_cmp_opt: Option<f32>::partial_cmp with NaN = None

namespace sb {

struct PfRows {
    const uint32_t* res_off;   // [n + 1]
    const uint32_t* ref_off;   // [n + 1]
    const uint8_t* seq;
    const float* mods;
    const float *nterm, *cterm, *mono;   // NaN = None
    const uint8_t *decoy, *missed, *semi;
    const uint32_t* ids;
};

// ------------------------------------------------------------------------------------------------ the index build from a device table
// Per peptide: its length, flags (decoy), ion count n_kinds * (L - 1) and kept fragment count n_kinds * max(0, L - 1 - min_ion_index)
// (database.rs:281-291); `bad` receives 1 for a peptide of length 0 or over 255 (the library's limit).
__global__ void k_pf_pep_meta(const uint32_t* __restrict__ res_off, const uint8_t* __restrict__ decoy, uint32_t n, uint32_t n_kinds, uint64_t min_ion_index,
                              uint8_t* __restrict__ len, uint8_t* __restrict__ flags, uint64_t* __restrict__ n_ions, uint64_t* __restrict__ n_frag,
                              uint32_t* __restrict__ bad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t L = res_off[i + 1] - res_off[i];
    if (L == 0 || L > 255) atomicOr(bad, 1u);
    len[i] = (uint8_t)L;
    flags[i] = decoy[i] ? 1 : 0;
    n_ions[i] = L ? n_kinds * (L - 1) : 0;
    n_frag[i] = (L && (L - 1) > min_ion_index) ? n_kinds * ((L - 1) - min_ion_index) : 0;
}

// ------------------------------------------------------------------------------------------------ keep-mask compaction
// Per row of a chunk's table: 1 when quick_score kept it, its residue count and its protein-reference count (0 for a dropped row).
__global__ void k_pf_keep_counts(const uint8_t* __restrict__ keep, const uint32_t* __restrict__ res_off, const uint32_t* __restrict__ ref_off, uint32_t n,
                                 uint32_t* __restrict__ kept, uint64_t* __restrict__ n_res, uint64_t* __restrict__ n_ref) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool k = keep[i] != 0;
    kept[i] = k ? 1u : 0u;
    n_res[i] = k ? res_off[i + 1] - res_off[i] : 0;
    n_ref[i] = k ? ref_off[i + 1] - ref_off[i] : 0;
}

// Appends the kept rows of one chunk's table at (row0, res0, ref0) of the growing table; row_at / res_at / ref_at are the exclusive scans
// of k_pf_keep_counts' outputs. Protein ids are already ranks in the whole FASTA's names table (the chunk was digested with that map).
__global__ void k_pf_gather(PfRows src, uint32_t n, const uint8_t* __restrict__ keep, const uint32_t* __restrict__ row_at, const uint64_t* __restrict__ res_at,
                            const uint64_t* __restrict__ ref_at, uint32_t row0, uint64_t res0, uint64_t ref0, uint32_t* __restrict__ res_off,
                            uint32_t* __restrict__ ref_off, uint8_t* __restrict__ seq, float* __restrict__ mods, float* __restrict__ nterm,
                            float* __restrict__ cterm, float* __restrict__ mono, uint8_t* __restrict__ decoy, uint8_t* __restrict__ missed,
                            uint8_t* __restrict__ semi, uint32_t* __restrict__ ids) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !keep[i]) return;
    const uint32_t j = row0 + row_at[i];
    const uint64_t r = res0 + res_at[i], f = ref0 + ref_at[i];
    res_off[j] = (uint32_t)r;
    ref_off[j] = (uint32_t)f;
    for (uint32_t a = src.res_off[i], b = 0; a < src.res_off[i + 1]; a++, b++) {
        seq[r + b] = src.seq[a];
        mods[r + b] = src.mods[a];
    }
    for (uint32_t a = src.ref_off[i], b = 0; a < src.ref_off[i + 1]; a++, b++) ids[f + b] = src.ids[a];
    nterm[j] = src.nterm[i];
    cterm[j] = src.cterm[i];
    mono[j] = src.mono[i];
    decoy[j] = src.decoy[i];
    missed[j] = src.missed[i];
    semi[j] = src.semi[i];
}

// ------------------------------------------------------------------------------------------------ reorder_peptides over stored rows
// Peptide::initial_sort (peptide.rs:34-52) of two stored rows: sequence bytes (then length), modifications by partial_cmp (an unordered
// pair ends the comparison as Equal; -0.0 == 0.0), nterm, then cterm with None < Some.
__device__ int pf_initial_sort(const PfRows& T, uint32_t a, uint32_t b) {
    const uint32_t oa = T.res_off[a], ob = T.res_off[b], la = T.res_off[a + 1] - oa, lb = T.res_off[b + 1] - ob, n = min(la, lb);
    for (uint32_t j = 0; j < n; j++) {
        const uint8_t x = T.seq[oa + j], y = T.seq[ob + j];
        if (x != y) return x < y ? -1 : 1;
    }
    if (la != lb) return la < lb ? -1 : 1;
    for (uint32_t j = 0; j < n; j++) {
        const float x = T.mods[oa + j], y = T.mods[ob + j];
        if (x < y) return -1;
        if (x > y) return 1;
        if (!(x == y)) return 0;
    }
    const int c = dg_cmp_opt(T.nterm[a], T.nterm[b]);
    return c ? c : dg_cmp_opt(T.cterm[a], T.cterm[b]);
}

// The merge-sort order of the rows of equal-mono runs: mono (total_cmp), then initial_sort; the sort is stable, so full ties keep the
// concatenation order (chunk order, then PeptideIx order within a chunk), which is the reference's.
struct PfRowLess {
    PfRows T;
    __device__ bool operator()(uint32_t a, uint32_t b) const {
        const uint32_t ka = f32_ukey(T.mono[a]), kb = f32_ukey(T.mono[b]);
        if (ka != kb) return ka < kb;
        return pf_initial_sort(T, a, b) < 0;
    }
};

// reorder_peptides' merge test (database.rs:236-248): mono, sequence, modifications, nterm and cterm equal under IEEE == (None == None).
__device__ bool pf_row_equal(const PfRows& T, uint32_t a, uint32_t b) {
    if (!(T.mono[a] == T.mono[b])) return false;
    const uint32_t oa = T.res_off[a], ob = T.res_off[b], L = T.res_off[a + 1] - oa;
    if (T.res_off[b + 1] - ob != L) return false;
    for (uint32_t j = 0; j < L; j++)
        if (T.seq[oa + j] != T.seq[ob + j] || !(T.mods[oa + j] == T.mods[ob + j])) return false;
    const float na = T.nterm[a], nb = T.nterm[b], ca = T.cterm[a], cb = T.cterm[b];
    return ((na != na && nb != nb) || na == nb) && ((ca != ca && cb != cb) || ca == cb);
}

__global__ void k_pf_merge_heads(PfRows T, const uint32_t* __restrict__ order, uint32_t N, uint32_t* __restrict__ head) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) head[i] = (i == 0 || !pf_row_equal(T, order[i - 1], order[i])) ? 1u : 0u;
}

// Per peptide (rows [first[k], first[k + 1]) of the sorted order): residue count and protein-reference count.
__global__ void k_pf_pep_counts(PfRows T, const uint32_t* __restrict__ order, const uint32_t* __restrict__ first, uint32_t n_pep,
                                uint64_t* __restrict__ n_res, uint64_t* __restrict__ n_ref) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_pep) return;
    uint64_t refs = 0;
    for (uint32_t i = first[k]; i < first[k + 1]; i++) refs += T.ref_off[order[i] + 1] - T.ref_off[order[i]];
    n_ref[k] = refs;
    const uint32_t r0 = order[first[k]];
    n_res[k] = T.res_off[r0 + 1] - T.res_off[r0];
}

// The output row of each peptide: the first row's fields, decoy the AND over the merged rows, protein ids concatenated in row order
// (sorted per peptide afterwards).
__global__ void k_pf_export(PfRows T, const uint32_t* __restrict__ order, const uint32_t* __restrict__ first, uint32_t n_pep,
                            const uint32_t* __restrict__ res_off, const uint32_t* __restrict__ ref_off, uint8_t* __restrict__ o_seq, float* __restrict__ o_mods,
                            float* __restrict__ o_nterm, float* __restrict__ o_cterm, float* __restrict__ o_mono, uint8_t* __restrict__ o_decoy,
                            uint8_t* __restrict__ o_missed, uint8_t* __restrict__ o_semi, uint32_t* __restrict__ o_ids) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_pep) return;
    const uint32_t r0 = order[first[k]], o = res_off[k];
    for (uint32_t a = T.res_off[r0], b = 0; a < T.res_off[r0 + 1]; a++, b++) {
        o_seq[o + b] = T.seq[a];
        o_mods[o + b] = T.mods[a];
    }
    o_nterm[k] = T.nterm[r0];
    o_cterm[k] = T.cterm[r0];
    o_mono[k] = T.mono[r0];
    o_missed[k] = T.missed[r0];
    o_semi[k] = T.semi[r0];
    bool decoy = true;
    uint32_t at = ref_off[k];
    for (uint32_t i = first[k]; i < first[k + 1]; i++) {
        const uint32_t r = order[i];
        decoy = decoy && T.decoy[r];
        for (uint32_t q = T.ref_off[r]; q < T.ref_off[r + 1]; q++) o_ids[at++] = T.ids[q];
    }
    o_decoy[k] = decoy ? 1 : 0;
}

}  // namespace sb
