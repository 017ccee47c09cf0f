// device_common.cuh — shared device-side definitions for the sage_b200 kernels (sm_90a, H100).
//
// Numeric contract (SURVEY.md §7 hard part 2): every f32 product / sum / quotient on the path is a separately
// rounded IEEE operation, exactly as rustc emits for the reference (no FMA contraction). We use the explicit
// round-to-nearest intrinsics AND compile with -fmad=false.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sb {

constexpr int K_MAX = 128;            // max preliminary candidates kept per spectrum: max(50, 2*report_psms)
constexpr uint32_t NARROW_CAP = 8192; // precursor windows up to this many peptides are counted in shared memory
constexpr int PRELIM_THREADS = 256;
constexpr int PRELIM_CTAS = 6;              // CTAs per SM of k_prelim_narrow (a persistent grid over its work list)
constexpr int SCORE_THREADS = 128;  // chosen by A/B on cfg2 against 64 and 256; must stay >= K_MAX for the rank sort
#ifndef SAGE_B200_SCORE_MIN_CTAS
#define SAGE_B200_SCORE_MIN_CTAS 10
#endif
constexpr int SCORE_MIN_CTAS = SAGE_B200_SCORE_MIN_CTAS;   // k_score CTAs per SM the register budget is held to (chosen by A/B on cfg2)
#ifndef SAGE_B200_SCORE_TILE
#define SAGE_B200_SCORE_TILE 1024
#endif
#ifndef SAGE_B200_SCORE_UNROLL
#define SAGE_B200_SCORE_UNROLL 1
#endif
#ifndef SAGE_B200_SCORE_MIN_CTAS_SPLIT
#define SAGE_B200_SCORE_MIN_CTAS_SPLIT 11   /* 40 registers, no spills; measured on cfg2, H100 SXM at 700 W on the kernel of that time (score phase, ms): 10 -> 1.176, 11 -> 1.141 (12 compiles to the same 40 registers) */
#endif
constexpr int SCORE_MIN_CTAS_SPLIT = SAGE_B200_SCORE_MIN_CTAS_SPLIT;   // k_score<true> keeps no records / order / marks in shared memory
constexpr uint32_t SCORE_UNROLL = SAGE_B200_SCORE_UNROLL;   // tasks per lane and iteration of k_score's phase B (1 or 2; chosen by A/B on cfg2)
constexpr uint32_t SCORE_TILE = SAGE_B200_SCORE_TILE;      // tasks (theoretical-fragment lookups) per shared-memory tile of k_score (multiple of 256)
constexpr int MAX_KINDS = 6;
// k_prelim_narrow_warp: cap 1024 x 2 warps x 24 CTAs/SM, chosen by A/B on cfg2 against caps 256..2048 and 4 / 8 warps per CTA (cap 2048:
// its 192 KB of shared memory per SM leaves too little L1 for the index lines)
constexpr uint32_t WARPQ_CAP = 1024;       // precursor windows up to this many peptides are counted by one warp (u16 counts: 2 KB of smem per warp)
constexpr int WARPQ_WARPS = 2;             // queries (warps) per CTA of k_prelim_narrow_warp
constexpr int WARPQ_MIN_CTAS = 24;         // CTAs per SM the register budget is held to
constexpr uint32_t PEP_LUT_CELLS = 65536;
constexpr uint32_t BUCKET_LUT_CELLS = 32768;   // ~5 cells per page on a 2M-peptide index: the LUT start is within one page of the answer

// mass.rs:5-8
constexpr float PROTON = 1.0072764f;
constexpr float NEUTRON = 1.00335f;

struct Tol { int kind; float lo, hi; };

// f32::total_cmp as an integer key
__device__ __forceinline__ int f32_key(float x) {
    int b = __float_as_int(x);
    return b ^ (int)(((unsigned)(b >> 31)) >> 1);
}

// x / c, correctly rounded, for the two constants of Tolerance::bounds (1e6, 100): q0 = x * rn(1/c), one FMA for the exact residual, one FMA
// to correct. Bit-identical to IEEE division for EVERY float with 1e-20 <= |x| <= 1e30 (exhaustively checked against x / c on the CPU by
// tests/test_div_const.py: 1.39e9 values per constant); anything outside that range takes the real division.
__device__ __forceinline__ float div_const_rn(float x, float c, float rc) {
    const float ax = fabsf(x);
    if (ax >= 1e-20f && ax <= 1e30f) {
        const float q0 = __fmul_rn(x, rc);
        return __fmaf_rn(__fmaf_rn(-q0, c, x), rc, q0);
    }
    return __fdiv_rn(x, c);
}

// Tolerance::bounds (mass.rs:21-35)
__device__ __forceinline__ void tol_bounds(const Tol& t, float c, float& lo, float& hi) {
    if (t.kind == 0) {
        lo = __fadd_rn(c, div_const_rn(__fmul_rn(c, t.lo), 1000000.0f, 1.0f / 1000000.0f));
        hi = __fadd_rn(c, div_const_rn(__fmul_rn(c, t.hi), 1000000.0f, 1.0f / 1000000.0f));
    } else if (t.kind == 1) {
        lo = __fadd_rn(c, div_const_rn(__fmul_rn(c, t.lo), 100.0f, 1.0f / 100.0f));
        hi = __fadd_rn(c, div_const_rn(__fmul_rn(c, t.hi), 100.0f, 1.0f / 100.0f));
    } else {
        lo = __fadd_rn(c, t.lo);
        hi = __fadd_rn(c, t.hi);
    }
}

// binary_search_slice (database.rs:549-561) over an abstract sorted sequence.
//   less_lo(i): key(slice[i], low) == Less        le_hi(i): key(slice[i], high) != Greater
template <class LessLo, class LeHi>
__device__ __forceinline__ void binary_search_slice(uint32_t n, LessLo less_lo, LeHi le_hi, uint32_t& left, uint32_t& right) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        uint32_t mid = lo + ((hi - lo) >> 1);
        if (less_lo(mid)) lo = mid + 1; else hi = mid;
    }
    left = lo == 0 ? 0 : lo - 1;
    lo = left; hi = n;
    while (lo < hi) {
        uint32_t mid = lo + ((hi - lo) >> 1);
        if (le_hi(mid)) lo = mid + 1; else hi = mid;
    }
    right = lo;
}

// max_fragment_charge (scoring.rs:239-247); opt < 0 == None. Returns the EXCLUSIVE upper bound of 1..N.
__device__ __forceinline__ uint32_t max_fragment_charge(int opt, uint32_t precursor_charge) {
    uint32_t m = opt >= 0 ? (uint32_t)(opt + 1) : precursor_charge;
    m &= 0xFF;  // u8 arithmetic in the reference (c + 1 on u8)
    uint32_t r = precursor_charge < m ? precursor_charge : m;
    return r < 2 ? 2 : r;
}

// PreScore (scoring.rs:43-49) packed so that u64 order == derived lexicographic Ord:
//   matched:u16 | peptide:u32 | precursor_charge:u8 | isotope_error:i8 (biased)
__device__ __forceinline__ uint64_t prescore_key(uint32_t matched, uint32_t peptide, uint32_t charge, int iso) {
    return ((uint64_t)matched << 48) | ((uint64_t)peptide << 16) | ((uint64_t)(charge & 0xFF) << 8) | (uint64_t)((uint32_t)(iso + 128) & 0xFF);
}
constexpr uint64_t PRESCORE_DEFAULT = ((uint64_t)0xFFFFFFFFull << 16) | 128ull;  // matched 0, PeptideIx::default()==MAX, charge 0, iso 0
__device__ __forceinline__ uint32_t key_matched(uint64_t k) { return (uint32_t)(k >> 48); }
__device__ __forceinline__ uint32_t key_peptide(uint64_t k) { return (uint32_t)(k >> 16); }
__device__ __forceinline__ uint32_t key_charge(uint64_t k) { return (uint32_t)(k >> 8) & 0xFF; }
__device__ __forceinline__ int key_iso(uint64_t k) { return (int)(k & 0xFF) - 128; }

// sift_down (heap.rs:40-60) on a min-heap of packed PreScore keys
__device__ __forceinline__ void sift_down(uint64_t* s, uint32_t len, uint32_t index) {
    while (index * 2 + 1 < len) {
        uint32_t smallest = index, l = index * 2 + 1, r = index * 2 + 2;
        if (s[l] < s[smallest]) smallest = l;
        if (r < len && s[r] < s[smallest]) smallest = r;
        if (smallest != index) {
            uint64_t t = s[smallest]; s[smallest] = s[index]; s[index] = t;
            index = smallest;
        } else break;
    }
}
// bounded_min_heapify (heap.rs:7-28), sequential (one thread), used on short lists
__device__ __forceinline__ void bounded_min_heapify_seq(uint64_t* s, uint32_t len, uint32_t k) {
    if (len <= k) return;
    for (uint32_t i = k / 2; i-- > 0;) sift_down(s, k, i);
    for (uint32_t i = k; i < len; i++) {
        if (s[i] > s[0]) {
            uint64_t t = s[i]; s[i] = s[0]; s[0] = t;
            sift_down(s, k, 0);
        }
    }
}

struct QueryDesc {
    uint32_t pre_lo;     // IndexedQuery::pre_idx_lo
    uint32_t pre_hi;     // IndexedQuery::pre_idx_hi
    uint32_t potential;  // pre_idx_hi - pre_idx_lo + 1 (scoring.rs:351); 0 = query slot unused
    uint32_t eff_lo;     // inclusive PeptideIx range accepted by the edge filter (database.rs:526-531)
    uint32_t eff_hi;     // eff_lo > eff_hi => nothing accepted
    uint8_t charge;      // precursor charge of this query
    int8_t iso;          // isotope error recorded in PreScore
    uint8_t nfc;         // fragment charges searched = max_fragment_charge - 1
    uint8_t mode;        // 0 unused, 1 narrow/index (smem counts), 2 wide (global counts), 3 narrow/peptide-centric
};

struct QueryHits {
    uint32_t n;            // explicit entries in keys[]
    uint32_t default_run;  // matched_peaks == 0: the untrimmed all-default Vec of this length (scoring.rs:376-378)
    uint32_t matched_peaks;
    uint32_t scored_candidates;
};

// ---- bulk asynchronous copy (TMA 1-D, cp.async.bulk) + mbarrier helpers (sm_90a). Used to stage spectrum peaks into shared memory.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");   // make the init visible to the async proxy
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// global -> shared bulk copy; src/dst 16-byte aligned, bytes a multiple of 16; completion is signalled on `bar` (complete_tx)
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes),
                 "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    }
}

// One ordered key list awaiting its exact heap replay (k_replay)
struct ReplaySlot { unsigned long long off; uint32_t item, n_list, state /*0 = replay pending, 1 = nothing to do*/, k; };

// Device counters (u64 slots)
enum { C_TASKS = 0, C_PAGES, C_ENTRIES, C_MATCHED, C_CANDS, C_PEPFLOATS, C_PSMS, C_QUERIES, C_WIDE, C_MAXPOT, C_WORK, C_ERR, C_PEPQ, C_PEPFALLBACK, C_WSLOT, C_WOVERFLOW, C_FRAGS,
       C_NLIST /* bump cursor of the narrow key-list arena */, C_NCTA /* queries listed in cta_items */, C_NLIST_NEED /* arena entries this chunk needs (exact upper bound) */,
       C_HITS /* bump cursor of the split scorer's hit arena (entries reserved = tasks of the spectrum) */,
       C_EXACT /* narrow queries listed in exact_items (>= 2^16 matches: recounted exactly by k_prelim_exact) */, C_COUNT };

struct DbView {
    const uint2* frag;        // {peptide_index, fragment_mz bits}, reference bucket layout
    const float* bucket_min;
    const float* pep_mono;
    const uint32_t* ion_off;  // n_pep+1, offsets into ions (n_kinds*(L-1) floats per peptide)
    const float* ions;
    const uint8_t* pep_len;
    const uint8_t* pep_flags; // bit0 decoy
    const uint8_t* pep_missed;
    uint32_t n_pep, n_bucket, bucket_size, n_kinds;
    uint32_t min_ion_index;   // fragments in the index are ions with index > min_ion_index (database.rs:281-291)
    uint32_t pep_centric_ok;  // index content verified == ions filtered by min_ion_index (peptide-centric counting allowed)
    uint32_t nterm_mask;      // bit k set when ion kind k is an N-terminal series (a/b/c)
    // search directories (results identical to the plain binary searches; nullptr = not built)
    const uint16_t* page_grid;  // [n_bucket][grid_n + 1]: page_grid[p][g] = #{entries of page p with PeptideIx < (g << grid_shift)}
    uint32_t grid_shift, grid_n;
    const uint32_t* bucket_lut; // [BUCKET_LUT_CELLS]: #{bucket_min < edge(c)}, conservative start for the bucket search
    float blut_base, blut_inv_w;
    const uint32_t* pep_lut;    // [PEP_LUT_CELLS + 1]: #{pep_mono < edge(c)} (last entry n_pep): brackets the precursor-window searches of k_setup_queries
    float plut_base, plut_inv_w;
    uint64_t n_frag;
    uint8_t kinds[MAX_KINDS];
};

// Secondary index for open search (k_prelim_wide): the same fragments grouped by PEPTIDE BLOCK (`block` consecutive PeptideIx == one
// shared-memory count tile) and sorted by m/z inside a block, so the entries matching one (peak, charge) probe inside one tile are a single
// contiguous run found through a per-block m/z LUT — instead of filtering every entry of the page slices (database.rs:514-534 visits ~9x more
// entries than match). Built lazily per db the first time a scorer meets a window wider than NARROW_CAP (sage_b200.cu: db_wide_index).
// Blocks hold ~2 M entries here, so a 2^18-cell u32 LUT per block is small next to them; narrow windows use NarrowIndexView instead.
struct WideIndexView {
    const uint2* frag;        // {PeptideIx, m/z bits}, block-major, ascending m/z inside a block; nullptr = not built (page-slice streaming is used)
    const uint64_t* blk_off;  // [n_block + 1]
    const uint32_t* lut;      // [n_block][cells + 1]: #{entries of the block with m/z < base + c / inv_w}
    uint32_t block, n_block, cells;
    float base, inv_w;
};

// Index copy for narrow precursor windows (k_prelim_narrow_warp<true>, k_prelim_narrow): the fragments grouped by blocks of `block` (<= 65536)
// consecutive PeptideIx, ascending m/z inside a block, as two parallel arrays — the m/z values alone (a run walk compares only these, 8 per
// 32-byte sector) and the PeptideIx offset within the block (read only for entries inside the probe's m/z bounds). Per block an m/z directory
// of `cells` u16 cells, about one per entry, so that the part of the directory that the resident queries touch stays in L2. Built lazily by
// the first narrow-search chunk (sage_b200.cu: db_narrow_index).
constexpr uint32_t NARROW_GROUP = 64;   // directory cells per u32 group base
struct NarrowIndexView {
    const float* mz;          // block-major, ascending m/z inside a block; nullptr = not built (the page index is probed instead)
    const uint16_t* pep;      // PeptideIx - block index * block, parallel to mz
    const uint64_t* blk_off;  // [n_block + 1]
    // start of the run of m/z >= edge(c), edge(c) = base + c / inv_w, as an entry of the block: grp[c / NARROW_GROUP] + dir[c]. Both count the
    // block's entries with m/z < the edge (grp at the group's first cell); dir is clamped to 65535, which can only move a start earlier.
    const uint16_t* dir;      // [n_block][cells]
    const uint32_t* grp;      // [n_block][cells / NARROW_GROUP]
    uint32_t block, n_block, cells;
    float base, inv_w;
};

struct ScorerView {
    Tol precursor_tol, fragment_tol;
    uint32_t min_matched_peaks;
    int min_iso, max_iso;
    uint32_t min_charge, max_charge;
    int override_charge, max_fragment_charge_opt, chimera, wide_window, annotate, score_type;
    uint32_t report_psms;
    uint32_t kparam;   // max(50, 2*report_psms)
    uint32_t n_iso;    // isotope errors folded per charge (1 when min==max)
    uint32_t n_ch_max; // charges folded per spectrum (upper bound)
    uint32_t qmax;     // n_iso * n_ch_max query slots per spectrum
    uint32_t lcap;     // list capacity for merges
    uint32_t pep_cap;  // precursor windows up to this many peptides use the peptide-centric kernel path (0 = never)
    uint32_t wide_tile;        // peptides per shared-memory tile of the wide kernel
    uint32_t wide_variant;     // A/B switch for the wide streaming filter (1 = m/z window as one unsigned compare)
    uint32_t wide_lmax;        // survivor-list capacity per query (<= WIDE_LMAX; smaller only in tests)
    const double* lnfact_tab;  // lnfact(n) for n < lnfact_n, computed on the host with libm log (scoring.rs:170-177)
    uint32_t lnfact_n;
    uint32_t log_variant;      // which build of glibc's log() the device reproduces (glibc_log.cuh): 0 = FMA-contracted, 1 = plain
    uint32_t score_fast;       // 1 (default): straight-line task body of k_score where its preconditions hold; 0: always the generic body (tests)
};

struct BatchView {
    uint32_t n;                 // spectra in this chunk
    uint32_t spectrum_base;     // index of the chunk's first spectrum in the caller's batch (Feature.spectrum is batch-relative)
    const uint32_t* peak_off;   // n+1
    const float* masses;
    const float* intens;
    const float* prec_mz;
    const uint8_t* prec_charge;
    const float* iso_lo;        // nullable
    const float* iso_hi;
    const float* tic;
    const float* rt;            // nullable
    const float* ims;           // nullable
    const uint32_t* order;      // spectrum processing order (ascending precursor window) for L2 locality; nullable = identity
    QueryDesc* queries;         // n * qmax
    QueryHits* hits;            // n * qmax
    uint64_t* hit_keys;         // n * qmax * kparam
    unsigned long long* counters;
    // Device-side work lists sized from what earlier chunks needed (no host round trip inside a chunk): when a capacity turns out too
    // small the affected queries produce no hits, the host sees need > capacity in the counters and re-runs the chunk with exact sizes.
    uint32_t* wide_items;             // compacted item ids of the open-search (mode 2) queries, wide_cap entries
    uint32_t* cta_items;              // compacted item ids of the narrow queries counted by a whole CTA (modes 1 and 3), n * qmax entries
    uint32_t* exact_items;            // item ids of the narrow queries with >= 2^16 matches (k_prelim_exact), n * qmax entries
    ReplaySlot* nslots;               // one per item (narrow kernels); k_setup_queries resets them to "nothing to replay"
    uint32_t wide_cap;
    unsigned long long nlist_cap;     // entries in the narrow key-list arena
};

}  // namespace sb
