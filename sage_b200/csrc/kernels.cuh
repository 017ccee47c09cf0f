// kernels.cuh — hand-written sm_90a (H100) kernels for the fragment-index search-and-score path.
//
//   k_setup_queries   IndexedDatabase::query per (spectrum, charge, isotope)      database.rs:402-425, scoring.rs:418-458
//   k_prelim_narrow   matched_peaks_with_isotope (counting), counts in smem, emits the ordered key list    scoring.rs:335-375, database.rs:480-536
//   k_prelim_wide     same for precursor windows > NARROW_CAP (open search): tiled smem counts, streamed page slices
//   k_replay          trim_hits == bounded_min_heapify + truncate, one thread per query                       scoring.rs:322-329, heap.rs:7-60
//   k_score           fold/trim of per-query hits, score_candidate, build_features, chimera loop, Fragments, quick_score   scoring.rs:255-767
//   k_process_ms2     SpectrumProcessor::process for MS2 (deisotope, top-N, sort, TIC)                          spectrum.rs:179-412
//   k_build_* / k_gen_fragments / k_bucket_keys ...  Parameters::build_from_peptides + search directories     database.rs:265-365
//
// All of this is integer/f32 gather-reduce work bound by memory latency/bandwidth; tensor cores are not used.
#pragma once
#include <type_traits>

#include "device_common.cuh"
#include "glibc_log.cuh"

// Paths k_score rarely takes (the generic peak lookup of unsorted spectra, the warp-per-candidate scorer that only serves remove_matched_peaks,
// the Fragments writer): kept out of line so that the hot loop's code stays compact in the instruction cache (chosen by A/B).
#ifndef SAGE_B200_RARE_NOINLINE
#define SAGE_B200_RARE_NOINLINE 0
#endif
#if SAGE_B200_RARE_NOINLINE
#define SB_RARE __noinline__
#else
#define SB_RARE __forceinline__
#endif

namespace sb {

// ------------------------------------------------------------------------------------------------ setup
// One thread per spectrum: enumerate the (charge, isotope) queries of Scorer::initial_hits and resolve each
// precursor window to a PeptideIx range (two binary searches over peptides[].monoisotopic).
// #{i : mono[i] < x} (le == false) or #{i : mono[i] <= x} (le == true) in f32::total_cmp order. The LUT cell of x brackets the answer to three
// cells (one early / one late absorb the float rounding of the cell index), the binary search over the bracket uses the exact keys.
__device__ __forceinline__ uint32_t pep_partition(const DbView& db, float x, bool le) {
    uint32_t lo = 0, hi = db.n_pep;
    if (db.pep_lut != nullptr) {
        const float t = (x - db.plut_base) * db.plut_inv_w;
        if (t == t) {
            const int c = (int)fminf(fmaxf(floorf(t), -2.0f), (float)PEP_LUT_CELLS + 2.0f);
            lo = __ldg(db.pep_lut + min(max(c - 1, 0), (int)PEP_LUT_CELLS));
            hi = __ldg(db.pep_lut + min(max(c + 2, 0), (int)PEP_LUT_CELLS));
        }
    }
    const int kx = f32_key(x);
    while (lo < hi) {
        const uint32_t mid = lo + ((hi - lo) >> 1);
        const int k = f32_key(__ldg(db.pep_mono + mid));
        if (le ? k <= kx : k < kx) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__global__ void k_setup_queries(DbView db, ScorerView sc, BatchView b, uint32_t* sort_key, uint32_t* sort_val) {
    // The chunk-wide sums below go through one atomic per CTA: 50 000 threads adding to the same cache line cost ~85 us of a 100 us kernel
    // (the L2 atomic unit serialises per address, ~0.85 cycles per lane).
    __shared__ unsigned long long s_sum[4][8];   // [nq, list_need, npepq, maxpot][warp]
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long nq = 0, nwide = 0, maxpot = 0, npepq = 0, list_need = 0, ncta = 0;
    if (s < b.n) {
    const float pmz = b.prec_mz[s];
    const uint32_t known = b.prec_charge[s];
    const float mz = __fsub_rn(pmz, PROTON);  // scoring.rs:420
    const bool fold = sc.wide_window || !(known != 0 && !sc.override_charge);
    uint32_t c0 = fold ? sc.min_charge : known;
    uint32_t c1 = fold ? sc.max_charge : known;
    QueryDesc* out = b.queries + (size_t)s * sc.qmax;
    uint32_t qi = 0;
    for (uint32_t z = c0; z <= c1 && qi < sc.qmax; z++) {
        const float precursor_mass = __fmul_rn(mz, (float)z);
        Tol ptol = sc.precursor_tol;
        if (sc.wide_window) {  // scoring.rs:428-431: isolation_window.unwrap_or(Da(-2.4,2.4)) * charge
            float lo = -2.4f, hi = 2.4f;
            if (b.iso_lo != nullptr && !isnan(b.iso_lo[s]) && !isnan(b.iso_hi[s])) { lo = b.iso_lo[s]; hi = b.iso_hi[s]; }
            ptol.kind = 2;
            ptol.lo = __fmul_rn(lo, (float)z);
            ptol.hi = __fmul_rn(hi, (float)z);
        }
        const uint32_t mfc = max_fragment_charge(sc.max_fragment_charge_opt, z);
        for (uint32_t ii = 0; ii < sc.n_iso; ii++, qi++) {
            // scoring.rs:391-415: isotope 0 is used whenever min == max
            const int iso = (sc.min_iso != sc.max_iso) ? sc.min_iso + (int)ii : 0;
            const float qmass = __fsub_rn(precursor_mass, __fmul_rn((float)iso, NEUTRON));  // scoring.rs:344
            float plo, phi;
            tol_bounds(ptol, qmass, plo, phi);
            // binary_search_slice (database.rs:549-561): left = partition_point(< lo).saturating_sub(1); right = left + partition_point(
            // slice[left..], <= hi) = max(left, global partition_point(<= hi))
            const uint32_t ppl = pep_partition(db, plo, false);
            const uint32_t left = ppl == 0 ? 0 : ppl - 1;
            const uint32_t right = max(left, pep_partition(db, phi, true));
            QueryDesc q;
            q.pre_lo = left;
            q.pre_hi = right;
            q.potential = right - left + 1;
            const bool lo_ok = left < db.n_pep && __ldg(db.pep_mono + left) >= plo;
            const bool hi_ok = right < db.n_pep && __ldg(db.pep_mono + right) <= phi;
            const long long elo = (long long)left + (lo_ok ? 0 : 1);
            const long long ehi = (long long)right - (hi_ok ? 0 : 1);
            if (ehi < elo) { q.eff_lo = 1; q.eff_hi = 0; } else { q.eff_lo = (uint32_t)elo; q.eff_hi = (uint32_t)ehi; }
            q.charge = (uint8_t)z;
            q.iso = (int8_t)iso;
            q.nfc = (uint8_t)(mfc - 1);
            // 2 = open search (k_prelim_wide), 3 = peptide-centric CTA, 4 = one warp per query (k_prelim_narrow_warp), 1 = one CTA per query
            q.mode = q.potential > NARROW_CAP ? 2 : ((db.pep_centric_ok && q.potential <= sc.pep_cap) ? 3 : (q.potential <= WARPQ_CAP ? 4 : 1));
            out[qi] = q;
            if (q.mode != 2 && q.potential > sc.kparam) list_need += q.potential;   // k_prelim_narrow reserves exactly this much of the arena
            if (q.mode == 4) b.counters[C_COUNT + qi] = 1ull;   // query slot qi is in use by some warp-counted query (benign race: everybody stores 1)
            ncta += (q.mode == 1 || q.mode == 3);
            nq++;
            if (q.mode == 2) {   // "no hits" until k_prelim_wide gets to it (it may not, when wide_cap is too small: the host then re-runs the chunk)
                nwide++;
                QueryHits h0; h0.n = 0; h0.default_run = q.potential; h0.matched_peaks = 0; h0.scored_candidates = 0;
                b.hits[(size_t)s * sc.qmax + qi] = h0;
            }
            if (q.mode == 3) npepq++;
            if (q.potential > maxpot) maxpot = q.potential;
        }
    }
    for (; qi < sc.qmax; qi++) {
        QueryDesc q = {};
        out[qi] = q;
    }
    if (sort_key) { sort_key[s] = out[0].mode ? out[0].pre_lo : 0xFFFFFFFFu; sort_val[s] = s; }
    if (nwide) {   // compact work list of the open-search queries (one reservation per spectrum)
        unsigned long long w = atomicAdd(b.counters + C_WIDE, nwide);
        for (uint32_t j = 0; j < sc.qmax; j++)
            if (out[j].mode == 2) { if (w < b.wide_cap) b.wide_items[w] = s * sc.qmax + j; w++; }
    }
    if (ncta) {
        unsigned long long w = atomicAdd(b.counters + C_NCTA, ncta);
        for (uint32_t j = 0; j < sc.qmax; j++)
            if (out[j].mode == 1 || out[j].mode == 3) b.cta_items[w++] = s * sc.qmax + j;
    }
    for (uint32_t j = 0; j < sc.qmax; j++) {
        ReplaySlot rs; rs.off = 0; rs.item = s * sc.qmax + j; rs.n_list = 0; rs.state = 1; rs.k = 0;
        b.nslots[(size_t)s * sc.qmax + j] = rs;
    }
    }
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int o = 16; o > 0; o >>= 1) {
        nq += __shfl_down_sync(0xffffffffu, nq, o);
        list_need += __shfl_down_sync(0xffffffffu, list_need, o);
        npepq += __shfl_down_sync(0xffffffffu, npepq, o);
        maxpot = max(maxpot, __shfl_down_sync(0xffffffffu, maxpot, o));
    }
    if (lane == 0) { s_sum[0][warp] = nq; s_sum[1][warp] = list_need; s_sum[2][warp] = npepq; s_sum[3][warp] = maxpot; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (uint32_t w = 1; w < (blockDim.x >> 5); w++) {
            nq += s_sum[0][w]; list_need += s_sum[1][w]; npepq += s_sum[2][w]; maxpot = max(maxpot, s_sum[3][w]);
        }
        if (nq) atomicAdd(b.counters + C_QUERIES, nq);
        if (list_need) atomicAdd(b.counters + C_NLIST_NEED, list_need);
        if (npepq) atomicAdd(b.counters + C_PEPQ, npepq);
        if (maxpot) atomicMax(b.counters + C_MAXPOT, maxpot);
    }
}


// --------------------------------------------------------------------------------------------- block helpers
__device__ __forceinline__ uint32_t block_sum_u32(uint32_t v, uint32_t* s_warp) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) s_warp[warp] = v;
    __syncthreads();
    uint32_t t = 0;
    for (uint32_t w = 0; w < nwarps; w++) t += s_warp[w];
    __syncthreads();
    return t;
}

// ------------------------------------------------------------------------------------------- sorted-array bucket LUT
// Membership tests against a sorted f32 array (spectrum peaks, or per-charge tolerance bounds) dominate the instruction count
// of this path. A 256-cell LUT over the array's value range gives a conservative lower bound of lower_bound(arr, x) in O(1);
// callers then advance linearly comparing the ACTUAL array values, so results stay exact.  start[c] = #{i : arr[i] < edge(c)},
// edge(c) = base + c*w (c >= 1), start[0] = 0.
constexpr uint32_t LUT_CELLS = 256;        // per-charge bound arrays of the peptide-centric prelim path
constexpr uint32_t SPEC_LUT_CELLS = 1024;  // spectrum peak LUT of k_score (~0.2 peaks per cell at 200 peaks)
struct LutParams { float base, inv_w; };

__device__ __forceinline__ LutParams lut_params(float first, float last, uint32_t cells = LUT_CELLS) {
    LutParams L;
    L.base = first;
    const float w = (last - first) / (float)cells;
    L.inv_w = (w > 0.0f && w < 3.0e38f) ? 1.0f / w : 0.0f;
    return L;
}
__device__ __forceinline__ float lut_edge(const LutParams& L, uint32_t c) { return L.inv_w > 0.0f ? L.base + (float)c * (1.0f / L.inv_w) : L.base; }
// Cooperative build: threads [t0, t0+stride, ...) fill start[0..LUT_CELLS)
__device__ __forceinline__ void lut_build(const float* arr, uint32_t n, const LutParams& L, uint16_t* start, uint32_t t0, uint32_t stride,
                                          uint32_t cells = LUT_CELLS) {
    for (uint32_t c = t0; c < cells; c += stride) {
        uint32_t lo = 0;
        if (c > 0 && L.inv_w > 0.0f) {
            const float e = lut_edge(L, c);
            uint32_t hi = n;
            while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (arr[m] < e) lo = m + 1; else hi = m; }
        }
        start[c] = (uint16_t)lo;
    }
}
// Same table for an ASCENDING array that carries a +inf sentinel at arr[n]: every thread owns a run of consecutive cells, finds the first
// one's count by binary search and walks forward for the others (start[c] is non-decreasing in c). O(cells / threads * log n + n) per thread
// with uniform trip counts; the values are those of lut_build by construction (same edge expression, same `<`). STRIDE = threads of the block.
template <uint32_t STRIDE>
__device__ __forceinline__ void lut_build_walk(const float* arr, uint32_t n, const LutParams& L, uint16_t* start, uint32_t t0, uint32_t cells) {
    const uint32_t per = (cells + STRIDE - 1) / STRIDE;
    const uint32_t c0 = t0 * per, c1 = min(cells, c0 + per);
    if (!(L.inv_w > 0.0f)) {
        for (uint32_t c = c0; c < c1; c++) start[c] = 0;
        return;
    }
    if (c0 >= c1) return;
    // lut_edge's cell width, divided once: the compiler keeps the IEEE division (reciprocal, refinement, slow-path test) inside the walk
    const float w = 1.0f / L.inv_w;
    uint32_t i = 0;
    if (c0 > 0) {
        const float e = L.base + (float)c0 * w;
        uint32_t hi = n;
        while (i < hi) { const uint32_t m = (i + hi) >> 1; if (arr[m] < e) i = m + 1; else hi = m; }
    }
    start[c0] = (uint16_t)i;
    for (uint32_t c = c0 + 1; c < c1; c++) {
        const float e = L.base + (float)c * w;
        while (arr[i] < e) i++;   // arr[n] = +inf stops the walk
        start[c] = (uint16_t)i;
    }
}
// A position s with arr[i] < x for all i < s (conservative: one cell early to absorb float rounding of the cell index).
__device__ __forceinline__ uint32_t lut_start(const LutParams& L, const uint16_t* start, float x, uint32_t cells = LUT_CELLS) {
    const float t = (x - L.base) * L.inv_w;
    int c = t > 1.0f ? (int)fminf(t, (float)(cells - 1)) - 1 : 0;
    return start[c];
}

// binary_search_slice(min_value, flo, fhi) (database.rs:487-492) -> [left, right) pages; uses the m/z LUT when built.
__device__ __forceinline__ void bucket_range(const DbView& db, float flo, float fhi, uint32_t& left, uint32_t& right) {
    if (db.bucket_lut == nullptr) {
        const int klo = f32_key(flo), khi = f32_key(fhi);
        binary_search_slice(db.n_bucket, [&](uint32_t i) { return f32_key(__ldg(db.bucket_min + i)) < klo; },
                            [&](uint32_t i) { return f32_key(__ldg(db.bucket_min + i)) <= khi; }, left, right);
        return;
    }
    // bucket_min holds positive finite m/z values, so float compares equal total_cmp here
    const float t = (flo - db.blut_base) * db.blut_inv_w;
    const int c = t > 1.0f ? (int)fminf(t, (float)(BUCKET_LUT_CELLS - 1)) - 1 : 0;
    const uint32_t pp0 = __ldg(db.bucket_lut + c);                        // <= partition_point(min < flo)
    // partition_point(min < flo): the element that stops the scan is min[pp] itself, and (for flo <= fhi) min[pp - 1] < flo <= fhi needs
    // no second look, so the scan for `right` resumes at pp with the value already in hand
    uint32_t pp = pp0;
    float v = 0.0f;
    bool have = false;
    while (pp < db.n_bucket) {
        v = __ldg(db.bucket_min + pp);
        if (!(v < flo)) { have = true; break; }
        pp++;
    }
    left = pp == 0 ? 0 : pp - 1;
    uint32_t r;
    if (pp > 0 && flo <= fhi) {
        r = pp;
        if (have && v <= fhi) {
            r++;
            while (r < db.n_bucket && __ldg(db.bucket_min + r) <= fhi) r++;
        }
    } else {
        r = left;
        while (r < db.n_bucket && __ldg(db.bucket_min + r) <= fhi) r++;
    }
    right = r;
}

// lower_bound over the PeptideIx column of a page sub-range: first e in [lo, hi) with slice[e].x >= key
__device__ __forceinline__ uint32_t page_lower_bound(const uint2* slice, uint32_t lo, uint32_t hi, uint32_t key) {
    while (lo < hi) {
        const uint32_t mid = lo + ((hi - lo) >> 1);
        if (__ldg(&slice[mid].x) < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// partition_point(|e| e.peptide_index < key) inside one page; uses the per-page PeptideIx grid when built.
__device__ __forceinline__ uint32_t page_lower_bound_dir(const DbView& db, uint32_t page, const uint2* slice, uint32_t pn, uint32_t key) {
    uint32_t lo = 0, hi = pn;
    if (db.page_grid != nullptr) {
        const uint32_t g = min(key >> db.grid_shift, db.grid_n - 1);
        const uint16_t* G = db.page_grid + (size_t)page * (db.grid_n + 1) + g;
        lo = __ldg(G);
        hi = (key >> db.grid_shift) >= db.grid_n ? pn : (uint32_t)__ldg(G + 1);
    }
    while (lo < hi) {
        const uint32_t mid = lo + ((hi - lo) >> 1);
        if (__ldg(&slice[mid].x) < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// One (peak, fragment charge) probe of matched_peaks_with_isotope (scoring.rs:358-374) against the fragment index: pages from the
// bucket minima, per page the PeptideIx window (grid cell + short binary search, then the forward walk that ends exactly at
// inner_right, database.rs:506-511), exact filter (database.rs:514-534), shared-memory count increment (u16 pairs in cnt32).
// PreScore::matched is a u16 and the reference's release build does not check overflow: a slot's count wraps, and every match that finds
// it at 0 (the first, and the first after each wrap) counts the candidate again in scored_candidates (scoring.rs:363-372). The counting
// kernels keep two u16 counts per 32-bit word, where an even slot's overflow would carry into its neighbour. No slot can pass 2^16 unless
// the query has >= 2^16 matches in all, a sum the kernels count anyway: such queries are listed for k_prelim_exact, which counts their
// window again with one u32 per slot and rewrites their keys, so the common path keeps its registers.
constexpr uint32_t EXACT_TRIGGER = 0x10000u;
constexpr uint32_t EXACT_SEG = NARROW_CAP / 2;   // window slots k_prelim_exact counts per pass
// One match of window slot idx: a u16 half of a packed word, or (EXACT) a u32 per slot of the segment [s0, s0 + EXACT_SEG).
template <bool EXACT>
__device__ __forceinline__ void count_match(uint32_t* cnt32, uint32_t idx, uint32_t s0) {
    if (EXACT) {
        if (idx - s0 < EXACT_SEG) atomicAdd(&cnt32[idx - s0], 1u);
    } else {
        atomicAdd(&cnt32[idx >> 1], 1u << ((idx & 1) * 16));
    }
}
template <bool EXACT = false>
__device__ __forceinline__ void index_probe(const DbView& db, const QueryDesc& q, float flo, float fhi, uint32_t* cnt32, uint32_t& matched, uint32_t& pages,
                                            uint32_t& entries, uint32_t s0 = 0) {
    uint32_t bl, br;
    bucket_range(db, flo, fhi, bl, br);
    for (uint32_t page = bl; page < br; page++) {
        const uint64_t pbase = (uint64_t)page * db.bucket_size;
        const uint64_t pend = min(pbase + db.bucket_size, db.n_frag);
        const uint2* slice = db.frag + pbase;
        const uint32_t pn = (uint32_t)(pend - pbase);
        const uint32_t pp = page_lower_bound_dir(db, page, slice, pn, q.pre_lo);
        const uint32_t il = pp == 0 ? 0 : pp - 1;   // inner_left = partition_point(pep < pre_lo).saturating_sub(1)
        // the reference also visits entry il = pp - 1; its PeptideIx is < pre_lo <= eff_lo, so it can never pass the filter: it is counted
        // in `entries` below but not fetched, and the walk starts at the lower bound itself
        uint32_t e = pp;
        for (; e < pn; e++) {
            const uint2 f = __ldg(&slice[e]);
            if (f.x > q.pre_hi) break;
            const float fmz = __uint_as_float(f.y);
            if (f.x >= q.eff_lo && f.x <= q.eff_hi && fmz >= flo && fmz <= fhi) {
                count_match<EXACT>(cnt32, f.x - q.pre_lo, s0);
                matched++;
            }
        }
        pages++;
        entries += e - il;
    }
}

// The same probe against the NARROW BLOCK INDEX (a second copy of the fragments: blocks of `nv.block` consecutive PeptideIx, ascending m/z inside
// a block, device_common.cuh: NarrowIndexView). A precursor window of a few hundred peptides lies in one or two blocks, so a probe is: directory
// cell of `flo` (one cell early: float rounding) -> walk the block's m/z values until one is > fhi; an entry inside [flo, fhi] reads its
// PeptideIx offset and counts when the PeptideIx is in the window. Same matched set as index_probe by construction (every index entry with
// PeptideIx in the window lies in these blocks); two dependent loads before the walk instead of five, no page loop, no bisection.
//
// One warp = 32 probes of one query. Most walks are one or two entries, but a peak at a fragment mass that MANY peptides share (y1 of K / R, b2
// of frequent dipeptides) matches a run of up to a few hundred entries: walked by its own lane that run set the trip count of the whole warp
// (CPU statistics of cfg2: mean 3.5 loads per probe, mean of the per-warp maximum 24). So a lane walks at most WALK_SOLO entries alone; runs
// still open after that are finished by the whole warp, 32 consecutive entries per step (coalesced 128-byte reads of m/z).
// The reference's page / entry work counters are not produced on this path (sage_b200.cu: option "narrow_index").
#ifndef SAGE_B200_WALK_SOLO
#define SAGE_B200_WALK_SOLO 8
#endif
constexpr uint32_t WALK_SOLO = SAGE_B200_WALK_SOLO;
// A lane's walk is a chain of dependent loads (each entry decides whether the next is needed), so it issues the loads of WALK_STEP entries, m/z
// and PeptideIx offset, at once. Counting kernel, H100 SXM at 700 W (ms, cfg2): WALK_STEP 1: 0.638; 2: 0.595; 4: 0.582 but 28 bytes of register
// spills at the 40 registers WARPQ_MIN_CTAS allows. Reading the offset only for entries inside [flo, fhi] (one more dependent load per match)
// measured slower: 0.630 on cfg2 at WALK_STEP 3, 12.24 against 11.55 ms on cfg3; in the warp-wide walk as well (cfg3 12.53 ms), so both
// walks read the offset with the m/z value. WALK_SOLO re-measured with the batched walk: 4: 0.699, 8: 0.630, 16: 0.639.
constexpr uint32_t WALK_STEP = 2;
// Directory cell a probe starts from: one cell before the cell of `flo`, so that edge(c) <= flo despite the rounding of both computations
// (tests/test_narrow_directory.py restates them on the CPU).
__device__ __forceinline__ uint32_t narrow_start_cell(const NarrowIndexView& nv, float flo) {
    const float tt = (flo - nv.base) * nv.inv_w;
    return tt > 1.0f ? (uint32_t)((int)fminf(tt, (float)(nv.cells - 1)) - 1) : 0u;
}
template <bool EXACT = false>
__device__ __forceinline__ void block_probe_warp(const NarrowIndexView& nv, const QueryDesc& q, uint32_t b0, uint32_t b1, bool act, float flo, float fhi,
                                                 uint32_t* cnt32, uint32_t& matched, uint32_t s0 = 0) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t c = narrow_start_cell(nv, flo);
    for (uint32_t blk = b0; blk <= b1; blk++) {   // warp-uniform: b0, b1 belong to the query
        const uint32_t base = (uint32_t)__ldg(nv.blk_off + blk);   // < 2^31 fragments (db_narrow_index)
        const uint32_t cnt = (uint32_t)__ldg(nv.blk_off + blk + 1) - base;
        const float* mz = nv.mz + base;
        const uint16_t* off = nv.pep + base;
        const uint32_t pep0 = blk * nv.block;
        uint32_t e = cnt;
        if (act) {
            e = __ldg(nv.grp + (size_t)blk * (nv.cells / NARROW_GROUP) + c / NARROW_GROUP) + __ldg(nv.dir + (size_t)blk * nv.cells + c);
            // WALK_STEP entries per step, their loads issued together (one memory latency per step instead of one per entry); past the block
            // end an entry reads as +inf, which ends the run like an m/z above fhi
            for (uint32_t k = 0; k < WALK_SOLO && e < cnt; k += WALK_STEP, e += WALK_STEP) {
                float m[WALK_STEP];
                uint32_t o[WALK_STEP];
#pragma unroll
                for (uint32_t j = 0; j < WALK_STEP; j++) {
                    const bool in = e + j < cnt;
                    m[j] = in ? __ldg(mz + e + j) : __int_as_float(0x7f800000);
                    o[j] = in ? __ldg(off + e + j) : 0u;
                }
                bool stop = false;
#pragma unroll
                for (uint32_t j = 0; j < WALK_STEP; j++) {
                    stop |= m[j] > fhi;
                    const uint32_t pid = pep0 + o[j];
                    if (!stop && m[j] >= flo && pid >= q.eff_lo && pid <= q.eff_hi) {
                        count_match<EXACT>(cnt32, pid - q.pre_lo, s0);
                        matched++;
                    }
                }
                if (stop) { e = cnt; break; }
            }
        }
        uint32_t pend = __ballot_sync(0xffffffffu, e < cnt);   // runs still open
        while (pend) {
            const int src = __ffs(pend) - 1;
            pend &= pend - 1;
            const uint32_t e0 = __shfl_sync(0xffffffffu, e, src);
            const float lo_s = __shfl_sync(0xffffffffu, flo, src), hi_s = __shfl_sync(0xffffffffu, fhi, src);
            for (uint32_t pos = e0; pos < cnt; pos += 32) {
                const uint32_t i = pos + lane;
                bool stop = i >= cnt;
                if (!stop) {
                    const float fmz = __ldg(mz + i);
                    const uint32_t pid = pep0 + __ldg(off + i);
                    stop = fmz > hi_s;
                    if (!stop && fmz >= lo_s) {
                        if (pid >= q.eff_lo && pid <= q.eff_hi) {
                            count_match<EXACT>(cnt32, pid - q.pre_lo, s0);
                            matched++;   // counted on the lane that saw the entry: the warp sums `matched` afterwards
                        }
                    }
                }
                if (__any_sync(0xffffffffu, stop)) break;
            }
        }
    }
}

// ------------------------------------------------------------------------------------- preliminary scoring, narrow
// One CTA per (spectrum, query); the dense per-window counts live in shared memory. Two interchangeable ways to fill them
// (identical counts: the matched set is {fragment in index : mz in [flo,fhi](peak*charge), PeptideIx in [eff_lo,eff_hi]}):
//
//  * index path (mode 1) — the reference's loop order: each thread owns (peak, fragment charge) probes: bucket binary search
//    over min_value, per-page binary search over PeptideIx, exact filter, shared-memory count increment.
//  * peptide-centric path (mode 3) — for small windows: the window's peptides are contiguous in the per-peptide ion table,
//    so one warp per peptide streams its ions (coalesced), and each lane counts the (peak, charge) pairs whose tolerance
//    interval contains its fragment with two binary searches over per-charge LO/HI bound arrays staged in shared memory
//    (bounds computed with the reference's f32 ops; both arrays are monotone in the peak mass, which is verified per
//    spectrum — otherwise the CTA falls back to the index path).
__device__ __forceinline__ void narrow_cta_query(const DbView& db, const ScorerView& sc, const BatchView& b, uint32_t pmax, uint64_t* nlist, uint32_t item,
                                                 float* bounds_smem, const NarrowIndexView& nv) {
    __shared__ uint32_t cnt32[NARROW_CAP / 2 + 1];
    __shared__ uint32_t s_warp[40];
    ReplaySlot* const nslots = b.nslots;
    const uint32_t s = item / sc.qmax;
    const QueryDesc q = b.queries[item];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = PRELIM_THREADS / 32;
    const uint32_t p0 = b.peak_off[s], np = b.peak_off[s + 1] - p0;
    const uint32_t nwords = (q.potential + 1) >> 1;
    for (uint32_t i = tid; i < nwords; i += PRELIM_THREADS) cnt32[i] = 0;
    // key-list space for the trim (only windows larger than k need one): bump-allocated from the chunk's arena, read after the barrier below
    __shared__ unsigned long long s_loff;
    if (tid == 0 && q.potential > sc.kparam) s_loff = atomicAdd(b.counters + C_NLIST, (unsigned long long)q.potential);

    const uint32_t nfc = q.nfc;
    const uint32_t ntask = np * nfc;
    uint32_t my_matched = 0, my_pages = 0, my_entries = 0;
    __shared__ LutParams s_lp[8];
    bool pep_path = q.mode == 3 && np > 0 && np < 65536 && nfc <= 8;
    // dynamic smem layout per fragment charge c: LO_c[pmax] HI_c[pmax] (floats) | sA_c[256] sB_c[256] (u16)
    float* const bnd = bounds_smem;
    uint16_t* const luts = reinterpret_cast<uint16_t*>(bounds_smem + 2 * (size_t)nfc * pmax);
    if (pep_path) {
        for (uint32_t t = tid; t < ntask; t += PRELIM_THREADS) {
            const uint32_t c = t / np, p = t - c * np;
            const float mass = __fmul_rn(__ldg(b.masses + p0 + p), (float)(c + 1));  // scoring.rs:360
            float flo, fhi;
            tol_bounds(sc.fragment_tol, mass, flo, fhi);
            bnd[(2 * c) * pmax + p] = flo;
            bnd[(2 * c + 1) * pmax + p] = fhi;
        }
        __syncthreads();
        bool bad = false;
        for (uint32_t t = tid; t < ntask; t += PRELIM_THREADS) {
            const uint32_t c = t / np, p = t - c * np;
            const float* lo_c = bnd + (2 * c) * pmax;
            const float* hi_c = lo_c + pmax;
            if (p > 0) bad |= !(lo_c[p] >= lo_c[p - 1]) || !(hi_c[p] >= hi_c[p - 1]);
            bad |= !(lo_c[p] == lo_c[p]) || !(hi_c[p] == hi_c[p]);
        }
        if (__syncthreads_or(bad)) {
            pep_path = false;
            if (tid == 0) atomicAdd(b.counters + C_PEPFALLBACK, 1ull);
        } else {
            for (uint32_t c = 0; c < nfc; c++) {
                const float* lo_c = bnd + (2 * c) * pmax;
                const float* hi_c = lo_c + pmax;
                const LutParams L = lut_params(lo_c[0], hi_c[np - 1]);
                if (tid == 0) s_lp[c] = L;
                lut_build(lo_c, np, L, luts + (2 * c) * LUT_CELLS, tid, PRELIM_THREADS);
                lut_build(hi_c, np, L, luts + (2 * c + 1) * LUT_CELLS, tid, PRELIM_THREADS);
            }
            __syncthreads();
        }
    } else {
        __syncthreads();
    }

    if (pep_path) {
        if (q.eff_lo <= q.eff_hi) {
            for (uint32_t pep = q.eff_lo + warp; pep <= q.eff_hi; pep += nwarps) {
                const uint32_t L = __ldg(db.pep_len + pep);
                const uint32_t nions = L - 1, tot = nions * db.n_kinds;
                const float* src = db.ions + __ldg(db.ion_off + pep);
                uint32_t c_here = 0;
                for (uint32_t j0 = 0; j0 < tot; j0 += 32) {
                    const uint32_t j = j0 + lane;
                    if (j < tot) {
                        const uint32_t k = j / nions, i = j - k * nions;
                        const bool keep = ((db.nterm_mask >> k) & 1) ? (i + 1) > db.min_ion_index : (nions - i) > db.min_ion_index;
                        if (keep) {
                            const float f = __ldg(src + j);
                            for (uint32_t c = 0; c < nfc; c++) {
                                const float* lo_c = bnd + (2 * c) * pmax;
                                const float* hi_c = lo_c + pmax;
                                const LutParams LP = s_lp[c];
                                // a = #{p : LO[p] <= f},  bb = #{p : HI[p] < f} (within [0,a)); pairs matched = a - bb
                                uint32_t a = lut_start(LP, luts + (2 * c) * LUT_CELLS, f);
                                while (a < np && lo_c[a] <= f) a++;
                                uint32_t bb = lut_start(LP, luts + (2 * c + 1) * LUT_CELLS, f);
                                while (bb < a && hi_c[bb] < f) bb++;
                                c_here += a - min(bb, a);
                            }
                        }
                    }
                }
                for (int o = 16; o > 0; o >>= 1) c_here += __shfl_down_sync(0xffffffffu, c_here, o);
                if (lane == 0 && c_here) {
                    const uint32_t idx = pep - q.pre_lo;
                    atomicAdd(&cnt32[idx >> 1], (c_here & 0xFFFFu) << ((idx & 1) * 16));
                    my_matched += c_here;
                }
            }
        }
    } else if (nv.mz != nullptr) {
        // small-block copy of the index: every warp takes 32 probes at a time (block_probe_warp finishes long runs warp-wide)
        const uint32_t blk0 = q.pre_lo / nv.block, blk1 = min(q.pre_hi, db.n_pep - 1) / nv.block;
        for (uint32_t t0 = warp * 32; t0 < ntask; t0 += PRELIM_THREADS) {
            const uint32_t t = t0 + lane;
            const bool act = t < ntask;
            float flo = 0.0f, fhi = 0.0f;
            if (act) {
                const uint32_t p = t / nfc, fc = t - p * nfc + 1;
                const float mass = __fmul_rn(__ldg(b.masses + p0 + p), (float)fc);  // scoring.rs:360
                tol_bounds(sc.fragment_tol, mass, flo, fhi);
            }
            block_probe_warp(nv, q, blk0, blk1, act, flo, fhi, cnt32, my_matched);
        }
    } else {
        for (uint32_t t = tid; t < ntask; t += PRELIM_THREADS) {
            const uint32_t p = t / nfc, fc = t - p * nfc + 1;
            const float mass = __fmul_rn(__ldg(b.masses + p0 + p), (float)fc);  // scoring.rs:360
            float flo, fhi;
            tol_bounds(sc.fragment_tol, mass, flo, fhi);
            index_probe(db, q, flo, fhi, cnt32, my_matched, my_pages, my_entries);
        }
    }
    // one block reduction for the three per-CTA sums (matched is needed by every thread, the work counters by thread 0 only)
    __shared__ uint32_t s_red[3][PRELIM_THREADS / 32];
    {
        uint32_t a = my_matched, p = my_pages, en = my_entries;
        for (int o = 16; o > 0; o >>= 1) {
            a += __shfl_down_sync(0xffffffffu, a, o);
            p += __shfl_down_sync(0xffffffffu, p, o);
            en += __shfl_down_sync(0xffffffffu, en, o);
        }
        if (lane == 0) { s_red[0][warp] = a; s_red[1][warp] = p; s_red[2][warp] = en; }
    }
    __syncthreads();
    uint32_t matched_total = 0;
    for (uint32_t w = 0; w < nwarps; w++) matched_total += s_red[0][w];
    if (tid == 0) {
        uint32_t pages_total = 0, entries_total = 0;
        for (uint32_t w = 0; w < nwarps; w++) { pages_total += s_red[1][w]; entries_total += s_red[2][w]; }
        atomicAdd(b.counters + C_TASKS, (unsigned long long)ntask);
        if (pages_total) atomicAdd(b.counters + C_PAGES, (unsigned long long)pages_total);
        if (entries_total) atomicAdd(b.counters + C_ENTRIES, (unsigned long long)entries_total);
        atomicAdd(b.counters + C_MATCHED, (unsigned long long)matched_total);
    }
    QueryHits* h = b.hits + item;
    if (matched_total == 0) {  // scoring.rs:376-378 returns the untrimmed all-default Vec
        if (tid == 0) {
            h->n = 0; h->default_run = q.potential; h->matched_peaks = 0; h->scored_candidates = 0;
            nslots[item].off = 0; nslots[item].item = item; nslots[item].n_list = 0; nslots[item].state = 1; nslots[item].k = 0;
        }
        return;
    }
    // trim_hits (scoring.rs:322-329), stage 1: emit the keys in dense order — the literal first k slots, then every later slot with
    // matched > 0 (zeros can never displace the heap root). k_replay performs the exact heap replay, one thread per query.
    const uint32_t n = q.potential, k = min(n, sc.kparam);
    auto cnt = [&](uint32_t i) -> uint32_t { return (cnt32[i >> 1] >> ((i & 1) * 16)) & 0xFFFFu; };
    ReplaySlot* slot = nslots + item;
    uint32_t nzc = 0;
    if (n <= k) {   // nothing to trim: the dense order is the result
        uint64_t* keys = b.hit_keys + (size_t)item * sc.kparam;
        for (uint32_t i = tid; i < n; i += PRELIM_THREADS) {
            const uint32_t c = cnt(i);
            nzc += c != 0;
            keys[i] = c ? prescore_key(c, q.pre_lo + i, q.charge, q.iso) : PRESCORE_DEFAULT;
        }
        const uint32_t nzt = block_sum_u32(nzc, s_warp);
        if (tid == 0) {
            h->n = n; h->default_run = 0; h->matched_peaks = matched_total; h->scored_candidates = nzt;
            slot->off = 0; slot->item = item; slot->n_list = 0; slot->state = 1; slot->k = k;
            if (matched_total >= EXACT_TRIGGER) b.exact_items[atomicAdd(b.counters + C_EXACT, 1ull)] = item;
        }
        return;
    }
    const unsigned long long loff = s_loff;
    if (loff + n > b.nlist_cap) {   // arena too small (the host sees C_NLIST_NEED > capacity and re-runs the chunk): leave "no hits"
        if (tid == 0) {
            h->n = 0; h->default_run = q.potential; h->matched_peaks = 0; h->scored_candidates = 0;
            slot->off = 0; slot->item = item; slot->n_list = 0; slot->state = 1; slot->k = 0;
        }
        return;
    }
    uint64_t* list = nlist + loff;
    for (uint32_t i = tid; i < k; i += PRELIM_THREADS) {
        const uint32_t c = cnt(i);
        nzc += c != 0;
        list[i] = c ? prescore_key(c, q.pre_lo + i, q.charge, q.iso) : PRESCORE_DEFAULT;
    }
    uint32_t wbase = k;   // next free list position (uniform across the CTA)
    for (uint32_t base = k; base < n; base += PRELIM_THREADS) {
        const uint32_t i = base + tid;
        const uint32_t c = i < n ? cnt(i) : 0;
        nzc += c != 0;
        const uint32_t ball = __ballot_sync(0xffffffffu, c != 0);
        if (lane == 0) s_warp[warp] = __popc(ball);
        __syncthreads();
        uint32_t off = 0, total = 0;
        for (uint32_t w = 0; w < nwarps; w++) {
            const uint32_t x = s_warp[w];
            if (w < warp) off += x;
            total += x;
        }
        if (c) list[wbase + off + __popc(ball & ((1u << lane) - 1))] = prescore_key(c, q.pre_lo + i, q.charge, q.iso);
        wbase += total;
        __syncthreads();
    }
    const uint32_t nzt = block_sum_u32(nzc, s_warp);
    if (tid == 0) {
        h->n = k; h->default_run = 0; h->matched_peaks = matched_total; h->scored_candidates = nzt;
        slot->off = loff; slot->item = item; slot->n_list = wbase; slot->state = 0; slot->k = k;
        if (matched_total >= EXACT_TRIGGER) b.exact_items[atomicAdd(b.counters + C_EXACT, 1ull)] = item;
    }
}

// Queries counted by a whole CTA (windows of WARPQ_CAP+1..NARROW_CAP peptides, and the peptide-centric path): a fixed-size grid walks the
// compacted list k_setup_queries wrote.
// The register budget holds the PRELIM_CTAS CTAs per SM the grid is sized for (without it ptxas picked a budget that spilled).
__global__ void __launch_bounds__(PRELIM_THREADS, PRELIM_CTAS) k_prelim_narrow(DbView db, ScorerView sc, BatchView b, uint32_t pmax, uint64_t* nlist, NarrowIndexView nv) {
    extern __shared__ float bounds_smem[];  // LO[nfc][np] then HI[nfc][np] (peptide-centric path only)
    const uint32_t total = (uint32_t)min(b.counters[C_NCTA], (unsigned long long)b.n * sc.qmax);
    for (uint32_t i = blockIdx.x; i < total; i += gridDim.x) {
        narrow_cta_query(db, sc, b, pmax, nlist, b.cta_items[i], bounds_smem, nv);
        __syncthreads();   // shared arrays are reused by the next query
    }
}

// One WARP per (spectrum, query) for windows of at most WARPQ_CAP peptides — the common case of a narrow search. The index path of
// narrow_cta_query without any block-wide barrier: each lane owns (peak, fragment charge) probes t = lane, lane + 32, ..., the dense u16
// counts of the window live in the warp's slice of shared memory, sums are warp shuffles, and the ordered key list for k_replay
// is emitted with ballots. grid = (ceil(n / WARPQ_WARPS) in precursor order, query slot): slot-major, so CTAs of slots no spectrum uses
// (e.g. the charge fold of known-charge spectra) sit at the end of the grid and leave after one cached load.
template <bool BLK>
__global__ void __launch_bounds__(WARPQ_WARPS * 32, WARPQ_MIN_CTAS) k_prelim_narrow_warp(DbView db, ScorerView sc, BatchView b, uint64_t* nlist, uint32_t s_lo,
                                                                                                uint32_t s_hi, NarrowIndexView nv) {
    __shared__ uint32_t cnt_all[WARPQ_WARPS][WARPQ_CAP / 2];
    if (b.counters[C_COUNT + blockIdx.y] == 0ull) return;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t pos = blockIdx.x * WARPQ_WARPS + warp;
    if (pos >= b.n) return;
    const uint32_t s = b.order ? b.order[pos] : pos;
    // [s_lo, s_hi): the spectra (caller order) whose peak masses are on the device when this launch runs — the host queues one launch per part
    // of the masses copy, each still walking its spectra in precursor order
    if (s < s_lo || s >= s_hi) return;
    const uint32_t item = s * sc.qmax + blockIdx.y;
    const QueryDesc q = b.queries[item];
    if (q.mode != 4) return;
    uint32_t* const cnt32 = cnt_all[warp];
    const uint32_t n = q.potential, k = min(n, sc.kparam);
    for (uint32_t i = lane; i < (n + 1) >> 1; i += 32) cnt32[i] = 0;
    unsigned long long loff = 0;
    if (n > k) {   // key-list space for the trim, bump-allocated from the chunk's arena
        if (lane == 0) loff = atomicAdd(b.counters + C_NLIST, (unsigned long long)n);
        loff = __shfl_sync(0xffffffffu, loff, 0);
    }
    __syncwarp();
    const uint32_t p0 = b.peak_off[s], np = b.peak_off[s + 1] - p0;
    const uint32_t nfc = q.nfc, ntask = np * nfc;
    uint32_t matched = 0, pages = 0, entries = 0;
    const uint32_t blk0 = BLK ? q.pre_lo / nv.block : 0u, blk1 = BLK ? min(q.pre_hi, db.n_pep - 1) / nv.block : 0u;
    for (uint32_t t0 = 0; t0 < ntask; t0 += 32) {   // warp-uniform trip count: the block path finishes long runs cooperatively
        const uint32_t t = t0 + lane;
        const bool act = t < ntask;
        float flo = 0.0f, fhi = 0.0f;
        if (act) {
            const uint32_t p = t / nfc, fc = t - p * nfc + 1;
            const float mass = __fmul_rn(__ldg(b.masses + p0 + p), (float)fc);  // scoring.rs:360
            tol_bounds(sc.fragment_tol, mass, flo, fhi);
        }
        if (BLK) block_probe_warp(nv, q, blk0, blk1, act, flo, fhi, cnt32, matched);
        else if (act) index_probe(db, q, flo, fhi, cnt32, matched, pages, entries);
    }
    for (int o = 16; o > 0; o >>= 1) {
        matched += __shfl_xor_sync(0xffffffffu, matched, o);
        pages += __shfl_xor_sync(0xffffffffu, pages, o);
        entries += __shfl_xor_sync(0xffffffffu, entries, o);
    }
    __syncwarp();   // all shared-memory increments of the warp are visible below
    if (lane == 0) {
        atomicAdd(b.counters + C_TASKS, (unsigned long long)ntask);
        if (pages) atomicAdd(b.counters + C_PAGES, (unsigned long long)pages);
        if (entries) atomicAdd(b.counters + C_ENTRIES, (unsigned long long)entries);
        if (matched) atomicAdd(b.counters + C_MATCHED, (unsigned long long)matched);
    }
    QueryHits* h = b.hits + item;
    ReplaySlot* slot = b.nslots + item;   // preset by k_setup_queries to "nothing to replay"
    if (matched == 0 || (n > k && loff + n > b.nlist_cap)) {
        // scoring.rs:376-378 returns the untrimmed all-default Vec; or the arena is too small (the host sees C_NLIST_NEED > capacity
        // and re-runs the chunk): leave "no hits"
        if (lane == 0) { h->n = 0; h->default_run = n; h->matched_peaks = 0; h->scored_candidates = 0; }
        return;
    }
    // trim_hits (scoring.rs:322-329), stage 1: the keys in dense order — the literal first k slots, then every later slot with
    // matched > 0 (zeros can never displace the heap root). k_replay performs the exact heap replay, one thread per query.
    auto cnt = [&](uint32_t i) -> uint32_t { return (cnt32[i >> 1] >> ((i & 1) * 16)) & 0xFFFFu; };
    uint32_t nzc = 0;
    uint64_t* dst = n <= k ? b.hit_keys + (size_t)item * sc.kparam : nlist + loff;   // n <= k: nothing to trim, the dense order is the result
    for (uint32_t i = lane; i < k; i += 32) {
        const uint32_t c = cnt(i);
        nzc += c != 0;
        dst[i] = c ? prescore_key(c, q.pre_lo + i, q.charge, q.iso) : PRESCORE_DEFAULT;
    }
    uint32_t wbase = k;
    for (uint32_t base = k; base < n; base += 32) {
        const uint32_t i = base + lane;
        const uint32_t c = i < n ? cnt(i) : 0;
        nzc += c != 0;
        const uint32_t ball = __ballot_sync(0xffffffffu, c != 0);
        if (c) dst[wbase + __popc(ball & ((1u << lane) - 1))] = prescore_key(c, q.pre_lo + i, q.charge, q.iso);
        wbase += __popc(ball);
    }
    for (int o = 16; o > 0; o >>= 1) nzc += __shfl_xor_sync(0xffffffffu, nzc, o);
    if (lane == 0) {
        h->n = k; h->default_run = 0; h->matched_peaks = matched; h->scored_candidates = nzc;
        if (n > k) { slot->off = loff; slot->n_list = wbase; slot->state = 0; slot->k = k; }
        if (matched >= EXACT_TRIGGER) b.exact_items[atomicAdd(b.counters + C_EXACT, 1ull)] = item;
    }
}

// The narrow queries with >= 2^16 matches (EXACT_TRIGGER), one CTA each: the window again in segments of EXACT_SEG slots with one u32 count
// per slot, then the keys the counting kernel wrote are rewritten with the reference's wrapped u16 counts, in the same dense order (the
// literal first k slots, then every later slot the query touched), and scored_candidates becomes the sum of ceil(count / 2^16). A slot whose
// count wrapped to exactly 0 keeps its PeptideIx: the reference set it when the count was 0, so it is scored, not PreScore::default().
__global__ void __launch_bounds__(PRELIM_THREADS) k_prelim_exact(DbView db, ScorerView sc, BatchView b, uint64_t* nlist, NarrowIndexView nv) {
    __shared__ uint32_t cnt32[EXACT_SEG];
    __shared__ uint32_t s_warp[PRELIM_THREADS / 32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = PRELIM_THREADS / 32;
    const uint32_t total = (uint32_t)min(b.counters[C_EXACT], (unsigned long long)b.n * sc.qmax);
    for (uint32_t it = blockIdx.x; it < total; it += gridDim.x) {
        const uint32_t item = b.exact_items[it];
        const uint32_t s = item / sc.qmax;
        const QueryDesc q = b.queries[item];
        const uint32_t p0 = b.peak_off[s], np = b.peak_off[s + 1] - p0;
        const uint32_t nfc = q.nfc, ntask = np * nfc;
        const uint32_t n = q.potential, k = min(n, sc.kparam);
        ReplaySlot* const slot = b.nslots + item;
        uint64_t* const dst = n <= k ? b.hit_keys + (size_t)item * sc.kparam : nlist + slot->off;
        uint32_t nzc = 0, wbase = k;
        for (uint32_t s0 = 0; s0 < n; s0 += EXACT_SEG) {
            for (uint32_t i = tid; i < EXACT_SEG; i += PRELIM_THREADS) cnt32[i] = 0;
            __syncthreads();
            uint32_t dm = 0, dp = 0, de = 0;
            if (nv.mz != nullptr) {
                const uint32_t blk0 = q.pre_lo / nv.block, blk1 = min(q.pre_hi, db.n_pep - 1) / nv.block;
                for (uint32_t t0 = warp * 32; t0 < ntask; t0 += PRELIM_THREADS) {
                    const uint32_t t = t0 + lane;
                    const bool act = t < ntask;
                    float flo = 0.0f, fhi = 0.0f;
                    if (act) {
                        const uint32_t p = t / nfc, fc = t - p * nfc + 1;
                        tol_bounds(sc.fragment_tol, __fmul_rn(__ldg(b.masses + p0 + p), (float)fc), flo, fhi);   // scoring.rs:360
                    }
                    block_probe_warp<true>(nv, q, blk0, blk1, act, flo, fhi, cnt32, dm, s0);
                }
            } else {
                for (uint32_t t = tid; t < ntask; t += PRELIM_THREADS) {
                    const uint32_t p = t / nfc, fc = t - p * nfc + 1;
                    float flo, fhi;
                    tol_bounds(sc.fragment_tol, __fmul_rn(__ldg(b.masses + p0 + p), (float)fc), flo, fhi);   // scoring.rs:360
                    index_probe<true>(db, q, flo, fhi, cnt32, dm, dp, de, s0);
                }
            }
            __syncthreads();
            const uint32_t s1 = min(n, s0 + EXACT_SEG);
            for (uint32_t base = s0; base < s1; base += PRELIM_THREADS) {   // uniform trip count: every thread reaches the barriers
                const uint32_t i = base + tid;
                const uint32_t c = i < s1 ? cnt32[i - s0] : 0u;
                nzc += (c >> 16) + ((c & 0xFFFFu) != 0u);   // ceil(c / 2^16)
                const uint64_t key = c ? prescore_key(c & 0xFFFFu, q.pre_lo + i, q.charge, q.iso) : PRESCORE_DEFAULT;
                if (i < k) dst[i] = key;   // k <= EXACT_SEG: the literal slots lie in the first segment
                const bool emit = i >= k && c != 0;
                const uint32_t ball = __ballot_sync(0xffffffffu, emit);
                if (lane == 0) s_warp[warp] = __popc(ball);
                __syncthreads();
                uint32_t off = 0, tot = 0;
                for (uint32_t w = 0; w < nwarps; w++) {
                    const uint32_t x = s_warp[w];
                    if (w < warp) off += x;
                    tot += x;
                }
                if (emit) dst[wbase + off + __popc(ball & ((1u << lane) - 1))] = key;
                wbase += tot;
                __syncthreads();
            }
        }
        const uint32_t nzt = block_sum_u32(nzc, s_warp);
        if (tid == 0) {
            b.hits[item].scored_candidates = nzt;
            if (n > k) slot->n_list = wbase;
        }
        __syncthreads();
    }
}

// --------------------------------------------------------------------------------------- preliminary scoring, wide
// Open-search windows (> NARROW_CAP peptides; ±500 Da spans ~40 % of a human index) make the dense count array megabytes long.
// Instead of a global scratch + L2/DRAM atomics, the window is processed in TILES of WIDE_TILE consecutive PeptideIx whose u16
// counts live in shared memory (1 CTA / SM, ~200 KB). Inside a page entries are sorted by PeptideIx, so the part of a page slice
// that belongs to a tile is a contiguous sub-slice: every page visit (peak, fragment charge, page) carries its position from
// tile to tile (one binary search per visit and tile), whole warps stream the sub-slices with coalesced 8-byte loads (4 in
// flight per lane), matches become shared-memory atomics, and after each tile the exact trim (heap replay in index order)
// consumes the tile's counts straight from shared memory. Every index entry of [inner_left, inner_right) is read exactly once.
// Shape of the open-search CTA: threads, peptides per count tile, CTAs per SM the shared-memory budget allows. Chosen by A/B on cfg4
// (block-index path) over 256..1024 threads, 16k..80k-peptide tiles, 1..3 CTAs per SM and walk unrolls 2..8.
// Two resident CTAs matter more than the tile size: the kernel is a chain of short phases separated by CTA-wide barriers (12 barrier-stalled
// warps per issued instruction with one CTA per SM), and a second CTA fills the gaps.
#ifndef SAGE_B200_WIDE_THREADS
#define SAGE_B200_WIDE_THREADS 512
#endif
#ifndef SAGE_B200_WIDE_TILE
#define SAGE_B200_WIDE_TILE (32 * 1024)
#endif
#ifndef SAGE_B200_WIDE_CTAS
#define SAGE_B200_WIDE_CTAS 2
#endif
constexpr int WIDE_THREADS = SAGE_B200_WIDE_THREADS;
constexpr int WIDE_CTAS = SAGE_B200_WIDE_CTAS;
constexpr bool WIDE_SMALL = WIDE_CTAS > 1;        // several CTAs per SM: every per-query table shrinks with the tile
constexpr uint32_t WIDE_TILE = SAGE_B200_WIDE_TILE;    // peptides per tile (u16 counts: 64 KB at 32 k)
constexpr uint32_t WIDE_VMAX = WIDE_SMALL ? 1024 : 2048;    // page visits whose running position is cached in smem
constexpr uint32_t WIDE_TCACHE = WIDE_SMALL ? 1024 : 2048;  // (peak, charge) probes whose bucket range is cached in smem
constexpr uint32_t WIDE_LMAX = 12288;        // survivor keys kept per query for the replay kernel (overflow -> in-kernel serial replay)
constexpr uint32_t WIDE_HLEV = 64;           // matched-count histogram levels (last level = ">= 63")
typedef ReplaySlot WideSlot;
struct WideRange { uint64_t start; uint32_t len; float flo, fhi; };

constexpr uint32_t WIDE_VCAP = WIDE_SMALL ? 512 : 1024;   // page visits per query handled by the boundary-table fast path
constexpr uint32_t WIDE_BT = 16;             // boundary columns (tiles + 1) of the fast path
struct WideSlow {                            // fallback: one search per (visit, tile), positions carried in `cur`
    uint32_t cur[WIDE_VMAX];
    uint32_t task_bl[WIDE_TCACHE];
    uint16_t task_nb[WIDE_TCACHE];
    WideRange ranges[WIDE_THREADS];
};
struct WideFast {                            // fast path: all tile boundaries of all page visits resolved once per query
    uint16_t B[WIDE_VCAP * WIDE_BT];         // B[v*nb1 + t] = lower_bound(page(v), first PeptideIx of tile t); column ntiles = inner_right
    uint32_t vpage[WIDE_VCAP];
    float vflo[WIDE_VCAP], vfhi[WIDE_VCAP];
};
constexpr uint32_t WIDE_TMAX = WIDE_SMALL ? 1024 : 2048;    // (peak, charge) probes per query handled by the block-index path
#ifndef SAGE_B200_WIDE_UNROLL
#define SAGE_B200_WIDE_UNROLL 2
#endif
constexpr int WIDE_WALK_UNROLL = SAGE_B200_WIDE_UNROLL;          // probes a warp walks concurrently (independent loads in flight)
constexpr uint32_t WIDE_SMAX = WIDE_SMALL ? 3072 : 6144;    // (block, probe) run starts resolved per block group (one batch of independent searches)
constexpr uint32_t WIDE_QCAP = WIDE_THREADS;  // slots a tile may queue as survivors (one per thread in the ordering step); more -> the tile is scanned instead
struct WideBlk {
    float flo[WIDE_TMAX], fhi[WIDE_TMAX];    // Tolerance::bounds of every probe of the query
    uint32_t qslot[WIDE_QCAP];               // tile-relative slots whose count reached the survivor level during the walk (unordered)
    uint32_t start[WIDE_SMAX];               // [tile of the current tile group][probe]: first entry of the block with m/z >= flo
};
struct WideSmem {
    uint32_t cnt32[WIDE_TILE / 2 + 4];   // + slack: a block-mode tile can hold TILE + 1 slots (the phantom slot pre_idx_hi == n_pep)
    union { WideSlow slow; WideFast fast; WideBlk blk; } u;
    uint64_t heap[K_MAX];
    uint64_t queue[2 * WIDE_THREADS];
    uint32_t s_warp[40];
    uint32_t hist[WIDE_HLEV];   // entries seen in earlier tiles with matched == level (level 63 = >= 63)
    uint32_t s_item, s_slot, s_level, s_listn, s_serial, s_nranges, s_nvis, s_fast, s_lit /* literal first-k slots already listed */;
    uint32_t s_qn /* survivor candidates queued in this tile */, s_tnext /* next probe group of this tile (dynamic distribution over the warps) */;
};


__global__ void __launch_bounds__(WIDE_THREADS, WIDE_CTAS) k_prelim_wide(DbView db, ScorerView sc, BatchView b, uint32_t n_items, uint64_t* wlist,
                                                                   WideSlot* wslots, WideIndexView wv) {
    extern __shared__ __align__(16) unsigned char wide_raw[];
    WideSmem& S = *reinterpret_cast<WideSmem*>(wide_raw);
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = WIDE_THREADS / 32;
    for (;;) {
        __syncthreads();
        if (tid == 0) {
            // next entry of the compacted open-search work list (k_setup_queries); slot == position in that list
            const unsigned long long nw = min(b.counters[C_WIDE], (unsigned long long)b.wide_cap);
            const unsigned long long w = atomicAdd(b.counters + C_WORK, 1ull);
            S.s_item = w < nw ? b.wide_items[w] : n_items;
            if (w < nw) {
                S.s_slot = (uint32_t)w;
                S.s_level = 1; S.s_listn = 0; S.s_serial = 0; S.s_lit = 0;
            }
        }
        if (tid < WIDE_HLEV) S.hist[tid] = 0;
        __syncthreads();
        const uint32_t item = S.s_item;
        if (item >= n_items) return;
        uint64_t* const list = wlist + (size_t)S.s_slot * WIDE_LMAX;
        const unsigned long long list_off = (unsigned long long)S.s_slot * WIDE_LMAX;
        const QueryDesc q = b.queries[item];
        const uint32_t s = item / sc.qmax;
        const uint32_t p0 = b.peak_off[s], np = b.peak_off[s + 1] - p0;
        const uint32_t nfc = q.nfc, ntask = np * nfc;
        const uint32_t n = q.potential;                       // dense slots of this window
        const uint32_t k = min(n, sc.kparam);                 // n > NARROW_CAP > k here
        const uint32_t TILE = sc.wide_tile;                   // <= WIDE_TILE (smaller only in tests, to exercise the multi-tile logic)
        // Block mode (secondary index present): tile t == peptide block b0 + t of the block-major, m/z-sorted index copy; a probe's matches inside
        // a tile are one contiguous run of that block. Otherwise (index not built / too many probes): page-slice streaming with two short leading
        // tiles that tighten the matched-count bound early (keeps the survivor lists short), then full tiles.
        const bool blockmode = wv.frag != nullptr && wv.block == TILE && ntask <= WIDE_TMAX;
        const uint32_t blk0 = blockmode ? q.pre_lo / TILE : 0;
        const uint32_t T0 = max(TILE / 8, 256u) & ~7u, T1 = max(TILE / 4, 256u) & ~7u;
        // Block mode: the part of the window inside its FIRST block is cut into up to three tiles (T0, T1, rest) like the leading tiles of the
        // page-slice path — without them the first tile runs at survivor level 1 over up to TILE slots and one query in eight overflowed its
        // survivor list (measured); a sub-block tile re-reads the probes' (short) runs of that block and keeps the PeptideIx of its own range.
        // (pre_idx_hi may be n_pep, one past the last peptide: that phantom slot never matches and belongs to the last real block's tile.)
        const uint32_t nblk = blockmode ? min(q.pre_hi, db.n_pep - 1) / TILE - blk0 + 1 : 0;
        const uint32_t n0 = blockmode ? (nblk == 1 ? n : (blk0 + 1) * TILE - q.pre_lo) : 0;    // dense slots inside the first block
        const uint32_t nfirst = n0 <= T0 ? 1 : (n0 <= T0 + T1 ? 2 : 3);
        const uint32_t ntiles = blockmode ? nfirst + nblk - 1 : (n <= T0 ? 1 : (n <= T0 + T1 ? 2 : 2 + (n - T0 - T1 + TILE - 1) / TILE));
        uint32_t my_matched = 0, my_pages = 0, nz = 0;
        uint32_t msum = 0;   // sum of all slot counts == matched_peaks of this query (replaces per-match counting in the streaming loop)
        long long my_entries = 0;
        auto tile_d0 = [&](uint32_t t) -> uint32_t { return t == 0 ? 0 : (t == 1 ? T0 : T0 + T1 + (t - 2) * TILE); };

        // ---- fast path setup: enumerate the page visits of every (peak, charge) probe and resolve all tile boundaries at once
        const uint32_t nb1 = ntiles + 1;
        if (tid == 0) { S.s_nvis = 0; S.s_fast = (!blockmode && nb1 <= WIDE_BT && db.bucket_size <= 65535u) ? 1u : 0u; }
        if (blockmode) {   // Tolerance::bounds of every (peak, fragment charge) probe, once per query
            for (uint32_t t = tid; t < ntask; t += WIDE_THREADS) {
                const uint32_t p = t / nfc, fc = t - p * nfc + 1;
                const float mass = __fmul_rn(__ldg(b.masses + p0 + p), (float)fc);  // scoring.rs:360
                tol_bounds(sc.fragment_tol, mass, S.u.blk.flo[t], S.u.blk.fhi[t]);
            }
        }
        __syncthreads();
        if (S.s_fast) {
            WideFast& F = S.u.fast;
            for (uint32_t t = tid; t < ntask; t += WIDE_THREADS) {
                const uint32_t p = t / nfc, fc = t - p * nfc + 1;
                const float mass = __fmul_rn(__ldg(b.masses + p0 + p), (float)fc);  // scoring.rs:360
                float flo, fhi;
                tol_bounds(sc.fragment_tol, mass, flo, fhi);
                uint32_t bl, br;
                bucket_range(db, flo, fhi, bl, br);
                const uint32_t nbk = br - bl;
                if (nbk) {
                    const uint32_t v0 = atomicAdd(&S.s_nvis, nbk);   // visit order is irrelevant for counting
                    if (v0 + nbk <= WIDE_VCAP) {
                        for (uint32_t r = 0; r < nbk; r++) { F.vpage[v0 + r] = bl + r; F.vflo[v0 + r] = flo; F.vfhi[v0 + r] = fhi; }
                    } else S.s_fast = 0;
                }
            }
            __syncthreads();
        }
        if (S.s_fast) {
            WideFast& F = S.u.fast;
            const uint32_t nvis = S.s_nvis;
            for (uint32_t j = tid; j < nvis * nb1; j += WIDE_THREADS) {
                const uint32_t v = j / nb1, t = j - v * nb1;
                const uint64_t pbase = (uint64_t)F.vpage[v] * db.bucket_size;
                const uint32_t pn = (uint32_t)(min(pbase + db.bucket_size, db.n_frag) - pbase);
                const uint32_t key = t == ntiles ? q.pre_hi + 1 : q.pre_lo + tile_d0(t);
                F.B[j] = (uint16_t)page_lower_bound_dir(db, F.vpage[v], db.frag + pbase, pn, key);
            }
            __syncthreads();
            for (uint32_t v = tid; v < nvis; v += WIDE_THREADS) {   // SURVEY §8d counters: inner_right - inner_left per page visit
                const uint32_t st = F.B[v * nb1], en = F.B[v * nb1 + ntiles];
                my_entries += (long long)en - (long long)(st == 0 ? 0 : st - 1);
                my_pages++;
            }
        }
        const bool fast = S.s_fast != 0;

        uint32_t grp0 = 0, grp_n = 0;   // current block group of the block-index path: blocks [grp0, grp0 + grp_n)
        for (uint32_t tile = 0; tile < ntiles; tile++) {
            const uint32_t tblk = blockmode ? (tile < nfirst ? blk0 : blk0 + tile - nfirst + 1) : 0;   // block this tile lies in
            if (blockmode && tblk >= grp0 + grp_n) {
                // ---- run starts of every (block, probe) pair of the next block group, all searches independent: LUT bracket (the cell of flo, one
                // early / two late to absorb the float rounding of the cell index), then the exact lower bound on the entries' m/z
                grp0 = tblk;
                grp_n = min(blk0 + nblk - tblk, max(1u, WIDE_SMAX / max(ntask, 1u)));
                __syncthreads();   // the previous group's starts are no longer read
                for (uint32_t w = tid; w < grp_n * ntask; w += WIDE_THREADS) {
                    const uint32_t g = w / ntask, j = w - g * ntask, blk = grp0 + g;
                    const uint2* const ent = wv.frag + wv.blk_off[blk];
                    const uint32_t blen = (uint32_t)(wv.blk_off[blk + 1] - wv.blk_off[blk]);
                    const uint32_t* const lutb = wv.lut + (size_t)blk * (wv.cells + 1);
                    const float flo = S.u.blk.flo[j];
                    uint32_t lo = blen, hi = blen;   // NaN bounds: empty run
                    if (flo == flo && S.u.blk.fhi[j] == S.u.blk.fhi[j]) {
                        lo = 0;
                        if (wv.inv_w > 0.0f) {
                            const float tt = (flo - wv.base) * wv.inv_w;
                            const int c = tt > 1.0f ? (int)fminf(tt, (float)(wv.cells - 1)) - 1 : 0;
                            lo = __ldg(lutb + c);
                            hi = __ldg(lutb + min((uint32_t)c + 3u, wv.cells));
                        }   // else no LUT (an index with m/z <= 0 or a degenerate range): the bisection runs over the whole block
                        while (lo < hi) {
                            const uint32_t mid = lo + ((hi - lo) >> 1);
                            if (__uint_as_float(__ldg(&ent[mid].y)) < flo) lo = mid + 1; else hi = mid;
                        }
                    }
                    S.u.blk.start[w] = lo;
                }
                __syncthreads();
            }
            // first dense slot of the tile / slots in the tile
            const uint32_t d0 = blockmode ? (tile < nfirst ? (tile == 0 ? 0 : (tile == 1 ? T0 : T0 + T1)) : tblk * TILE - q.pre_lo)
                                          : (tile == 0 ? 0 : (tile == 1 ? T0 : T0 + T1 + (tile - 2) * TILE));
            const uint32_t dn = blockmode ? (tile < nfirst ? (tile == 0 ? min(T0, n0) : (tile == 1 ? min(T1, n0 - T0) : n0 - T0 - T1))
                                                           : (tile + 1 == ntiles ? q.pre_hi + 1 - (q.pre_lo + d0) : TILE))   // <= TILE + 1 (phantom slot)
                                          : min(tile == 0 ? T0 : (tile == 1 ? T1 : TILE), n - d0);
            const uint32_t pep_lo = q.pre_lo + d0;                         // PeptideIx of slot d0
            const bool last_tile = tile + 1 == ntiles;
            const bool tile_entered_serial = S.s_serial != 0;  // uniform: s_serial only changes between barriers at the end of a tile
            // exclusive PeptideIx bound of the tile; the last tile ends at pre_hi + 1 so that its end == inner_right (database.rs:506-511)
            const uint32_t pep_hi_excl = last_tile ? q.pre_hi + 1 : pep_lo + dn;
            {   // zero the tile's counts, 16 bytes per store
                uint4* const z = reinterpret_cast<uint4*>(S.cnt32);
                for (uint32_t i = tid; i < ((dn + 1) / 2 + 3) / 4; i += WIDE_THREADS) z[i] = make_uint4(0, 0, 0, 0);
            }
            if (tid == 0) { S.s_qn = 0; S.s_tnext = 0; }
            // Block mode counts matched_peaks / scored_candidates while it walks (the atomic returns the slot's previous count), and — once the
            // survivor level is >= 2, i.e. from the second tile on — queues the few slots whose count reaches the level instead of scanning all
            // `dn` counts of the tile afterwards.
            const uint32_t tile_level = S.s_level;
            const bool use_q = blockmode && tile_level >= 2 && !tile_entered_serial;
            __syncthreads();
            if (blockmode) {
                // every probe's matches inside this tile are ONE run of the block's m/z-sorted entries, located through the per-block m/z LUT;
                // exact filter on the values (database.rs:526-533: PeptideIx inside the edge-filtered window, m/z inside [flo, fhi])
                const uint32_t blk = tblk;
                const uint2* const ent = wv.frag + wv.blk_off[blk];
                const uint32_t blen = (uint32_t)(wv.blk_off[blk + 1] - wv.blk_off[blk]);
                const uint32_t t_lo = max(q.eff_lo, pep_lo);
                const uint32_t t_hi = min(q.eff_hi, pep_hi_excl - 1);
                const bool t_any = q.eff_lo <= q.eff_hi && t_lo <= t_hi;
                const uint32_t t_span = t_any ? t_hi - t_lo : 0u;
                // The run starts of all probes were resolved for this tile group in one batch of independent searches (below the tile loop
                // header); a warp walks WIDE_WALK_UNROLL runs at a time, 32 coalesced entries per run and step. Groups of probes are handed
                // out dynamically (run lengths vary). Measured and slower: starting the walk at the LUT cell instead of the
                // exact lower bound (most fetched entries lie before the run), one thread per probe (~280 threads
                // in flight per SM cannot hide the dependent-load latency).
                const uint32_t* const starts = S.u.blk.start + (tblk - grp0) * ntask;
                for (;;) {
                    uint32_t j0 = 0;
                    if (lane == 0) j0 = atomicAdd(&S.s_tnext, (uint32_t)WIDE_WALK_UNROLL);
                    j0 = __shfl_sync(0xffffffffu, j0, 0);
                    if (!t_any || j0 >= ntask) break;
                    float fhi[WIDE_WALK_UNROLL];
                    uint32_t pos[WIDE_WALK_UNROLL];
                    bool live[WIDE_WALK_UNROLL];
#pragma unroll
                    for (int u = 0; u < WIDE_WALK_UNROLL; u++) {
                        const uint32_t j = j0 + u;
                        live[u] = j < ntask;
                        fhi[u] = live[u] ? S.u.blk.fhi[j] : 0.0f;
                        pos[u] = live[u] ? starts[j] : blen;
                    }
                    for (;;) {
                        uint2 f[WIDE_WALK_UNROLL];
#pragma unroll
                        for (int u = 0; u < WIDE_WALK_UNROLL; u++) {
                            const uint32_t e = pos[u] + lane;
                            f[u] = (live[u] && e < blen) ? __ldg(ent + e) : make_uint2(0xFFFFFFFFu, 0x7F800000u);   // past the block: +inf ends the run
                        }
                        bool any_live = false;
#pragma unroll
                        for (int u = 0; u < WIDE_WALK_UNROLL; u++) {
                            const float m = __uint_as_float(f[u].y);
                            const bool in = m <= fhi[u];   // (m >= flo holds from the run start on; NaN bounds match nothing: starts == block end)
                            if (in && f[u].x - t_lo <= t_span) {
                                const uint32_t idx = f[u].x - pep_lo, sh = (idx & 1) * 16;
                                const uint32_t prev = (atomicAdd(&S.cnt32[idx >> 1], 1u << sh) >> sh) & 0xFFFFu;   // this slot's count before this match
                                msum++;
                                nz += prev == 0;
                                if (use_q && prev + 1 == tile_level) {   // exactly one match sees the slot cross the level
                                    const uint32_t qi = atomicAdd(&S.s_qn, 1u);
                                    if (qi < WIDE_QCAP) S.u.blk.qslot[qi] = idx;
                                }
                            }
                            // entries ascend in m/z: the run continues only while the last entry fetched is still <= fhi
                            live[u] = live[u] && __shfl_sync(0xffffffffu, in, 31);
                            pos[u] += 32;
                            any_live |= live[u];
                        }
                        if (!any_live) break;
                    }
                }
            } else if (fast) {
                // stream every visit's sub-slice of this tile: one warp walks two visits at a time, 4 coalesced 8-byte entries per lane
                // from each (8 loads = 2 KB in flight per warp, 32 KB per CTA)
                const WideFast& F = S.u.fast;
                const uint32_t nvis = S.s_nvis;
                // tile-specific accepted PeptideIx range as one unsigned compare: (pep - t_lo) <= t_span
                const uint32_t t_lo = max(q.eff_lo, pep_lo);
                const uint32_t t_hi = min(q.eff_hi, pep_hi_excl - 1);
                const bool t_any = q.eff_lo <= q.eff_hi && t_lo <= t_hi;
                const uint32_t t_span = t_any ? t_hi - t_lo : 0u;
                for (uint32_t v0 = warp * 2; t_any && v0 < nvis; v0 += nwarps * 2) {
                    const uint32_t v1 = min(v0 + 1, nvis - 1);
                    const uint32_t stA = F.B[v0 * nb1 + tile], lnA = F.B[v0 * nb1 + tile + 1] - stA;
                    const uint32_t stB = F.B[v1 * nb1 + tile], lnB = v0 + 1 < nvis ? F.B[v1 * nb1 + tile + 1] - stB : 0;
                    const uint2* srcA = db.frag + (uint64_t)F.vpage[v0] * db.bucket_size + stA;
                    const uint2* srcB = db.frag + (uint64_t)F.vpage[v1] * db.bucket_size + stB;
                    // m/z window as one unsigned compare on the bit patterns (exact for flo > 0: positive floats order like their bits);
                    // otherwise an always-false bit window and the float compare decides
                    const float floA = F.vflo[v0], fhiA = F.vfhi[v0], floB = F.vflo[v1], fhiB = F.vfhi[v1];
                    const bool bitsA = floA > 0.0f && fhiA >= floA, bitsB = floB > 0.0f && fhiB >= floB;
                    const uint32_t lbA = __float_as_uint(floA), spA = __float_as_uint(fhiA) - lbA;
                    const uint32_t lbB = __float_as_uint(floB), spB = __float_as_uint(fhiB) - lbB;
                    const uint32_t mx = max(lnA, lnB);
                    for (uint32_t e0 = 0; e0 < mx; e0 += 128) {
                        uint2 fa[4], fb[4];
#pragma unroll
                        for (int u = 0; u < 4; u++) {
                            const uint32_t e = e0 + u * 32 + lane;
                            fa[u] = e < lnA ? __ldg(srcA + e) : make_uint2(0xFFFFFFFFu, 0x7FC00000u);
                            fb[u] = e < lnB ? __ldg(srcB + e) : make_uint2(0xFFFFFFFFu, 0x7FC00000u);
                        }
#pragma unroll
                        for (int u = 0; u < 4; u++) {
                            bool ha = fa[u].x - t_lo <= t_span, hb = fb[u].x - t_lo <= t_span;
                            if (bitsA && sc.wide_variant) ha = ha && (fa[u].y - lbA <= spA);
                            else { const float m = __uint_as_float(fa[u].y); ha = ha && m >= floA && m <= fhiA; }
                            if (bitsB && sc.wide_variant) hb = hb && (fb[u].y - lbB <= spB);
                            else { const float m = __uint_as_float(fb[u].y); hb = hb && m >= floB && m <= fhiB; }
                            if (ha) { const uint32_t idx = fa[u].x - pep_lo; atomicAdd(&S.cnt32[idx >> 1], 1u << ((idx & 1) * 16)); }
                            if (hb) { const uint32_t idx = fb[u].x - pep_lo; atomicAdd(&S.cnt32[idx >> 1], 1u << ((idx & 1) * 16)); }
                        }
                    }
                }
            } else
            for (uint32_t tbase = 0; tbase < ntask; tbase += WIDE_THREADS) {
                const uint32_t t = tbase + tid;
                uint32_t bl = 0, nb = 0;
                float flo = 0.f, fhi = 0.f;
                if (t < ntask) {
                    const uint32_t p = t / nfc, fc = t - p * nfc + 1;
                    const float mass = __fmul_rn(__ldg(b.masses + p0 + p), (float)fc);  // scoring.rs:360
                    tol_bounds(sc.fragment_tol, mass, flo, fhi);
                    if (tile == 0 || t >= WIDE_TCACHE) {
                        const int klo = f32_key(flo), khi = f32_key(fhi);
                        uint32_t br;
                        binary_search_slice(db.n_bucket, [&](uint32_t i) { return f32_key(__ldg(db.bucket_min + i)) < klo; },
                                            [&](uint32_t i) { return f32_key(__ldg(db.bucket_min + i)) <= khi; }, bl, br);
                        nb = br - bl;
                        if (t < WIDE_TCACHE) { S.u.slow.task_bl[t] = bl; S.u.slow.task_nb[t] = (uint16_t)min(nb, 0xFFFFu); }
                        if (nb > 0xFFFFu && t < WIDE_TCACHE) S.u.slow.task_nb[t] = 0xFFFF;  // (absurd tolerances) recomputed below
                    } else {
                        bl = S.u.slow.task_bl[t];
                        nb = S.u.slow.task_nb[t];
                        if (nb == 0xFFFFu) {
                            const int klo = f32_key(flo), khi = f32_key(fhi);
                            uint32_t br;
                            binary_search_slice(db.n_bucket, [&](uint32_t i) { return f32_key(__ldg(db.bucket_min + i)) < klo; },
                                                [&](uint32_t i) { return f32_key(__ldg(db.bucket_min + i)) <= khi; }, bl, br);
                            nb = br - bl;
                        }
                    }
                }
                for (uint32_t round = 0;; round++) {
                    const bool have = round < nb;
                    if (!__syncthreads_or(have)) break;
                    WideRange r;
                    r.start = 0; r.len = 0; r.flo = flo; r.fhi = fhi;
                    if (have) {
                        const uint32_t page = bl + round;
                        const uint64_t pbase = (uint64_t)page * db.bucket_size;
                        const uint32_t pn = (uint32_t)(min(pbase + db.bucket_size, db.n_frag) - pbase);
                        const uint2* slice = db.frag + pbase;
                        const uint64_t vid64 = (uint64_t)round * ntask + t;
                        const bool cached = vid64 < WIDE_VMAX;
                        uint32_t start;
                        if (tile == 0) {
                            start = page_lower_bound(slice, 0, pn, q.pre_lo);            // partition_point(pep < pre_idx_lo)
                            my_pages++;
                            my_entries -= (long long)(start == 0 ? 0 : start - 1);       // inner_left = saturating_sub(.., 1)
                        } else {
                            start = cached ? S.u.slow.cur[(uint32_t)vid64] : page_lower_bound(slice, 0, pn, pep_lo);
                        }
                        const uint32_t end = page_lower_bound(slice, start, pn, pep_hi_excl);
                        if (cached) S.u.slow.cur[(uint32_t)vid64] = end;
                        if (last_tile) my_entries += (long long)end;                     // inner_right
                        r.start = pbase + start;
                        r.len = end - start;
                    }
                    if (tid == 0) S.s_nranges = 0;
                    __syncthreads();
                    if (r.len) S.u.slow.ranges[atomicAdd(&S.s_nranges, 1u)] = r;   // order is irrelevant for counting
                    __syncthreads();
                    // all threads walk the ranges together; 8 independent ranges (one 8-byte entry each per thread) are in flight at a
                    // time, so a 512-thread CTA keeps 32 KB of index loads outstanding
                    const uint32_t nr = S.s_nranges;
                    for (uint32_t r0 = 0; r0 < nr; r0 += 8) {
                        uint32_t maxlen = 0;
#pragma unroll
                        for (int u = 0; u < 8; u++) maxlen = max(maxlen, r0 + u < nr ? S.u.slow.ranges[r0 + u].len : 0u);
                        for (uint32_t e = tid; e < maxlen; e += WIDE_THREADS) {
                            uint2 f[8];
#pragma unroll
                            for (int u = 0; u < 8; u++) {
                                const bool ok = r0 + u < nr && e < S.u.slow.ranges[r0 + u].len;
                                f[u] = ok ? __ldg(db.frag + S.u.slow.ranges[r0 + u].start + e) : make_uint2(0xFFFFFFFFu, 0x7FC00000u);
                            }
#pragma unroll
                            for (int u = 0; u < 8; u++) {
                                const float fmz = __uint_as_float(f[u].y);
                                if (f[u].x >= q.eff_lo && f[u].x <= q.eff_hi) {
                                    const WideRange& rr = S.u.slow.ranges[min(r0 + u, nr - 1)];
                                    if (fmz >= rr.flo && fmz <= rr.fhi) {
                                        const uint32_t idx = f[u].x - pep_lo;   // < dn by construction of the sub-slice
                                        atomicAdd(&S.cnt32[idx >> 1], 1u << ((idx & 1) * 16));
                                        my_matched++;
                                    }
                                }
                            }
                        }
                    }
                    __syncthreads();
                }
            }
            __syncthreads();
            // ---- trim, stage 1 (parallel): the heap replay itself is inherently serial (its ORDER is observable), so this CTA only
            // emits, in dense order, the keys that can still enter the heap: the literal first k slots, then every slot whose matched
            // count reaches `level` = the largest m with >= k earlier slots (previous tiles) having matched >= m  (such a key is
            // preceded by k strictly greater keys, so bounded_min_heapify can never take it). k_replay_wide replays them, one
            // thread per query. If a list overflows, this CTA replays it itself and continues serially (s_serial).
            auto cnt = [&](uint32_t i) -> uint32_t { return (S.cnt32[i >> 1] >> ((i & 1) * 16)) & 0xFFFFu; };
            uint32_t scan_from = 0;
            {   // the literal first k dense slots open the list (they may spread over several tiles when the leading block-mode tiles are short)
                const uint32_t lit0 = S.s_lit, nlit = min(k - lit0, dn);   // uniform: s_lit only changes behind the barrier below
                if (nlit) {
                    for (uint32_t i = tid; i < nlit; i += WIDE_THREADS) {
                        const uint32_t c = cnt(i);
                        if (!blockmode) { nz += c != 0; msum += c; }   // block mode counted both while walking
                        if (c) atomicAdd(&S.hist[min(c, WIDE_HLEV - 1)], 1u);
                        list[lit0 + i] = c ? prescore_key(c, pep_lo + i, q.charge, q.iso) : PRESCORE_DEFAULT;
                    }
                    __syncthreads();
                    if (tid == 0) { S.s_lit = lit0 + nlit; S.s_listn = lit0 + nlit; }
                    scan_from = nlit;
                    __syncthreads();
                }
            }
            if (!S.s_serial) {
                const uint32_t level = S.s_level;
                const bool qmode = use_q && S.s_qn <= WIDE_QCAP;   // uniform
                uint32_t total = 0;
                bool overflow = false;
                if (qmode) {
                    // the tile's survivors are the queued slots (count >= level at the end of the walk, each queued exactly once); order them by
                    // slot with a rank count (a few dozen entries per tile), skip the literal slots, emit in dense order
                    const uint32_t nq = S.s_qn;
                    const uint32_t myslot = tid < nq ? S.u.blk.qslot[tid] : 0xFFFFFFFFu;
                    const bool valid = tid < nq && myslot >= scan_from;
                    total = (uint32_t)__syncthreads_count(valid);
                    overflow = S.s_listn + total > sc.wide_lmax;
                    if (valid && !overflow) {
                        uint32_t rank = 0;
                        for (uint32_t j = 0; j < nq; j++) {
                            const uint32_t sj = S.u.blk.qslot[j];
                            rank += sj < myslot && sj >= scan_from;
                        }
                        const uint32_t c = cnt(myslot);
                        list[S.s_listn + rank] = prescore_key(c, pep_lo + myslot, q.charge, q.iso);
                        atomicAdd(&S.hist[min(c, WIDE_HLEV - 1)], 1u);
                    }
                } else {
                // each warp owns a contiguous segment (multiple of 256 slots, 8-aligned); a lane reads 8 slots with one 16-byte load.
                // pass 1 counts survivors and feeds the histogram, pass 2 writes them in dense order
                const uint32_t base0 = scan_from & ~7u;
                const uint32_t span = dn - base0;
                const uint32_t seg = ((span + nwarps - 1) / nwarps + 255) & ~255u;
                const uint32_t w_lo = base0 + warp * seg, w_hi = min(dn, w_lo + seg);
                const uint4* cnt128 = reinterpret_cast<const uint4*>(S.cnt32);
                uint32_t wcount = 0;
                // branch-free SIMD-in-register pass over packed u16 pairs: non-zero slots (scored_candidates) and survivors (matched >= level).
                // Only survivors feed the histogram: slots below `level` cannot raise it (level is monotone), so skipping them keeps the bound valid.
                const uint32_t lvl2 = level | (level << 16);
                for (uint32_t i0 = w_lo; i0 < w_hi; i0 += 256) {
                    const uint32_t i = i0 + 8 * lane;
                    if (i >= w_hi) continue;
                    const uint4 w4 = cnt128[i >> 3];
                    if ((w4.x | w4.y | w4.z | w4.w) == 0) continue;
                    const uint32_t ww[4] = {w4.x, w4.y, w4.z, w4.w};
                    const bool edge = i < scan_from || i + 8 > dn;   // first / last 16-byte group of the scanned range: mask slot by slot
                    if (!edge) {
                        uint32_t nzm = 0, svm = 0;
#pragma unroll
                        for (int u = 0; u < 4; u++) {
                            nzm += __popc(__vcmpne2(ww[u], 0u));
                            svm += __popc(__vcmpgeu2(ww[u], lvl2) & __vcmpne2(ww[u], 0u));
                            if (!blockmode) msum += (ww[u] & 0xFFFFu) + (ww[u] >> 16);
                        }
                        if (!blockmode) nz += nzm >> 4;
                        wcount += svm >> 4;
                        if (svm == 0) continue;
                    }
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const uint32_t c = (ww[u >> 1] >> ((u & 1) * 16)) & 0xFFFFu;
                        if (c && i + u >= scan_from && i + u < dn) {
                            if (edge) { wcount += c >= level; if (!blockmode) { nz++; msum += c; } }
                            if (c >= level) atomicAdd(&S.hist[min(c, WIDE_HLEV - 1)], 1u);
                        }
                    }
                }
                for (int o = 16; o > 0; o >>= 1) wcount += __shfl_down_sync(0xffffffffu, wcount, o);
                if (lane == 0) S.s_warp[warp] = wcount;
                __syncthreads();
                uint32_t woff = S.s_listn;
                for (uint32_t w = 0; w < nwarps; w++) {
                    const uint32_t x = S.s_warp[w];
                    if (w < warp) woff += x;
                    total += x;
                }
                overflow = S.s_listn + total > sc.wide_lmax;
                if (!overflow && S.s_warp[warp] != 0) {
                    for (uint32_t i0 = w_lo; i0 < w_hi; i0 += 256) {
                        const uint32_t i = i0 + 8 * lane;
                        uint32_t cc[8];
                        uint32_t mine = 0;
                        uint4 w4 = make_uint4(0, 0, 0, 0);
                        if (i < w_hi) w4 = cnt128[i >> 3];
                        const uint32_t ww[4] = {w4.x, w4.y, w4.z, w4.w};
                        uint32_t pre = 0;
#pragma unroll
                        for (int u = 0; u < 4; u++) pre |= __vcmpgeu2(ww[u], lvl2) & __vcmpne2(ww[u], 0u);
                        if (!__any_sync(0xffffffffu, pre != 0)) continue;
#pragma unroll
                        for (int u = 0; u < 8; u++) {
                            const uint32_t c = (ww[u >> 1] >> ((u & 1) * 16)) & 0xFFFFu;
                            cc[u] = (c >= level && c != 0 && i + u >= scan_from && i + u < dn) ? c : 0;
                            mine += cc[u] != 0;
                        }
                        if (!__any_sync(0xffffffffu, mine != 0)) continue;
                        uint32_t incl = mine;
                        for (int o = 1; o < 32; o <<= 1) {
                            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
                            if (lane >= (uint32_t)o) incl += v;
                        }
                        uint32_t pos = woff + incl - mine;
#pragma unroll
                        for (int u = 0; u < 8; u++)
                            if (cc[u]) list[pos++] = prescore_key(cc[u], q.pre_lo + d0 + i + u, q.charge, q.iso);
                        woff += __shfl_sync(0xffffffffu, incl, 31);
                    }
                }
                }   // scan / queue
                __syncthreads();
                if (tid == 0) {
                    if (!overflow) {
                        S.s_listn += total;
                        uint32_t acc = 0, lv = 1;  // new level: largest m >= 1 with #(matched >= m) >= k among the slots seen so far
                        for (int l = WIDE_HLEV - 1; l >= 1; l--) {
                            acc += S.hist[l];
                            if (acc >= k) { lv = (uint32_t)l; break; }
                        }
                        S.s_level = lv;
                    } else {
                        // replay what was listed so far (heap.rs:7-28), then go serial for this tile and the rest of the query
                        const uint32_t nl = S.s_listn;
                        for (uint32_t i = 0; i < k; i++) S.heap[i] = list[i];
                        for (uint32_t i = k / 2; i-- > 0;) sift_down(S.heap, k, i);
                        for (uint32_t j = k; j < nl; j++) {
                            const uint64_t kq = list[j];
                            if (kq > S.heap[0]) { S.heap[0] = kq; sift_down(S.heap, k, 0); }
                        }
                        S.s_serial = 1;
                        atomicAdd(b.counters + C_WOVERFLOW, 1ull);
                    }
                }
                __syncthreads();
            }
            if (S.s_serial) {
                const bool count_nz = tile_entered_serial && !blockmode;  // pass 1 above (or the block-mode walk) already counted this tile's non-zero slots otherwise
                for (uint32_t base = scan_from; base < dn; base += 2 * WIDE_THREADS) {
                    uint64_t key[2];
                    uint32_t ncand = 0;
                    const uint64_t hmin = S.heap[0];
#pragma unroll
                    for (int u = 0; u < 2; u++) {
                        const uint32_t i = base + 2 * tid + u;
                        const uint32_t c = i < dn ? cnt(i) : 0;
                        if (count_nz) { nz += c != 0; msum += c; }
                        const uint64_t kk = prescore_key(c, q.pre_lo + d0 + i, q.charge, q.iso);
                        if (c != 0 && kk > hmin) key[ncand++] = kk;
                    }
                    if (__syncthreads_or(ncand != 0)) {
                        uint32_t incl = ncand;
                        for (int o = 1; o < 32; o <<= 1) {
                            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
                            if (lane >= (uint32_t)o) incl += v;
                        }
                        if (lane == 31) S.s_warp[warp] = incl;
                        __syncthreads();
                        uint32_t off = 0, total = 0;
                        for (uint32_t w = 0; w < nwarps; w++) {
                            const uint32_t x = S.s_warp[w];
                            if (w < warp) off += x;
                            total += x;
                        }
                        off += incl - ncand;
                        for (uint32_t u = 0; u < ncand; u++) S.queue[off + u] = key[u];
                        __syncthreads();
                        if (tid == 0) {
                            for (uint32_t j = 0; j < total; j++) {
                                const uint64_t kq = S.queue[j];
                                if (kq > S.heap[0]) { S.heap[0] = kq; sift_down(S.heap, k, 0); }
                            }
                        }
                        __syncthreads();
                    }
                }
            }
            __syncthreads();
        }
        (void)my_matched;
        const uint32_t matched_total = block_sum_u32(msum, S.s_warp);
        const uint32_t pages_total = block_sum_u32(my_pages, S.s_warp);
        const uint32_t nonzero_total = block_sum_u32(nz, S.s_warp);
        // entries: sum of (inner_right - inner_left) over page visits; per-thread partial sums can be negative, total is not
        long long ent = my_entries;
        for (int o = 16; o > 0; o >>= 1) ent += __shfl_down_sync(0xffffffffu, ent, o);
        if (lane == 0 && ent) atomicAdd(b.counters + C_ENTRIES, (unsigned long long)ent);
        if (tid == 0) {
            atomicAdd(b.counters + C_TASKS, (unsigned long long)ntask);
            atomicAdd(b.counters + C_PAGES, (unsigned long long)pages_total);
            atomicAdd(b.counters + C_MATCHED, (unsigned long long)matched_total);
        }
        QueryHits* h = b.hits + item;
        WideSlot* slot = wslots + S.s_slot;
        if (matched_total == 0) {
            if (tid == 0) {
                h->n = 0; h->default_run = q.potential; h->matched_peaks = 0; h->scored_candidates = 0;
                slot->off = list_off; slot->item = item; slot->n_list = 0; slot->state = 1; slot->k = k;
            }
            continue;
        }
        if (S.s_serial) {
            uint64_t* keys = b.hit_keys + (size_t)item * sc.kparam;
            for (uint32_t i = tid; i < k; i += WIDE_THREADS) keys[i] = S.heap[i];
        }
        if (tid == 0) {
            h->n = k; h->default_run = 0; h->matched_peaks = matched_total; h->scored_candidates = nonzero_total;
            slot->off = list_off; slot->item = item; slot->n_list = S.s_listn; slot->state = S.s_serial ? 1 : 0; slot->k = k;
        }
    }
}

// SURVEY.md §8d work counters of the open-search queries in the REFERENCE's terms (pages visited, entries of [inner_left, inner_right) the
// filter database.rs:514 walks): the block-index path of k_prelim_wide never touches the page layout, so the counters that feed the
// algorithmic-bytes figure are produced here, one warp per query, from the bucket minima and the page-grid directory alone (no entry is read).
__global__ void __launch_bounds__(256) k_wide_account(DbView db, ScorerView sc, BatchView b) {
    const uint32_t lane = threadIdx.x & 31, w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const unsigned long long nw = min(b.counters[C_WIDE], (unsigned long long)b.wide_cap);
    if (w >= nw) return;
    const uint32_t item = b.wide_items[w];
    const QueryDesc q = b.queries[item];
    const uint32_t s = item / sc.qmax;
    const uint32_t p0 = b.peak_off[s], np = b.peak_off[s + 1] - p0;
    const uint32_t nfc = q.nfc, ntask = np * nfc;
    if (ntask > WIDE_TMAX) return;   // such a query took the page-slice path of k_prelim_wide, which counts for itself
    unsigned long long pages = 0, entries = 0;
    for (uint32_t t = lane; t < ntask; t += 32) {
        const uint32_t p = t / nfc, fc = t - p * nfc + 1;
        const float mass = __fmul_rn(__ldg(b.masses + p0 + p), (float)fc);  // scoring.rs:360
        float flo, fhi;
        tol_bounds(sc.fragment_tol, mass, flo, fhi);
        uint32_t bl, br;
        bucket_range(db, flo, fhi, bl, br);
        for (uint32_t page = bl; page < br; page++) {
            const uint64_t pbase = (uint64_t)page * db.bucket_size;
            const uint32_t pn = (uint32_t)(min(pbase + db.bucket_size, db.n_frag) - pbase);
            const uint32_t st = page_lower_bound_dir(db, page, db.frag + pbase, pn, q.pre_lo);        // partition_point(pep < pre_idx_lo)
            const uint32_t en = page_lower_bound_dir(db, page, db.frag + pbase, pn, q.pre_hi + 1);    // inner_right
            entries += en - (st == 0 ? 0 : st - 1);                                                     // inner_left = saturating_sub(.., 1)
            pages++;
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        pages += __shfl_down_sync(0xffffffffu, pages, o);
        entries += __shfl_down_sync(0xffffffffu, entries, o);
    }
    if (lane == 0) {
        if (pages) atomicAdd(b.counters + C_PAGES, pages);
        if (entries) atomicAdd(b.counters + C_ENTRIES, entries);
    }
}

// trim, stage 2: bounded_min_heapify (heap.rs:7-28) over each query's ordered key list, ONE THREAD PER QUERY, so that the inherently
// serial replays (their result ORDER is observable) of all queries of the batch run concurrently instead of stalling a whole CTA each.
// Heaps live in shared memory, interleaved by thread. Used by both preliminary-scoring kernels.
constexpr int REPLAY_THREADS = 128;
// COMPACT (narrow windows, <= NARROW_CAP peptides): inside one query precursor charge and isotope error are constants and PeptideIx - pre_idx_lo
// fits 16 bits, so the heap holds 32-bit keys (matched << 16 | PeptideIx - pre_idx_lo; PreScore::default() -> 0x0000FFFF, below every real key,
// which has matched >= 1): same order as the packed 64-bit PreScore, half the shared memory (twice the resident CTAs) and half the LDS traffic.
template <bool COMPACT>
__global__ void __launch_bounds__(REPLAY_THREADS) k_replay(ScorerView sc, BatchView b, const uint64_t* lists, const ReplaySlot* slots, uint32_t n_slots,
                                                           const unsigned long long* n_slots_dev, uint32_t n_spectra) {
    typedef typename std::conditional<COMPACT, uint32_t, uint64_t>::type key_t;
    extern __shared__ __align__(8) unsigned char rheap_raw[];
    key_t* const rheap = reinterpret_cast<key_t*>(rheap_raw);  // [kparam][REPLAY_THREADS]
    uint32_t slot = blockIdx.x * REPLAY_THREADS + threadIdx.x;
    if (n_slots_dev != nullptr) n_slots = (uint32_t)min((unsigned long long)n_slots, *n_slots_dev);   // slots actually filled (device-side count)
    if (slot >= n_slots) return;
    // per-item slots (narrow kernels): walk them query-slot-major, so the lanes of a warp hold queries of the same slot — with known-charge
    // spectra only slot 0 has work, and item-major order would leave two lanes in three idle
    // (and in precursor order: neighbouring windows have similar sizes, so the lanes of a warp replay lists of similar length)
    if (n_spectra) { const uint32_t pos = slot % n_spectra; slot = (b.order ? b.order[pos] : pos) * sc.qmax + slot / n_spectra; }
    const ReplaySlot ws = slots[slot];
    if (ws.state != 0) return;
    const uint64_t* list = lists + ws.off;
    const uint32_t k = ws.k, tid = threadIdx.x;
    uint32_t pre_lo = 0, q_charge = 0;
    int q_iso = 0;
    if (COMPACT) { const QueryDesc q = b.queries[ws.item]; pre_lo = q.pre_lo; q_charge = q.charge; q_iso = q.iso; }
    auto pack = [&](uint64_t k64) -> key_t {
        if (!COMPACT) return (key_t)k64;
        return (key_t)(key_peptide(k64) == 0xFFFFFFFFu ? 0x0000FFFFu : ((key_matched(k64) << 16) | (key_peptide(k64) - pre_lo)));
    };
    auto unpack = [&](key_t kk) -> uint64_t {
        if (!COMPACT) return (uint64_t)kk;
        const uint32_t v = (uint32_t)kk;
        return v == 0x0000FFFFu ? PRESCORE_DEFAULT : prescore_key(v >> 16, pre_lo + (v & 0xFFFFu), q_charge, q_iso);
    };
    auto H = [&](uint32_t i) -> key_t& { return rheap[i * REPLAY_THREADS + tid]; };
    // sift_down (heap.rs:31-60) of `val` from `index`, written with a hole: children smaller than val move up, val lands where the swaps
    // of the reference would have carried it (same path: the smaller child, the left one on ties, and only if it is < val)
    auto sift = [&](uint32_t index, key_t val) {
        for (;;) {
            const uint32_t l = index * 2 + 1;
            if (l >= k) break;
            uint32_t c = l;
            key_t cv = H(l);
            if (l + 1 < k) { const key_t cr = H(l + 1); if (cr < cv) { cv = cr; c = l + 1; } }
            if (!(cv < val)) break;
            H(index) = cv;
            index = c;
        }
        H(index) = val;
    };
    for (uint32_t i = 0; i < k; i++) H(i) = pack(__ldg(list + i));
    for (uint32_t i = k / 2; i-- > 0;) sift(i, H(i));
    key_t root = H(0);
    uint64_t nxt = k < ws.n_list ? __ldg(list + k) : 0;
    for (uint32_t j = k; j < ws.n_list; j++) {
        const key_t kq = pack(nxt);
        if (j + 1 < ws.n_list) nxt = __ldg(list + j + 1);   // in flight while the heap is updated
        if (kq > root) { sift(0, kq); root = H(0); }
    }
    uint64_t* keys = b.hit_keys + (size_t)ws.item * sc.kparam;
    for (uint32_t i = 0; i < k; i++) keys[i] = unpack(H(i));
}

// ------------------------------------------------------------------------------------------------ scoring
struct ScoreRec {
    double hyperscore;
    uint32_t peptide;
    uint32_t matched_b, matched_y;
    float summed_b, summed_y;
    uint32_t longest_b, longest_y;
    float ppm_difference;
    uint32_t charge;
    int iso;
    uint32_t valid;
    uint32_t plen;
};

// select_most_intense_peak (spectrum.rs:134-159), offset None — exact binary_search_slice emulation (any input)
__device__ SB_RARE int select_most_intense_peak(const float* masses, const float* intens, uint32_t n, float center, const Tol& tol) {
    float lo, hi;
    tol_bounds(tol, center, lo, hi);
    lo = __fadd_rn(lo, 0.0f);
    hi = __fadd_rn(hi, 0.0f);
    const int klo = f32_key(lo), khi = f32_key(hi);
    uint32_t i, j;
    binary_search_slice(n, [&](uint32_t k) { return f32_key(masses[k]) < klo; }, [&](uint32_t k) { return f32_key(masses[k]) <= khi; }, i, j);
    int best = -1;
    float max_int = 0.0f;
    for (uint32_t idx = i; idx < j; idx++) {
        const float m = masses[idx];
        if (m >= lo && m <= hi) {
            const float it = intens[idx];
            if (it >= max_int) { max_int = it; best = (int)idx; }
        }
    }
    return best;
}
// Same result for spectra whose masses are verified ascending, positive and non-NaN: the in-window peaks are then one contiguous
// run, found from the bucket LUT and scanned in index order with the reference's comparisons (>= keeps the last of equal maxima).
__device__ __forceinline__ int select_most_intense_peak_lut(const float* masses, const float* intens, uint32_t n, float center, const Tol& tol,
                                                            const LutParams& LP, const uint16_t* lut) {
    float lo, hi;
    tol_bounds(tol, center, lo, hi);
    lo = __fadd_rn(lo, 0.0f);
    hi = __fadd_rn(hi, 0.0f);
    uint32_t idx = lut_start(LP, lut, lo, SPEC_LUT_CELLS);
    while (idx < n && masses[idx] < lo) idx++;
    int best = -1;
    float max_int = 0.0f;
    while (idx < n) {
        const float m = masses[idx];
        if (!(m <= hi)) break;
        const float it = intens[idx];
        if (it >= max_int) { max_int = it; best = (int)idx; }
        idx++;
    }
    return best;
}

// f64::ln as the host libm computes it (glibc_log.cuh): variant selected by the host probe
__device__ __forceinline__ double ref_ln(const ScorerView& sc, double x) { return glog::glibc_log_v(x, (int)sc.log_variant); }
// lnfact (scoring.rs:170-177)
__device__ __forceinline__ double lnfact(const ScorerView& sc, uint32_t n) {
    if (n < sc.lnfact_n) return __ldg(sc.lnfact_tab + n);
    if (n == 0) return 1.0;
    const double x = (double)n;
    return x * ref_ln(sc, x) - x + 0.5 * ref_ln(sc, x) + 0.5 * ref_ln(sc, 3.14159265358979323846 * 2.0 * x);
}
// ScoreType::score (scoring.rs:179-201)
__device__ __forceinline__ double hyperscore_of(const ScorerView& sc, uint32_t mb, uint32_t my, float sb, float sy) {
    double s;
    if (sc.score_type == 0) {
        const double i = (double)__fadd_rn(sb, 1.0f) * (double)__fadd_rn(sy, 1.0f);
        s = ref_ln(sc, i) + lnfact(sc, mb) + lnfact(sc, my);
    } else {
        // f32::ln_1p is libm's log1pf: reproduced operation by operation (glibc_log.cuh, checked against glibc on every float)
        const float si = __fadd_rn(sb, sy);
        s = (double)glog::glibc_log1pf(si) + lnfact(sc, mb) + lnfact(sc, my);
    }
    return isfinite(s) ? s : 255.0;
}

// Run (scoring.rs:771-793)
struct Run {
    uint32_t start, length, last, longest;
    __device__ __forceinline__ void matched(uint32_t index) {
        if (last == index) return;
        if (start + length == index) { length += 1; longest = max(longest, length); }
        else { start = index; length = 1; longest = max(longest, length); }
        last = index;
    }
};

// One warp scores one candidate (score_candidate, scoring.rs:675-767). Lanes look up theoretical fragments in parallel (ions
// precomputed per peptide) and each computes its own ppm term; matched fragments are then folded in the reference's order
// (kind, ion index, charge) with a ballot loop so the f32 accumulations (summed_b/y, ppm_difference) are bit-identical.
struct SpecView { const float* masses; const float* intens; uint32_t np; bool use_lut; LutParams lp; const uint16_t* lut; };

__device__ SB_RARE void score_candidate_warp(const DbView& db, const ScorerView& sc, uint64_t key, const SpecView& sp, ScoreRec* out,
                                                     uint8_t* mark /*nullable: remove_matched_peaks marks*/) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t pep = key_peptide(key), charge = key_charge(key);
    const uint32_t L = __ldg(db.pep_len + pep);
    const uint32_t nions = L - 1;
    const uint32_t nfc = max_fragment_charge(sc.max_fragment_charge_opt, charge) - 1;
    const float* ions = db.ions + __ldg(db.ion_off + pep);
    const uint32_t per_kind = nions * nfc, total = per_kind * db.n_kinds;
    uint32_t mb = 0, my = 0;
    float sb = 0.f, sy = 0.f, ppm = 0.f;
    Run brun = {0, 0, 0, 0}, yrun = {0, 0, 0, 0};
    for (uint32_t base = 0; base < total; base += 32) {
        const uint32_t f = base + lane;
        int pk = -1;
        float term = 0.f, inten = 0.f;
        uint32_t idx = 0;
        bool is_n = false;
        if (f < total) {
            // f = (kind * nions + idx) * nfc + (fc - 1); nfc is 1..3 in practice: divide by compile-time constants
            uint32_t ki, fc;
            switch (nfc) {
                case 1: ki = f; fc = 1; break;
                case 2: ki = f >> 1; fc = (f & 1) + 1; break;
                case 3: ki = f / 3; fc = f - ki * 3 + 1; break;
                default: ki = f / nfc; fc = f - ki * nfc + 1; break;
            }
            uint32_t kind_i = ki >= nions;   // two ion kinds (b/y) in practice: one compare; more kinds finish in the loop
            idx = ki - (kind_i ? nions : 0);
            while (idx >= nions) { idx -= nions; kind_i++; }   // <= n_kinds - 2 iterations
            is_n = (db.nterm_mask >> kind_i) & 1;
            // scoring.rs:707 fragment / charge (ions[kind_i * nions + idx] == ions[ki]): x / 1 and x / 2 are exact as x and x * 0.5 (|x| >= 2^-125)
            const float ion = __ldg(ions + ki);
            const float mz = fc == 1 ? ion : (fc == 2 && fabsf(ion) >= 1e-30f) ? __fmul_rn(ion, 0.5f) : __fdiv_rn(ion, (float)fc);
            pk = sp.use_lut ? select_most_intense_peak_lut(sp.masses, sp.intens, sp.np, mz, sc.fragment_tol, sp.lp, sp.lut)
                            : select_most_intense_peak(sp.masses, sp.intens, sp.np, mz, sc.fragment_tol);
            if (pk >= 0 && mark == nullptr) {
                const float peak_mass = sp.masses[pk];
                inten = sp.intens[pk];
                // scoring.rs:719-720: peak_intensity * (mz - peak_mass).abs() * 2E6 / (mz + peak_mass)
                term = __fdiv_rn(__fmul_rn(__fmul_rn(inten, fabsf(__fsub_rn(mz, peak_mass))), 2E6f), __fadd_rn(mz, peak_mass));
            }
        }
        if (mark != nullptr) {
            if (pk >= 0) mark[pk] = 1;
            continue;
        }
        uint32_t mask = __ballot_sync(0xffffffffu, pk >= 0);
        const uint32_t maskn = __ballot_sync(0xffffffffu, pk >= 0 && is_n);
        mb += __popc(maskn);
        my += __popc(mask & ~maskn);
        while (mask) {
            const int src = __ffs(mask) - 1;
            mask &= mask - 1;
            const float t = __shfl_sync(0xffffffffu, term, src);
            const float it = __shfl_sync(0xffffffffu, inten, src);
            const uint32_t ib = __shfl_sync(0xffffffffu, idx, src);
            ppm = __fadd_rn(ppm, t);
            if ((maskn >> src) & 1) { sb = __fadd_rn(sb, it); brun.matched(ib); }
            else { sy = __fadd_rn(sy, it); yrun.matched(ib); }
        }
    }
    if (mark == nullptr && lane == 0) {
        ScoreRec r;
        r.peptide = pep; r.charge = charge; r.iso = key_iso(key);
        r.matched_b = mb & 0xFFFF; r.matched_y = my & 0xFFFF; r.summed_b = sb; r.summed_y = sy;
        r.longest_b = brun.longest; r.longest_y = yrun.longest;
        r.hyperscore = 0.0;          // (this warp-per-candidate variant only serves remove_matched_peaks / tests; score_candidates_flat fills real records)
        r.ppm_difference = ppm;
        r.valid = 0;
        r.plen = L;
        *out = r;
    }
}

struct FeatureOut {  // layout == sage_b200_feature
    uint32_t spectrum, peptide_idx, peptide_len, rank;
    int32_t label;
    float expmass, calcmass;
    uint32_t charge;
    float rt, ims, delta_mass, isotope_error, average_ppm;
    uint32_t _pad0;
    double hyperscore, delta_next, delta_best;
    uint32_t matched_peaks, longest_b, longest_y;
    float longest_y_pct;
    uint32_t missed_cleavages;
    float matched_intensity_pct;
    uint32_t scored_candidates;
    float ms2_intensity;
    double poisson;
    uint32_t fragment_offset, fragment_count;
};
static_assert(sizeof(FeatureOut) == 128, "feature layout");
static_assert(SCORE_THREADS >= K_MAX, "k_score ranks candidates one per thread");

// Append a per-query hit list to a merge buffer (InitialHits += , scoring.rs:60-67). All-default runs are capped at
// kparam entries: defaults beyond the first k positions can never displace the heap root, so the replay is unchanged.
__device__ __forceinline__ uint32_t append_hits(uint64_t* buf, uint32_t len, uint32_t cap, const QueryHits& h, const uint64_t* keys, uint32_t kparam) {
    if (h.n) {
        for (uint32_t i = 0; i < h.n && len < cap; i++) buf[len++] = keys[i];
    } else {
        const uint32_t d = min(h.default_run, kparam);
        for (uint32_t i = 0; i < d && len < cap; i++) buf[len++] = PRESCORE_DEFAULT;
    }
    return len;
}

struct FragmentOut { int32_t kind, charge, ordinal; float intensity, mz_calculated, mz_experimental; };  // == sage_b200_fragment

// score_candidate (scoring.rs:675-767) for ALL candidates of a spectrum at once. A candidate is L-1 ions x kinds x fragment charges sorted-array
// lookups (~45 for a tryptic peptide at z = 2); one warp per candidate leaves a third of the lanes idle and pays every prologue per candidate.
// Here the lookups of the <= k candidates are flattened into one task list t = base[c] + f (f = (kind*nions + idx)*nfc + fc-1, the reference's
// loop order), processed in tiles of `tile` tasks:
//   phase B  every lane owns one task: candidate header from smem (cursor advanced incrementally, tasks of a lane ascend), theoretical m/z
//            from the ion table, Tolerance::bounds, first peak >= lo through the spectrum LUT. A task whose peak lies inside the window is a
//            hit: one bit in the per-tile mask (warp ballot) and an entry in the warp's compact hit list.
//   phase B' the warp walks its hit list densely (about one task in five hits; doing this inside phase B would run the matched branch with
//            2-3 of 32 lanes): most intense peak of the window (last of equals), ppm term, (term, intensity) to smem.
//   fold     thread c folds candidate c's matched tasks in ascending f — exactly the reference's order of `ppm_difference +=`, `summed_b/y +=`,
//            Run::matched — keeping its partial sums in registers from tile to tile (tiles need not align with candidates).
// FAST (uniform per spectrum: LUT usable, ppm fragment tolerance of sane magnitude) is the straight-line version of the task body: division-free
// bounds and fragment / charge for charges 1..3 (div_const_rn: bit-identical to IEEE division, tests/test_div_const.py), sentinel-terminated
// scans; tasks outside its preconditions (ion outside [1, 1e20], more than 3 fragment charges) take the generic body. Results are
// bit-identical to score_candidate_warp either way (same f32 operations in the same order).
struct __align__(16) CandHdr { uint32_t ion_off, base, next; uint16_t nions; uint8_t nfc, pad; };

__device__ __forceinline__ bool fast_tol_ok(float t) { const float a = fabsf(t); return t == 0.0f || (a >= 1e-9f && a <= 1e6f); }

// ---- split scoring (k_score<true> -> k_fold -> k_features). A spectrum's CTA spends a third of its life in phases that keep one thread per
// candidate (or one thread) busy: the ordered fold, the records (f64 ln), the rank count and the Feature rows. With SPLIT the CTA only matches:
// it leaves the hits of its candidates in task order in a global arena and the candidate headers beside them; k_fold then folds ONE CANDIDATE PER
// THREAD over all spectra of the chunk (dense lanes instead of 39 of 128), k_features ranks and writes the rows, again one thread per candidate.
// Same arithmetic in the same order: sums, runs, ppm, hyperscore, rank, rows are bit-identical to the fused kernel (tests run both).
struct CandOut { uint64_t key; uint32_t h0, hcnt; uint16_t nions; uint8_t nfc, plen; uint32_t pad; };   // hits [h0, h0 + hcnt) of the spectrum's arena slice
struct SpecMeta { unsigned long long hit_base, matched_peaks, scored; uint32_t ncand, pad; };
struct SplitOut {
    CandOut* cand;              // [n][kparam]
    SpecMeta* meta;             // [n]
    uint16_t* hit_k;            // kind << 13 | ion index
    float* hit_i;               // matched intensity
    float* hit_t;               // ppm term
    unsigned long long hit_cap; // entries of the three hit arrays
    struct ScoreRec* recs;      // [n][kparam]
    unsigned long long* hkey;   // [n][kparam] sort key of build_features: order-preserving integer image of the hyperscore, 0 = below min_matched_peaks
    unsigned long long* counters;
};

// Order-preserving map f64 -> u64 (x < y <=> key(x) < key(y) for non-NaN x, y; -0.0 is folded into +0.0 first) and its inverse. The rank count of
// k_features compares these keys: 64-bit integer compares instead of FP64 ones (on the FP64 pipe that kernel was several times slower).
__device__ __forceinline__ unsigned long long f64_sort_key(double d) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(d + 0.0);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double f64_from_sort_key(unsigned long long k) {
    const unsigned long long u = (k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k;
    return __longlong_as_double((long long)u);
}

// Optional per-phase cycle accounting of k_score (variant builds only: -DSAGE_B200_PHASE_CLOCKS=1): thread 0 of every CTA adds the cycles
// between consecutive marks to g_phase[i]; read back with sage_b200_debug_phase_cycles (tools/phase_cycles.py).
#if SAGE_B200_PHASE_CLOCKS
__device__ unsigned long long g_phase[16];
__shared__ long long s_ph_prev;
#define PH_START() do { if (threadIdx.x == 0) s_ph_prev = clock64(); } while (0)
#define PH(i) do { if (threadIdx.x == 0) { const long long n_ = clock64(); atomicAdd(&g_phase[i], (unsigned long long)(n_ - s_ph_prev)); s_ph_prev = n_; } } while (0)
#else
#define PH_START() do {} while (0)
#define PH(i) do {} while (0)
#endif

// Shared-memory tile of score_candidates_flat. Static (compile-time addresses: no base-pointer arithmetic in the task loop).
struct ScoreTile {
    CandHdr hdr[K_MAX + 1];        // candidate headers + sentinel
    union {
        double hkey[K_MAX];        // fused: sort keys of build_features (hyperscore, -inf when below min_matched_peaks)
        uint8_t cand[SCORE_TILE];  // SPLIT: candidate of each task slot of the tile (phase B writes it, the emit reads it for the hits)
    };
    float term[SCORE_TILE];        // phase B: m/z of a hit; phase B': its ppm term
    float inten[SCORE_TILE];       // phase B: index of the first in-window peak; phase B': matched intensity
    uint32_t mask[SCORE_TILE / 32];
    uint16_t hits[SCORE_TILE];     // per-warp compact lists of hit slots (bit 15: already final, skip in phase B')
    uint16_t lut[SPEC_LUT_CELLS];  // spectrum LUT (spectrum_lut_setup)
    uint32_t scan[SCORE_THREADS / 32];
    unsigned long long hit_base;   // SPLIT: this spectrum's slice of the hit arena
    uint32_t hit_room;             // SPLIT: 0 when the arena is too small (the host re-runs the chunk with the exact size)
};
static_assert(SCORE_TILE <= sizeof(double) * K_MAX && K_MAX <= 255, "the slot -> candidate bytes fit in hkey's bytes and hold a candidate index");

// (kind, ion index) of entry ki of a candidate's ion table (kinds concatenated, `nions` ions each): kind << 13 | index (<= 6 kinds, < 255 ions)
__device__ __forceinline__ uint32_t kind_index(uint32_t ki, uint32_t nions) {
    uint32_t kind = ki >= nions;   // two ion kinds (b/y) in practice: one compare; more kinds finish in the loop
    uint32_t idx = ki - (kind ? nions : 0);
    while (idx >= nions) { idx -= nions; kind++; }
    return kind << 13 | idx;
}

// One task of phase B, FAST preconditions checked by the caller (nfc <= 3, ion in [1, 1e20]): returns true when the tolerance window of the
// theoretical fragment holds at least one peak; mz / first in-window peak are left in `mz`, `idx`.
__device__ __forceinline__ bool fast_task(float ion, uint32_t fc, float tlo, float thi, const SpecView& sp, const uint16_t* lut, const float* pm, float& mz,
                                          uint32_t& idx) {
    // scoring.rs:707 fragment / charge: x / 1, x / 2 exact as x, x * 0.5; x / 3 through div_const_rn's two FMAs
    const float q3 = __fmul_rn(ion, 1.0f / 3.0f);
    const float third = __fmaf_rn(__fmaf_rn(-q3, 3.0f, ion), 1.0f / 3.0f, q3);
    mz = fc == 1 ? ion : (fc == 2 ? __fmul_rn(ion, 0.5f) : third);
    // Tolerance::bounds, ppm (mass.rs:21-35): c + c*t/1e6 with the division as in div_const_rn (|c*t| is inside its proven range)
    const float pl = __fmul_rn(mz, tlo), ph = __fmul_rn(mz, thi);
    const float ql = __fmul_rn(pl, 1.0f / 1000000.0f), qh = __fmul_rn(ph, 1.0f / 1000000.0f);
    const float lo = __fadd_rn(mz, __fmaf_rn(__fmaf_rn(-ql, 1000000.0f, pl), 1.0f / 1000000.0f, ql));
    const float hi = __fadd_rn(mz, __fmaf_rn(__fmaf_rn(-qh, 1000000.0f, ph), 1.0f / 1000000.0f, qh));
    // select_most_intense_peak (spectrum.rs:134-159), first half: the first peak >= lo (LUT start one cell early, then the exact values)
    const float tt = __fmul_rn(__fsub_rn(lo, sp.lp.base), sp.lp.inv_w);
    const int cc = tt > 1.0f ? (int)fminf(tt, (float)(SPEC_LUT_CELLS - 1)) - 1 : 0;
    idx = lut[cc];
    while (pm[idx] < lo) idx++;   // masses[np] = +inf ends the scan
    return pm[idx] <= hi;
}

template <bool FAST, bool SPLIT>
__device__ __forceinline__ void score_candidates_flat(const DbView& db, const ScorerView& sc, const uint64_t* cur, uint32_t ncand, const SpecView& sp,
                                                      ScoreTile& S, ScoreRec* recs, const SplitOut& so, uint32_t spec) {
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = SCORE_THREADS / 32;
    constexpr uint32_t tile = SCORE_TILE;
    // ---- phase A: candidate headers + exclusive scan of the task counts
    uint64_t key = 0;
    uint32_t L = 0, nions = 0, nfc = 1, total = 0, ion_off = 0;
    if (tid < ncand) {
        key = cur[tid];
        const uint32_t pep = key_peptide(key);
        L = __ldg(db.pep_len + pep);
        nions = L - 1;
        nfc = max_fragment_charge(sc.max_fragment_charge_opt, key_charge(key)) - 1;
        total = nions * nfc * db.n_kinds;
        ion_off = __ldg(db.ion_off + pep);
    }
    uint32_t incl = total;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= (uint32_t)o) incl += v;
    }
    if (lane == 31) S.scan[warp] = incl;
    __syncthreads();
    uint32_t base = incl - total, T = 0;
#pragma unroll
    for (uint32_t w = 0; w < nwarps; w++) {
        const uint32_t x = S.scan[w];
        if (w < warp) base += x;
        T += x;
    }
    if (tid < ncand) { CandHdr h; h.ion_off = ion_off; h.base = base; h.next = base + total; h.nions = (uint16_t)nions; h.nfc = (uint8_t)nfc; h.pad = 0; S.hdr[tid] = h; }
    if (tid == 0) { CandHdr h; h.ion_off = 0; h.base = T; h.next = 0xFFFFFFFFu; h.nions = 0; h.nfc = 1; h.pad = 0; S.hdr[ncand] = h; }   // sentinel: stops every cursor
    uint32_t hcnt = 0, hits_before = 0;   // SPLIT: hits of candidate tid so far / hits of the tiles done
    if (SPLIT && tid == 0) {   // reserve T entries (an upper bound: a task has at most one hit); the hits are written compactly from the slice's start
        const unsigned long long hb = atomicAdd(so.counters + C_HITS, (unsigned long long)T);
        const bool room = hb + T <= so.hit_cap;
        S.hit_base = hb;
        S.hit_room = room ? 1u : 0u;
        so.meta[spec].hit_base = hb;
        if (!room) so.meta[spec].ncand = 0;
    }
    // fold state of candidate tid (registers, carried across tiles)
    uint32_t mb = 0, my = 0;
    float sb = 0.f, sy = 0.f, ppm = 0.f;
    Run brun = {0, 0, 0, 0}, yrun = {0, 0, 0, 0};
    const float tlo = sc.fragment_tol.lo, thi = sc.fragment_tol.hi;
    const float* const pm = sp.masses;
    const float* const pi = sp.intens;
    // generic task body: any tolerance kind, any charge, with or without the LUT; writes the final (term, intensity)
    auto generic_task = [&](const CandHdr& h, uint32_t f, uint32_t slot) -> bool {
        uint32_t ki, fc;
        switch (h.nfc) {
            case 1: ki = f; fc = 1; break;
            case 2: ki = f >> 1; fc = (f & 1) + 1; break;
            case 3: ki = f / 3; fc = f - ki * 3 + 1; break;
            default: ki = f / h.nfc; fc = f - ki * h.nfc + 1; break;
        }
        // scoring.rs:707 fragment / charge: x / 1 and x / 2 are exact as x and x * 0.5 (|x| >= 2^-125)
        const float ion = __ldg(db.ions + h.ion_off + ki);
        const float mz = fc == 1 ? ion : (fc == 2 && fabsf(ion) >= 1e-30f) ? __fmul_rn(ion, 0.5f) : __fdiv_rn(ion, (float)fc);
        const int pk = sp.use_lut ? select_most_intense_peak_lut(pm, pi, sp.np, mz, sc.fragment_tol, sp.lp, S.lut)
                                  : select_most_intense_peak(pm, pi, sp.np, mz, sc.fragment_tol);
        if (pk < 0) return false;
        const float peak_mass = pm[pk], inten = pi[pk];
        // scoring.rs:719-720: peak_intensity * (mz - peak_mass).abs() * 2E6 / (mz + peak_mass)
        S.term[slot] = __fdiv_rn(__fmul_rn(__fmul_rn(inten, fabsf(__fsub_rn(mz, peak_mass))), 2E6f), __fadd_rn(mz, peak_mass));
        S.inten[slot] = inten;
        return true;
    };
    for (uint32_t t0 = 0; t0 < T; t0 += tile) {
        const uint32_t tn = min(tile, T - t0);
        __syncthreads();   // headers written / previous tile's fold done with the tile arrays
        PH(t0 == 0 ? 3 : 5);
        // ---- phase B: each warp takes a contiguous run of the tile; per iteration a lane owns SCORE_UNROLL tasks 32 apart (with 2: two
        // independent dependency chains, both ion loads issued before either is used)
        constexpr uint32_t STEP = 32 * SCORE_UNROLL;
        const uint32_t chunk = (((tn + nwarps - 1) / nwarps) + STEP - 1) & ~(STEP - 1);
        const uint32_t w_lo = min(tn, warp * chunk), w_hi = min(tn, w_lo + chunk);
        uint32_t c = 0, wcount = 0;
        if (w_lo < w_hi) {   // cursor start, once per warp: the last candidate whose tasks start at or before the warp's first task (bases ascend)
            const uint32_t t_first = t0 + w_lo;
            uint32_t n_le = 0;
#pragma unroll
            for (uint32_t k = 0; k < (uint32_t)K_MAX; k += 32)
                n_le += (uint32_t)__popc(__ballot_sync(0xffffffffu, k + lane < ncand && S.hdr[k + lane].base <= t_first));
            c = n_le - 1;   // base[0] = 0 <= t_first; no lane's first task lies before t_first
        }
        CandHdr h = S.hdr[c];
        for (uint32_t s0 = w_lo; s0 < w_hi; s0 += STEP) {
            const uint32_t slotA = s0 + lane, slotB = slotA + 32;
            const bool inA = slotA < w_hi, inB = SCORE_UNROLL == 2 && slotB < w_hi;
            bool hitA = false, hitB = false, finalA = false, finalB = false;   // final: (term, intensity) already written (generic body)
            // headers of both tasks (the cursor only moves forward: task B lies 32 behind task A of the next iteration)
            uint32_t fA = 0, fB = 0;
            CandHdr hA = h, hB = h;
            if (inA) {
                const uint32_t t = t0 + slotA;
                while (t >= h.next) { c++; h = S.hdr[c]; }   // skips zero-length candidates; the sentinel's next = 2^32 - 1 > t
                hA = h; fA = t - h.base;
                if (SPLIT) S.cand[slotA] = (uint8_t)c;   // the candidate of a hit, for the emit (written for every task: one store either way)
            }
            if (inB) {
                const uint32_t t = t0 + slotB;
                while (t >= h.next) { c++; h = S.hdr[c]; }
                hB = h; fB = t - h.base;
                if (SPLIT) S.cand[slotB] = (uint8_t)c;
            }
            if (FAST) {
                // f = (kind*nions + idx)*nfc + fc-1, nfc in 1..3: branch-free decode; both loads in flight before the first use
                const bool okA = inA && hA.nfc <= 3, okB = inB && hB.nfc <= 3;
                const uint32_t kiA = hA.nfc == 1 ? fA : (hA.nfc == 2 ? fA >> 1 : __umulhi(fA, 0xAAAAAAABu) >> 1);
                const uint32_t kiB = hB.nfc == 1 ? fB : (hB.nfc == 2 ? fB >> 1 : __umulhi(fB, 0xAAAAAAABu) >> 1);
                const float ionA = okA ? __ldg(db.ions + hA.ion_off + kiA) : 0.0f;
                const float ionB = okB ? __ldg(db.ions + hB.ion_off + kiB) : 0.0f;
                const bool fastA = okA && ionA >= 1.0f && ionA <= 1e20f, fastB = okB && ionB >= 1.0f && ionB <= 1e20f;
                float mzA = 0.f, mzB = 0.f;
                uint32_t idxA = 0, idxB = 0;
                if (fastA) hitA = fast_task(ionA, fA - kiA * hA.nfc + 1, tlo, thi, sp, S.lut, pm, mzA, idxA);
                if (fastB) hitB = fast_task(ionB, fB - kiB * hB.nfc + 1, tlo, thi, sp, S.lut, pm, mzB, idxB);
                if (hitA) { S.term[slotA] = mzA; S.inten[slotA] = __uint_as_float(idxA); }
                if (hitB) { S.term[slotB] = mzB; S.inten[slotB] = __uint_as_float(idxB); }
                if (inA && !fastA) hitA = finalA = generic_task(hA, fA, slotA);   // outside the fast preconditions (rare)
                if (inB && !fastB) hitB = finalB = generic_task(hB, fB, slotB);
            } else {
                if (inA) hitA = generic_task(hA, fA, slotA);
                if (inB) hitB = generic_task(hB, fB, slotB);
            }
            const uint32_t ballA = __ballot_sync(0xffffffffu, hitA), ballB = __ballot_sync(0xffffffffu, hitB);
            if (lane == 0) { S.mask[s0 >> 5] = ballA; if (SCORE_UNROLL == 2) S.mask[(s0 >> 5) + 1] = ballB; }   // (the second word may lie past tn: never read)
            if (FAST) {
                const uint32_t lt = (1u << lane) - 1;
                if (hitA) S.hits[w_lo + wcount + __popc(ballA & lt)] = (uint16_t)(slotA | (finalA ? 0x8000u : 0u));
                wcount += __popc(ballA);
                if (SCORE_UNROLL == 2) {
                    if (hitB) S.hits[w_lo + wcount + __popc(ballB & lt)] = (uint16_t)(slotB | (finalB ? 0x8000u : 0u));
                    wcount += __popc(ballB);
                }
            }
        }
        if (FAST) {
            // ---- phase B': the warp's hits, one per lane
            __syncwarp();
            for (uint32_t e = lane; e < wcount; e += 32) {
                const uint32_t ent = S.hits[w_lo + e];
                if (ent & 0x8000u) continue;
                const uint32_t slot = ent;
                const float mz = S.term[slot];
                uint32_t idx = __float_as_uint(S.inten[slot]);
                const float ph = __fmul_rn(mz, thi), qh = __fmul_rn(ph, 1.0f / 1000000.0f);
                const float hi = __fadd_rn(mz, __fmaf_rn(__fmaf_rn(-qh, 1000000.0f, ph), 1.0f / 1000000.0f, qh));
                // spectrum.rs:146-157: max_int starts at 0.0, `>=` keeps the last of equal maxima; a window of negative intensities matches nothing
                int best = -1;
                float max_int = 0.0f;
                float m;
                do {
                    const float it = pi[idx];
                    if (it >= max_int) { max_int = it; best = (int)idx; }
                    m = pm[++idx];
                } while (m <= hi);
                if (best >= 0) {
                    const float peak_mass = pm[best];
                    // scoring.rs:719-720: peak_intensity * (mz - peak_mass).abs() * 2E6 / (mz + peak_mass)
                    S.term[slot] = __fdiv_rn(__fmul_rn(__fmul_rn(max_int, fabsf(__fsub_rn(mz, peak_mass))), 2E6f), __fadd_rn(mz, peak_mass));
                    S.inten[slot] = max_int;
                } else {
                    atomicAnd(&S.mask[slot >> 5], ~(1u << (slot & 31)));   // not a match after all
                }
            }
        }
        __syncthreads();
        PH(4);
        if (SPLIT) {
            // ---- emit: the tile's hits go to the arena in task order. Position = hits of earlier tiles + set bits below the slot.
            const uint32_t nwords = (tn + 31) >> 5;
            const uint32_t mw = lane < nwords ? S.mask[lane] : 0u;   // every warp scans the (<= 32) words of the tile
            uint32_t incl = (uint32_t)__popc(mw);
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= (uint32_t)o) incl += v;
            }
            const uint32_t pre = incl - (uint32_t)__popc(mw), tile_total = __shfl_sync(0xffffffffu, incl, 31);
            // four threads per 32-slot word, eight slots each
            const uint32_t word = tid >> 2, q8 = (tid & 3) * 8;
            const uint32_t wm = word < nwords ? S.mask[word] : 0u;
            const uint32_t p = __shfl_sync(0xffffffffu, pre, word & 31);
            uint32_t m8 = (wm >> q8) & 0xFFu;
            const bool room = S.hit_room != 0;
            while (m8) {
                const uint32_t bit = q8 + (uint32_t)__ffs(m8) - 1;
                m8 &= m8 - 1;
                const uint32_t slot = (word << 5) + bit;
                const CandHdr hh = S.hdr[S.cand[slot]];
                const uint32_t f = t0 + slot - hh.base;
                const uint32_t ki = hh.nfc == 1 ? f : (hh.nfc == 2 ? f >> 1 : f / hh.nfc);
                if (room) {
                    const unsigned long long g = S.hit_base + hits_before + p + (uint32_t)__popc(wm & ((1u << bit) - 1u));
                    so.hit_k[g] = (uint16_t)kind_index(ki, hh.nions);
                    so.hit_i[g] = S.inten[slot];
                    so.hit_t[g] = S.term[slot];
                }
            }
            if (tid < ncand && total) {   // hits of candidate tid in this tile
                const uint32_t a = max(base, t0), b = min(base + total, t0 + tn);
                if (a < b) {
                    const uint32_t sa = a - t0, se = b - t0 - 1;
                    for (uint32_t w = sa >> 5; w <= se >> 5; w++) {
                        uint32_t m = S.mask[w];
                        if (w == sa >> 5) m &= 0xffffffffu << (sa & 31);
                        if (w == se >> 5) m &= 0xffffffffu >> (31 - (se & 31));
                        hcnt += (uint32_t)__popc(m);
                    }
                }
            }
            hits_before += tile_total;
            continue;
        }
        // ---- fold: thread c walks the set bits of candidate c's slice of the tile in ascending task order
        if (tid < ncand && total) {
            const uint32_t a = max(base, t0), b = min(base + total, t0 + tn);
            if (a < b) {
                const uint32_t sa = a - t0, se = b - t0 - 1;   // first / last slot (inclusive)
                for (uint32_t w = sa >> 5; w <= se >> 5; w++) {
                    uint32_t m = S.mask[w];
                    if (w == sa >> 5) m &= 0xffffffffu << (sa & 31);
                    if (w == se >> 5) m &= 0xffffffffu >> (31 - (se & 31));
                    while (m) {
                        const uint32_t slot = (w << 5) + (uint32_t)__ffs(m) - 1;
                        m &= m - 1;
                        const uint32_t f = t0 + slot - base;
                        uint32_t ki;
                        switch (nfc) {
                            case 1: ki = f; break;
                            case 2: ki = f >> 1; break;
                            case 3: ki = f / 3; break;
                            default: ki = f / nfc; break;
                        }
                        uint32_t kind_i = ki >= nions;   // two ion kinds (b/y) in practice: one compare; more kinds finish in the loop
                        uint32_t idx = ki - (kind_i ? nions : 0);
                        while (idx >= nions) { idx -= nions; kind_i++; }
                        const float it = S.inten[slot];
                        ppm = __fadd_rn(ppm, S.term[slot]);
                        if ((db.nterm_mask >> kind_i) & 1) { mb++; sb = __fadd_rn(sb, it); brun.matched(idx); }
                        else { my++; sy = __fadd_rn(sy, it); yrun.matched(idx); }
                    }
                }
            }
        }
    }
    if (SPLIT) {   // candidate headers: hits of candidate c start where the hits of candidates 0..c-1 end (task order)
        uint32_t inc2 = hcnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, inc2, o);
            if (lane >= (uint32_t)o) inc2 += v;
        }
        __syncthreads();   // S.scan is free again; every thread is done with the tile arrays
        if (lane == 31) S.scan[warp] = inc2;
        __syncthreads();
        uint32_t h0 = inc2 - hcnt;
#pragma unroll
        for (uint32_t w = 0; w < nwarps; w++) if (w < warp) h0 += S.scan[w];
        if (tid < ncand) {   // the candidate's fields are read back from shared memory: kept in registers, they spilled across the tile loop
            const CandHdr h = S.hdr[tid];
            CandOut co;
            co.key = cur[tid]; co.h0 = h0; co.hcnt = hcnt; co.nions = h.nions; co.nfc = h.nfc; co.plen = (uint8_t)(h.nions + 1); co.pad = 0;
            so.cand[(size_t)spec * sc.kparam + tid] = co;
        }
        return;
    }
    if (tid < ncand) {
        ScoreRec r;
        r.peptide = key_peptide(key); r.charge = key_charge(key); r.iso = key_iso(key);
        r.matched_b = mb & 0xFFFF; r.matched_y = my & 0xFFFF; r.summed_b = sb; r.summed_y = sy;
        r.longest_b = brun.longest; r.longest_y = yrun.longest;
        r.hyperscore = hyperscore_of(sc, r.matched_b, r.matched_y, sb, sy);                  // scoring.rs:756
        r.ppm_difference = __fdiv_rn(ppm, __fadd_rn(sb, sy));                                // scoring.rs:759
        r.valid = ((r.matched_b + r.matched_y) & 0xFFFF) >= sc.min_matched_peaks;            // scoring.rs:491
        r.plen = L;
        recs[tid] = r;
        S.hkey[tid] = r.valid ? r.hyperscore : -INFINITY;   // sort key: valid scores are finite (non-finite -> 255.0), so -inf never outranks one
    }
}

// Fragments of one reported PSM (scoring.rs:738-751), written by one warp in the reference's order (kind, ion index, charge) to
// out[0 .. matched_b + matched_y). Same lookups as score_candidate_warp on the same spectrum state.
__device__ SB_RARE void annotate_candidate_warp(const DbView& db, const ScorerView& sc, uint32_t pep, uint32_t charge, const SpecView& sp,
                                                        FragmentOut* out, uint32_t cap_left) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t L = __ldg(db.pep_len + pep);
    const uint32_t nions = L - 1;
    const uint32_t nfc = max_fragment_charge(sc.max_fragment_charge_opt, charge) - 1;
    const float* ions = db.ions + __ldg(db.ion_off + pep);
    const uint32_t total = nions * nfc * db.n_kinds;
    uint32_t written = 0;
    for (uint32_t base = 0; base < total; base += 32) {
        const uint32_t f = base + lane;
        int pk = -1;
        float mz = 0.f;
        uint32_t idx = 0, kind_i = 0, fc = 1;
        if (f < total) {
            const uint32_t ki = f / nfc;
            fc = f - ki * nfc + 1;
            idx = ki;
            while (idx >= nions) { idx -= nions; kind_i++; }
            mz = __fdiv_rn(__ldg(ions + ki), (float)fc);
            pk = sp.use_lut ? select_most_intense_peak_lut(sp.masses, sp.intens, sp.np, mz, sc.fragment_tol, sp.lp, sp.lut)
                            : select_most_intense_peak(sp.masses, sp.intens, sp.np, mz, sc.fragment_tol);
        }
        const uint32_t ball = __ballot_sync(0xffffffffu, pk >= 0);
        if (pk >= 0) {
            const uint32_t pos = written + __popc(ball & ((1u << lane) - 1));
            if (pos < cap_left) {
                const bool is_n = (db.nterm_mask >> kind_i) & 1;
                FragmentOut o;
                o.kind = db.kinds[kind_i];
                o.charge = (int32_t)fc;
                o.ordinal = is_n ? (int32_t)idx + 1 : (int32_t)(L == 0 ? 0 : L - 1) - (int32_t)idx;   // scoring.rs:739-744
                o.intensity = sp.intens[pk];
                o.mz_calculated = __fadd_rn(mz, PROTON);            // scoring.rs:723
                o.mz_experimental = __fadd_rn(sp.masses[pk], PROTON);  // scoring.rs:722
                out[pos] = o;
            }
        }
        written += __popc(ball);
    }
}

// Validates that the (possibly peak-depleted) spectrum is ascending, positive and NaN-free and builds the bucket LUT; otherwise the
// exact binary-search emulation is used for this spectrum.
__device__ __forceinline__ bool spectrum_lut_setup(const float* masses /*masses[np] == +inf*/, uint32_t np, uint16_t* lut, LutParams& lp) {
    bool bad = np == 0 || np >= 65536;
    for (uint32_t i = threadIdx.x; i < np; i += SCORE_THREADS) {
        const float m = masses[i];
        bad |= !(m > 0.0f) || (i > 0 && !(m >= masses[i - 1]));
    }
    if (__syncthreads_or(bad)) return false;
    lp = lut_params(masses[0], masses[np - 1], SPEC_LUT_CELLS);
    lut_build_walk<SCORE_THREADS>(masses, np, lp, lut, threadIdx.x, SPEC_LUT_CELLS);   // masses verified ascending above; masses[np] == +inf (k_score)
    __syncthreads();
    return true;
}

// One CTA per spectrum. SPLIT: matching only (see SplitOut); the caller guarantees no chimera, no annotation, quick_mode 0, no debug dump.
template <bool SPLIT>
__global__ void __launch_bounds__(SCORE_THREADS, SPLIT ? SCORE_MIN_CTAS_SPLIT : SCORE_MIN_CTAS) k_score(DbView db, ScorerView sc, BatchView b, FeatureOut* features, uint32_t* counts, uint32_t pmax,
                                                         uint64_t* dbg_keys /*nullable: initial_hits dump*/, uint32_t* dbg_meta, FragmentOut* frag_out /*nullable*/,
                                                         unsigned long long frag_cap, uint32_t quick_mode /*0 score, 1 keep all prelim, 2 low-memory*/,
                                                         uint8_t* keep /*quick_score: one byte per peptide*/, SplitOut so) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    // dynamic layout: masses_raw[pmax+4] intens_raw[pmax+4] cur[lcap] tot[lcap] recs[kparam] order[kparam] mark[pmax]   (pmax % 4 == 0)
    float* masses_raw = reinterpret_cast<float*>(smem_raw);
    float* intens_raw = masses_raw + pmax + 4;
    uint64_t* cur = reinterpret_cast<uint64_t*>(intens_raw + pmax + 4);
    uint64_t* tot = cur + sc.lcap;
    ScoreRec* recs = reinterpret_cast<ScoreRec*>(tot + sc.lcap);
    uint32_t* order = reinterpret_cast<uint32_t*>(recs + sc.kparam);
    uint8_t* mark = reinterpret_cast<uint8_t*>(order + sc.kparam);
    __shared__ __align__(16) ScoreTile S;   // static: headers, sort keys, spectrum LUT and the task tile of score_candidates_flat
    uint16_t* const lut = S.lut;
    __shared__ uint32_t s_ntot, s_ncand, s_np, s_nvalid;
    __shared__ unsigned long long s_matched_peaks, s_scored;
    __shared__ float s_tic;

    const uint32_t s = b.order ? b.order[blockIdx.x] : blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = SCORE_THREADS / 32;
    PH_START();
    const uint32_t p0 = b.peak_off[s];
    uint32_t np = b.peak_off[s + 1] - p0;
    // Stage the spectrum's peaks with the bulk-async copy engine (TMA 1-D): two cp.async.bulk copies complete on an mbarrier while the
    // prologue below folds the preliminary hits. Copies start at the 16-byte boundary below the first peak (`head` floats of slack).
    __shared__ __align__(8) uint64_t s_bar;
    const uint32_t a0 = p0 & ~3u, head = p0 - a0;
    const uint32_t bytes = ((head + np) * 4 + 15) & ~15u;
    float* masses = masses_raw + head;
    float* intens = intens_raw + head;
    if (tid == 0) {   // one thread initialises the barrier and issues both copies; everyone else first touches s_bar after the prologue's barrier
        mbar_init(&s_bar, 1);
        if (np) {
            mbar_arrive_expect_tx(&s_bar, 2 * bytes);
            bulk_copy_g2s(masses_raw, b.masses + a0, bytes, &s_bar);
            bulk_copy_g2s(intens_raw, b.intens + a0, bytes, &s_bar);
        }
    }

    const QueryDesc* qd = b.queries + (size_t)s * sc.qmax;
    const QueryHits* qh = b.hits + (size_t)s * sc.qmax;
    const uint64_t* qk = b.hit_keys + (size_t)s * sc.qmax * sc.kparam;
    const bool iso_fold = sc.min_iso != sc.max_iso;
    const bool single = !iso_fold && (sc.qmax == 1 || qd[1].mode == 0) && qd[0].mode != 0;
    if (single) {
        // one query, nothing to fold: trim_hits on a list of <= k entries is the identity (scoring.rs:460 after :380). Parallel copy,
        // then an order-preserving filter of PreScore::default() entries (scoring.rs:489).
        const QueryHits h = qh[0];
        const uint32_t n = h.n ? h.n : min(h.default_run, sc.kparam);
        for (uint32_t i = tid; i < n; i += SCORE_THREADS) tot[i] = h.n ? qk[i] : PRESCORE_DEFAULT;
        __syncthreads();
        if (warp == 0) {
            uint32_t w = 0;
            for (uint32_t base = 0; base < n; base += 32) {
                const uint32_t i = base + lane;
                const uint64_t k = i < n ? tot[i] : PRESCORE_DEFAULT;
                const bool keep = i < n && key_peptide(k) != 0xFFFFFFFFu;
                const uint32_t ball = __ballot_sync(0xffffffffu, keep);
                if (keep) cur[w + __popc(ball & ((1u << lane) - 1))] = k;
                w += __popc(ball);
            }
            if (lane == 0) { s_ntot = n; s_ncand = w; s_matched_peaks = h.matched_peaks; s_scored = h.scored_candidates; s_np = np; s_tic = b.tic[s]; }
        }
    } else if (tid == 0) {
        // ---- fold the per-query hits: matched_peaks (isotope fold, scoring.rs:384-416) then initial_hits (charge fold, :418-462)
        unsigned long long mp = 0, scd = 0;
        uint32_t ntot = 0;
        uint32_t nq = 0;
        while (nq < sc.qmax && qd[nq].mode != 0) nq++;
        const uint32_t nch = sc.n_iso ? nq / sc.n_iso : 0;
        for (uint32_t ci = 0; ci < nch; ci++) {
            uint32_t ncur = 0;
            for (uint32_t ii = 0; ii < sc.n_iso; ii++) {
                const uint32_t qi = ci * sc.n_iso + ii;
                mp += qh[qi].matched_peaks;
                scd += qh[qi].scored_candidates;
                ncur = append_hits(cur, ncur, sc.lcap, qh[qi], qk + (size_t)qi * sc.kparam, sc.kparam);
            }
            if (iso_fold) {  // trim_hits on the concatenation (scoring.rs:405)
                const uint32_t k = min(ncur, sc.kparam);
                bounded_min_heapify_seq(cur, ncur, k);
                ncur = k;
            }
            for (uint32_t i = 0; i < ncur && ntot < sc.lcap; i++) tot[ntot++] = cur[i];
        }
        {  // final trim_hits (scoring.rs:460)
            const uint32_t k = min(ntot, sc.kparam);
            bounded_min_heapify_seq(tot, ntot, k);
            ntot = k;
        }
        s_ntot = ntot;
        s_matched_peaks = mp;
        s_scored = scd;
        // build_features filter: peptide != PeptideIx::default() (scoring.rs:489), order preserved
        uint32_t nc = 0;
        for (uint32_t i = 0; i < ntot; i++)
            if (key_peptide(tot[i]) != 0xFFFFFFFFu) cur[nc++] = tot[i];
        s_ncand = nc;
        s_np = np;
        s_tic = b.tic[s];
    }
    __syncthreads();
    PH(0);
    if (dbg_keys != nullptr) {  // white-box dump of initial_hits
        for (uint32_t i = tid; i < s_ntot; i += SCORE_THREADS) dbg_keys[(size_t)s * sc.kparam + i] = tot[i];
        if (tid == 0) { dbg_meta[s * 4 + 0] = s_ntot; dbg_meta[s * 4 + 1] = (uint32_t)s_matched_peaks; dbg_meta[s * 4 + 2] = (uint32_t)s_scored; }
    }
    if (np) mbar_wait(&s_bar, 0);   // peaks have landed in shared memory
    PH(1);
    if (tid == 0) masses[np] = INFINITY;   // sentinel behind the last peak (slack of the staging buffer): ends the LUT walk and the peak scans
    const uint32_t ncand = s_ncand;
    if (SPLIT && tid == 0) {
        SpecMeta m;
        m.hit_base = 0; m.matched_peaks = s_matched_peaks; m.scored = s_scored; m.ncand = ncand; m.pad = 0;
        so.meta[s] = m;
    }
    // quick_score accumulates into keep[] across chunks; a chunk whose work lists overflowed (the host re-runs it with exact sizes) has partial hit
    // sets and must not leave marks behind. Both counters are final after k_setup_queries.
    const bool lists_fit = b.counters[C_NLIST_NEED] <= b.nlist_cap && b.counters[C_WIDE] <= (unsigned long long)b.wide_cap;
    if (quick_mode != 0 && !lists_fit) return;
    if (quick_mode == 1) {   // Scorer::quick_score, prefilter_low_memory == false (scoring.rs:291-296): every preliminary peptide is kept
        for (uint32_t i = tid; i < ncand; i += SCORE_THREADS) keep[key_peptide(cur[i])] = 1;
        return;
    }
    const float mzp = __fsub_rn(b.prec_mz[s], PROTON);
    const double lambda = (double)s_matched_peaks / (double)s_scored;  // scoring.rs:499
    const uint32_t rounds = sc.chimera ? sc.report_psms : 1;
    const uint32_t per_round = sc.chimera ? 1 : sc.report_psms;
    uint32_t nout = 0;
    SpecView sv;
    sv.masses = masses; sv.intens = intens; sv.lut = lut;
    for (uint32_t round = 0; round < rounds && ncand; round++) {
        np = s_np;
        sv.np = np;
        sv.use_lut = spectrum_lut_setup(masses, np, lut, sv.lp);
        PH(2);
        if (tid == 0) s_nvalid = 0;
        if (sv.use_lut && sc.score_fast && sc.fragment_tol.kind == 0 && fast_tol_ok(sc.fragment_tol.lo) && fast_tol_ok(sc.fragment_tol.hi))
            score_candidates_flat<true, SPLIT>(db, sc, cur, ncand, sv, S, recs, so, s);
        else
            score_candidates_flat<false, SPLIT>(db, sc, cur, ncand, sv, S, recs, so, s);
        if (SPLIT) return;   // k_fold / k_features take it from here
        __syncthreads();
        PH(5);
        if (quick_mode == 2) {
            // Scorer::quick_score, low-memory branch (scoring.rs:270-290): bounded_min_heapify(score_vector, report_psms) compares Score
            // with its DERIVED PartialOrd whose first field is the peptide index (heap.rs uses < and >), so the kept set is the
            // report_psms entries with the largest PeptideIx among those reaching min_matched_peaks (entries of one peptide are
            // interchangeable for the keep[] marks).
            if (tid < ncand && recs[tid].valid) {
                const uint32_t pme = recs[tid].peptide;
                uint32_t pos = 0;
                for (uint32_t j = 0; j < ncand; j++) {
                    if (!recs[j].valid) continue;
                    const uint32_t pj = recs[j].peptide;
                    pos += (pj > pme) || (pj == pme && j < tid);
                }
                if (pos < sc.report_psms) keep[pme] = 1;
            }
            return;
        }
        // stable sort by hyperscore descending (scoring.rs:495) via rank counting
        uint32_t my_floats = 0;
        if (tid < ncand) {
            my_floats = 2 * recs[tid].plen + 2;
            if (recs[tid].valid) {
                const double h = S.hkey[tid];   // == hyperscore; entries below min_matched_peaks hold -inf and never count
                uint32_t pos = 0;
                for (uint32_t j = 0; j < ncand; j++) {
                    const double hj = S.hkey[j];
                    pos += (hj > h) || (hj == h && j < tid);
                }
                order[pos] = tid;
                atomicAdd(&s_nvalid, 1u);
            }
        }
        if (tid < ((ncand + 31) & ~31u)) {  // SURVEY.md §8d peptide-record term: 2L+2 floats per scored candidate
            for (int o = 16; o > 0; o >>= 1) my_floats += __shfl_down_sync(0xffffffffu, my_floats, o);
            if (lane == 0 && my_floats) atomicAdd(b.counters + C_PEPFLOATS, (unsigned long long)my_floats);
        }
        if (tid == 0) atomicAdd(b.counters + C_CANDS, (unsigned long long)ncand);
        __syncthreads();
        const uint32_t nvalid = s_nvalid;
        const uint32_t emit = min(per_round, nvalid);
        if (tid < emit) {
            const ScoreRec r = recs[order[tid]];
            const double next = tid + 1 < nvalid ? recs[order[tid + 1]].hyperscore : 0.0;
            const double best = recs[order[0]].hyperscore;
            const uint32_t k = (r.matched_b + r.matched_y) & 0xFFFF;
            const double log10_poisson = ((double)k * ref_ln(sc, lambda) - lambda - lnfact(sc, k)) / 2.302585092994045684;
            const float precursor_mass = __fmul_rn(mzp, (float)r.charge);
            const float iso = __fmul_rn((float)r.iso, NEUTRON);
            const float mono = db.pep_mono[r.peptide];
            // scoring.rs:530-531
            const float delta_mass = __fdiv_rn(__fmul_rn(__fsub_rn(__fsub_rn(precursor_mass, mono), iso), 2E6f), __fadd_rn(__fsub_rn(precursor_mass, iso), mono));
            const uint32_t plen = r.plen;
            const float sum = __fadd_rn(r.summed_b, r.summed_y);
            FeatureOut f;
            f.spectrum = b.spectrum_base + s; f.peptide_idx = r.peptide; f.peptide_len = plen;
            f.rank = sc.chimera ? round + 1 : tid + 1;
            f.label = (db.pep_flags[r.peptide] & 1) ? -1 : 1;
            f.expmass = precursor_mass; f.calcmass = mono; f.charge = r.charge;
            f.rt = b.rt ? b.rt[s] : 0.0f;
            f.ims = (b.ims && !isnan(b.ims[s])) ? b.ims[s] : 0.0f;
            f.delta_mass = delta_mass; f.isotope_error = iso; f.average_ppm = r.ppm_difference; f._pad0 = 0;
            f.hyperscore = r.hyperscore; f.delta_next = r.hyperscore - next; f.delta_best = best - r.hyperscore;
            f.matched_peaks = k; f.longest_b = r.longest_b; f.longest_y = r.longest_y;
            f.longest_y_pct = __fdiv_rn((float)r.longest_y, (float)plen);
            f.missed_cleavages = db.pep_missed[r.peptide];
            f.matched_intensity_pct = __fdiv_rn(__fmul_rn(100.0f, sum), s_tic);
            f.scored_candidates = (uint32_t)s_scored;
            f.ms2_intensity = sum;
            f.poisson = isfinite(log10_poisson) ? log10_poisson : -INFINITY;
            f.fragment_offset = 0; f.fragment_count = 0;
            features[(size_t)s * sc.report_psms + nout + tid] = f;
        }
        if (frag_out != nullptr && emit) {   // annotate_matches: Fragments of every PSM reported in this round (scoring.rs:738-751)
            __syncthreads();
            for (uint32_t e = warp; e < emit; e += nwarps) {
                const ScoreRec r = recs[order[e]];
                const uint32_t cnt = (r.matched_b + r.matched_y) & 0xFFFF;
                unsigned long long off = 0;
                if (lane == 0) off = atomicAdd(b.counters + C_FRAGS, (unsigned long long)cnt);
                off = __shfl_sync(0xffffffffu, off, 0);
                const uint32_t cap_left = off >= frag_cap ? 0u : (uint32_t)min((unsigned long long)cnt, frag_cap - off);
                annotate_candidate_warp(db, sc, r.peptide, r.charge, sv, frag_out + (off < frag_cap ? off : 0), cap_left);
                if (lane == 0) {
                    FeatureOut* fo = features + (size_t)s * sc.report_psms + nout + e;
                    fo->fragment_offset = (uint32_t)off;
                    fo->fragment_count = cnt;
                }
            }
        }
        nout += emit;
        if (!sc.chimera || emit == 0 || round + 1 == rounds) break;
        // ---- remove_matched_peaks (scoring.rs:598-644) for the PSM just accepted
        for (uint32_t i = tid; i < np; i += SCORE_THREADS) mark[i] = 0;
        __syncthreads();
        if (warp == 0) {
            const ScoreRec r = recs[order[0]];
            score_candidate_warp(db, sc, prescore_key(0, r.peptide, r.charge, r.iso), sv, nullptr, mark);
        }
        __syncthreads();
        // a peak is removed when its (mass, intensity) pair equals a marked one (Vec::contains on (f32,f32))
        for (uint32_t i = tid; i < np; i += SCORE_THREADS) {
            if (mark[i]) continue;
            const float m = masses[i], it = intens[i];
            bool rm = false;
            for (int j = (int)i - 1; j >= 0 && masses[j] == m && !rm; j--) rm = mark[j] == 1 && intens[j] == it;
            for (uint32_t j = i + 1; j < np && masses[j] == m && !rm; j++) rm = mark[j] == 1 && intens[j] == it;
            if (rm) mark[i] = 2;
        }
        __syncthreads();
        if (warp == 0) {
            uint32_t w = 0;
            for (uint32_t base = 0; base < np; base += 32) {
                const uint32_t i = base + lane;
                const bool keep = i < np && mark[i] == 0;
                const float m = i < np ? masses[i] : 0.f, it = i < np ? intens[i] : 0.f;
                const uint32_t ball = __ballot_sync(0xffffffffu, keep);
                __syncwarp();
                if (keep) {
                    const uint32_t d = w + __popc(ball & ((1u << lane) - 1));
                    masses[d] = m;
                    intens[d] = it;
                }
                w += __popc(ball);
                __syncwarp();
            }
            if (lane == 0) {
                float t = 0.0f;  // iter().sum::<f32>() (scoring.rs:643)
                for (uint32_t i = 0; i < w; i++) t = __fadd_rn(t, intens[i]);
                s_tic = t;
                s_np = w;
                masses[w] = INFINITY;   // sentinel follows the shrunken peak list
            }
        }
        __syncthreads();
    }
    PH(6);
    if (tid == 0) {
        counts[s] = nout;
        if (nout) atomicAdd(b.counters + C_PSMS, (unsigned long long)nout);
    }
}

// SPLIT, second kernel: one thread per (spectrum, candidate) folds the candidate's hits in the reference's order (score_candidate,
// scoring.rs:675-767: per matched fragment in (kind, ion index, charge) order — the arena order) and writes the ScoreRec.
__global__ void __launch_bounds__(128) k_fold(DbView db, ScorerView sc, SplitOut so, uint32_t n) {
    __shared__ unsigned long long s_floats[4];
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t s = (uint32_t)(i / sc.kparam), c = (uint32_t)(i - (uint64_t)s * sc.kparam);
    const bool me = s < n && c < so.meta[s].ncand;
    // SURVEY.md §8d peptide-record term: 2L+2 floats per scored candidate (one atomic per CTA)
    unsigned long long a_floats = me ? 2ull * so.cand[(size_t)s * sc.kparam + c].plen + 2ull : 0ull;
    for (int o = 16; o > 0; o >>= 1) a_floats += __shfl_down_sync(0xffffffffu, a_floats, o);
    if ((threadIdx.x & 31) == 0) s_floats[threadIdx.x >> 5] = a_floats;
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned long long t = s_floats[0] + s_floats[1] + s_floats[2] + s_floats[3];
        if (t) atomicAdd(so.counters + C_PEPFLOATS, t);
    }
    if (!me) return;
    const SpecMeta m = so.meta[s];
    const CandOut co = so.cand[(size_t)s * sc.kparam + c];
    uint32_t mb = 0, my = 0;
    float sb = 0.f, sy = 0.f, ppm = 0.f;
    Run brun = {0, 0, 0, 0}, yrun = {0, 0, 0, 0};
    const unsigned long long h0 = m.hit_base + co.h0;
    for (uint32_t k = 0; k < co.hcnt; k++) {
        const uint32_t x = so.hit_k[h0 + k];
        const float it = so.hit_i[h0 + k];
        ppm = __fadd_rn(ppm, so.hit_t[h0 + k]);
        const uint32_t kind_i = x >> 13, idx = x & 0x1FFFu;
        if ((db.nterm_mask >> kind_i) & 1) { mb++; sb = __fadd_rn(sb, it); brun.matched(idx); }
        else { my++; sy = __fadd_rn(sy, it); yrun.matched(idx); }
    }
    ScoreRec r;
    r.peptide = key_peptide(co.key); r.charge = key_charge(co.key); r.iso = key_iso(co.key);
    r.matched_b = mb & 0xFFFF; r.matched_y = my & 0xFFFF; r.summed_b = sb; r.summed_y = sy;
    r.longest_b = brun.longest; r.longest_y = yrun.longest;
    r.hyperscore = hyperscore_of(sc, r.matched_b, r.matched_y, sb, sy);                  // scoring.rs:756
    r.ppm_difference = __fdiv_rn(ppm, __fadd_rn(sb, sy));                                // scoring.rs:759
    r.valid = ((r.matched_b + r.matched_y) & 0xFFFF) >= sc.min_matched_peaks;            // scoring.rs:491
    r.plen = co.plen;
    so.recs[(size_t)s * sc.kparam + c] = r;
    so.hkey[(size_t)s * sc.kparam + c] = r.valid ? f64_sort_key(r.hyperscore) : 0ull;   // valid scores are finite, so their keys are > 0
}

// SPLIT, third kernel: the sort of build_features (scoring.rs:495: stable, by hyperscore descending) as a rank count over integer sort keys — one
// thread per (spectrum, candidate), nothing but the count: a candidate among the report_psms best leaves its index in the spectrum's rank slot
// (slots are preset to "empty"). Everything a row needs beyond that is computed by k_rows, one thread per (spectrum, rank): done here by the one
// ranked lane of a warp, those ~1000 instructions (f64 ln, 128-byte row) would cost every warp, and so would the best / next-best bookkeeping.
constexpr uint32_t RANK_EMPTY = 0xFFFFFFFFu;
__global__ void __launch_bounds__(128) k_features(ScorerView sc, uint32_t n, SplitOut so, uint32_t* rank_slots) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t s = (uint32_t)(i / sc.kparam), c = (uint32_t)(i - (uint64_t)s * sc.kparam);
    if (s >= n) return;
    const uint32_t ncand = so.meta[s].ncand;
    if (c >= ncand) return;
    const unsigned long long* hk = so.hkey + (size_t)s * sc.kparam;
    const unsigned long long h = hk[c];
    if (h == 0) return;   // below min_matched_peaks: never ranked
    uint32_t pos = 0;
    for (uint32_t j = 0; j < ncand; j++) {
        const unsigned long long hj = hk[j];
        pos += (hj > h) || (hj == h && j < c);
    }
    if (pos < sc.report_psms) rank_slots[(size_t)s * sc.report_psms + pos] = c;
}

// SPLIT, fourth kernel: the Feature rows (scoring.rs:499-593), one thread per (spectrum, rank). delta_next needs the hyperscore ranked right behind
// the row's candidate (0.0 when there is none), delta_best the best one: both are re-derived here from the sort keys.
__global__ void __launch_bounds__(128) k_rows(DbView db, ScorerView sc, BatchView b, SplitOut so, const uint32_t* rank_slots, uint32_t* counts, FeatureOut* features) {
    __shared__ unsigned long long s_acc[2][4];
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t s = (uint32_t)(i / sc.report_psms), pos = (uint32_t)(i - (uint64_t)s * sc.report_psms);
    unsigned long long a_cands = 0, a_psms = 0;
    if (s < b.n) {
        const SpecMeta m = so.meta[s];
        const uint32_t cand = rank_slots[(size_t)s * sc.report_psms + pos];
        if (pos == 0) {   // ranks are dense from 0: the count is the number of filled slots
            uint32_t cnt = 0;
            while (cnt < sc.report_psms && rank_slots[(size_t)s * sc.report_psms + cnt] != RANK_EMPTY) cnt++;
            counts[s] = cnt;
            a_cands = m.ncand; a_psms = cnt;
        }
        if (cand != RANK_EMPTY) {
            const unsigned long long* hk = so.hkey + (size_t)s * sc.kparam;
            const unsigned long long h = hk[cand];
            unsigned long long knext = 0, kbest = 0;
            for (uint32_t j = 0; j < m.ncand; j++) {
                const unsigned long long hj = hk[j];
                kbest = max(kbest, hj);
                const bool higher = (hj > h) || (hj == h && j < cand);
                if (!higher && j != cand) knext = max(knext, hj);   // ranked behind this candidate
            }
            const double next = knext != 0 ? f64_from_sort_key(knext) : 0.0, best = f64_from_sort_key(kbest);   // scoring.rs:512-516
            const ScoreRec r = so.recs[(size_t)s * sc.kparam + cand];
            const double lambda = (double)m.matched_peaks / (double)m.scored;  // scoring.rs:499
            const float mzp = __fsub_rn(b.prec_mz[s], PROTON);
            const uint32_t k = (r.matched_b + r.matched_y) & 0xFFFF;
            const double log10_poisson = ((double)k * ref_ln(sc, lambda) - lambda - lnfact(sc, k)) / 2.302585092994045684;
            const float precursor_mass = __fmul_rn(mzp, (float)r.charge);
            const float iso = __fmul_rn((float)r.iso, NEUTRON);
            const float mono = db.pep_mono[r.peptide];
            // scoring.rs:530-531
            const float delta_mass = __fdiv_rn(__fmul_rn(__fsub_rn(__fsub_rn(precursor_mass, mono), iso), 2E6f), __fadd_rn(__fsub_rn(precursor_mass, iso), mono));
            const uint32_t plen = r.plen;
            const float sum = __fadd_rn(r.summed_b, r.summed_y);
            FeatureOut f;
            f.spectrum = b.spectrum_base + s; f.peptide_idx = r.peptide; f.peptide_len = plen;
            f.rank = pos + 1;
            f.label = (db.pep_flags[r.peptide] & 1) ? -1 : 1;
            f.expmass = precursor_mass; f.calcmass = mono; f.charge = r.charge;
            f.rt = b.rt ? b.rt[s] : 0.0f;
            f.ims = (b.ims && !isnan(b.ims[s])) ? b.ims[s] : 0.0f;
            f.delta_mass = delta_mass; f.isotope_error = iso; f.average_ppm = r.ppm_difference; f._pad0 = 0;
            f.hyperscore = r.hyperscore; f.delta_next = r.hyperscore - next; f.delta_best = best - r.hyperscore;
            f.matched_peaks = k; f.longest_b = r.longest_b; f.longest_y = r.longest_y;
            f.longest_y_pct = __fdiv_rn((float)r.longest_y, (float)plen);
            f.missed_cleavages = db.pep_missed[r.peptide];
            f.matched_intensity_pct = __fdiv_rn(__fmul_rn(100.0f, sum), b.tic[s]);
            f.scored_candidates = (uint32_t)m.scored;
            f.ms2_intensity = sum;
            f.poisson = isfinite(log10_poisson) ? log10_poisson : -INFINITY;
            f.fragment_offset = 0; f.fragment_count = 0;
            features[(size_t)s * sc.report_psms + pos] = f;
        }
    }
    // chunk-wide sums: one atomic per CTA and counter
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int o = 16; o > 0; o >>= 1) {
        a_cands += __shfl_down_sync(0xffffffffu, a_cands, o);
        a_psms += __shfl_down_sync(0xffffffffu, a_psms, o);
    }
    if (lane == 0) { s_acc[0][warp] = a_cands; s_acc[1][warp] = a_psms; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (uint32_t w = 1; w < (blockDim.x >> 5); w++) { a_cands += s_acc[0][w]; a_psms += s_acc[1][w]; }
        if (a_cands) atomicAdd(b.counters + C_CANDS, a_cands);
        if (a_psms) atomicAdd(b.counters + C_PSMS, a_psms);
    }
}

// ------------------------------------------------------------------------------------------- spectrum preprocessing (SURVEY §8 row f2)
// SpectrumProcessor::process for centroided MS2 spectra (spectrum.rs:279-412): deisotope (spectrum.rs:179-227), sort by intensity,
// drop isotope-envelope members, MH+ -> M with the assigned charge, keep the top N, sort by mass, total ion current.
// One warp per spectrum: the deisotoping pass is a sequential recurrence (lane 0), the two sorts are warp bitonic sorts in smem.
struct ProcParams { uint32_t take_top_n; uint32_t deisotope; float min_deisotope_mz; };

__device__ __forceinline__ void warp_bitonic(uint64_t* keys, uint32_t* vals, uint32_t n2) {
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t k = 2; k <= n2; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = lane; i < n2; i += 32) {
                const uint32_t l = i ^ j;
                if (l > i) {
                    const bool asc = (i & k) == 0;
                    const uint64_t a = keys[i], c = keys[l];
                    if ((a > c) == asc) { keys[i] = c; keys[l] = a; const uint32_t t = vals[i]; vals[i] = vals[l]; vals[l] = t; }
                }
            }
            __syncwarp();
        }
    }
}
__device__ __forceinline__ uint32_t f32_ukey(float x) { return (uint32_t)f32_key(x) ^ 0x80000000u; }   // unsigned order == total_cmp order

__global__ void __launch_bounds__(32) k_process_ms2(ProcParams pp, uint32_t n, const uint32_t* peak_off, const float* mz_in, const float* int_in,
                                                      const uint8_t* prec_charge, uint32_t pmax, uint32_t p2max, float* out_mass, float* out_int,
                                                      uint32_t* out_count, float* out_tic) {
    extern __shared__ __align__(16) unsigned char praw[];
    uint64_t* keys = reinterpret_cast<uint64_t*>(praw);          // [p2max]
    uint32_t* vals = reinterpret_cast<uint32_t*>(keys + p2max);   // [p2max]
    float* mz = reinterpret_cast<float*>(vals + p2max);           // [pmax]
    float* it0 = mz + pmax;                                       // original intensities
    float* acc = it0 + pmax;                                      // Deisotoped::intensity
    float* omass = acc + pmax;                                    // kept peaks (mass, intensity), <= take_top_n of them
    float* oint = omass + pmax;
    uint8_t* chg = reinterpret_cast<uint8_t*>(oint + pmax);       // Deisotoped::charge (0 = None)
    uint8_t* env = chg + pmax;                                    // Deisotoped::envelope.is_some()
    const uint32_t s = blockIdx.x, lane = threadIdx.x;
    if (s >= n) return;
    const uint32_t p0 = peak_off[s], np = peak_off[s + 1] - p0;
    for (uint32_t i = lane; i < np; i += 32) { mz[i] = mz_in[p0 + i]; it0[i] = int_in[p0 + i]; acc[i] = it0[i]; chg[i] = 0; env[i] = 0; }
    __syncwarp();
    uint32_t nkeep = 0;
    if (pp.deisotope) {
        if (lane == 0 && np > 0) {   // deisotope(mz, int, charge, 10.0, min_deisotope_mz), spectrum.rs:179-227
            const uint32_t max_charge = prec_charge[s] ? prec_charge[s] : 3;   // spectrum.rs:289-293
            const float ppm = 10.0f;
            for (uint32_t i = np; i-- > 0;) {
                uint32_t j = i == 0 ? 0 : i - 1;
                const float tol = __fdiv_rn(__fmul_rn(ppm, mz[i]), 1000000.0f);   // ppm_to_delta_mass(mz[i], ppm)
                while (__fsub_rn(mz[i], mz[j]) <= __fadd_rn(NEUTRON, tol) && mz[j] >= pp.min_deisotope_mz) {
                    const float delta = __fsub_rn(mz[i], mz[j]);
                    for (uint32_t c = 1; c <= max_charge; c++) {
                        const float iso = __fdiv_rn(NEUTRON, (float)c);
                        if (fabsf(__fsub_rn(delta, iso)) <= tol && it0[i] < it0[j]) {
                            if (chg[i] != 0 && chg[i] != c) continue;   // already part of an envelope with another charge
                            acc[j] = __fadd_rn(acc[j], acc[i]);
                            chg[j] = (uint8_t)c;
                            chg[i] = (uint8_t)c;
                            env[i] = 1;
                        }
                    }
                    j = j == 0 ? 0 : j - 1;
                    if (j == 0) break;
                }
            }
        }
        __syncwarp();
        // sort by (intensity descending, mz ascending)  spectrum.rs:303-307
        uint32_t n2 = 1;
        while (n2 < np) n2 <<= 1;
        for (uint32_t i = lane; i < n2; i += 32) {
            if (i < np) { keys[i] = ((uint64_t)(~f32_ukey(acc[i])) << 32) | f32_ukey(mz[i]); vals[i] = i; }
            else { keys[i] = ~0ull; vals[i] = 0xFFFFFFFFu; }
        }
        __syncwarp();
        warp_bitonic(keys, vals, n2);
        // keep non-envelope peaks, MH+ -> M, first take_top_n  (spectrum.rs:309-321)
        for (uint32_t base = 0; base < np && nkeep < pp.take_top_n; base += 32) {
            const uint32_t i = base + lane;
            const uint32_t src = i < np ? vals[i] : 0xFFFFFFFFu;
            const bool keep = src != 0xFFFFFFFFu && env[src] == 0;
            const uint32_t ball = __ballot_sync(0xffffffffu, keep);
            const uint32_t pos = nkeep + __popc(ball & ((1u << lane) - 1));
            if (keep && pos < pp.take_top_n) {
                omass[pos] = __fmul_rn(__fsub_rn(mz[src], PROTON), (float)(chg[src] ? chg[src] : 1));
                oint[pos] = acc[src];
            }
            nkeep = min(nkeep + (uint32_t)__popc(ball), pp.take_top_n);
        }
        __syncwarp();
    } else {
        // (mz - PROTON) * 1.0, bounded_min_heapify(peaks, take_top_n) with Peak's Ord (intensity, then mass), truncate  spectrum.rs:323-334
        for (uint32_t i = lane; i < np; i += 32) { omass[i] = __fmul_rn(__fsub_rn(mz[i], PROTON), 1.0f); oint[i] = it0[i]; }
        __syncwarp();
        const uint32_t k = pp.take_top_n;
        if (np > k) {
            if (lane == 0) {
                auto pkey = [&](uint32_t i) -> uint64_t { return ((uint64_t)f32_ukey(oint[i]) << 32) | f32_ukey(omass[i]); };
                for (uint32_t i = 0; i < np; i++) { keys[i] = pkey(i); vals[i] = i; }   // heap over (key, original index)
                auto sift = [&](uint32_t index) {
                    while (index * 2 + 1 < k) {
                        uint32_t sm = index, l = index * 2 + 1, r = index * 2 + 2;
                        if (keys[l] < keys[sm]) sm = l;
                        if (r < k && keys[r] < keys[sm]) sm = r;
                        if (sm == index) break;
                        const uint64_t tk = keys[sm]; keys[sm] = keys[index]; keys[index] = tk;
                        const uint32_t tv = vals[sm]; vals[sm] = vals[index]; vals[index] = tv;
                        index = sm;
                    }
                };
                for (uint32_t i = k / 2; i-- > 0;) sift(i);
                for (uint32_t i = k; i < np; i++) {
                    if (keys[i] > keys[0]) {
                        const uint64_t tk = keys[i]; keys[i] = keys[0]; keys[0] = tk;
                        const uint32_t tv = vals[i]; vals[i] = vals[0]; vals[0] = tv;
                        sift(0);
                    }
                }
                for (uint32_t i = 0; i < k; i++) { mz[i] = omass[vals[i]]; acc[i] = oint[vals[i]]; }   // heap order
                for (uint32_t i = 0; i < k; i++) { omass[i] = mz[i]; oint[i] = acc[i]; }
            }
            __syncwarp();
            nkeep = k;
        } else nkeep = np;
    }
    // stable sort by mass (spectrum.rs:393), then SoA + TIC (spectrum.rs:394-398)
    uint32_t m2 = 1;
    while (m2 < nkeep) m2 <<= 1;
    for (uint32_t i = lane; i < m2; i += 32) {
        if (i < nkeep) { keys[i] = ((uint64_t)f32_ukey(omass[i]) << 32) | i; vals[i] = i; }
        else { keys[i] = ~0ull; vals[i] = 0xFFFFFFFFu; }
    }
    __syncwarp();
    warp_bitonic(keys, vals, m2);
    for (uint32_t i = lane; i < nkeep; i += 32) { out_mass[p0 + i] = omass[vals[i]]; out_int[p0 + i] = oint[vals[i]]; }
    __syncwarp();
    if (lane == 0) {
        float t = 0.0f;
        for (uint32_t i = 0; i < nkeep; i++) t = __fadd_rn(t, oint[vals[i]]);
        out_tic[s] = t;
        out_count[s] = nkeep;
    }
}

// ------------------------------------------------------------------------------------------- TMT reporter ions (SURVEY §8 row f4)
// find_reporter_ions (tmt.rs:193-211): one thread per (spectrum, label); select_most_intense_peak with offset Some(-PROTON) (spectrum.rs:134-159).
__global__ void k_find_reporter_ions(uint32_t n, uint32_t n_labels, const uint32_t* peak_off, const float* masses, const float* intens, const float* labels,
                                     Tol tol, float* out) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= (uint64_t)n * n_labels) return;
    const uint32_t s = (uint32_t)(j / n_labels), l = (uint32_t)(j - (uint64_t)s * n_labels);
    const uint32_t p0 = peak_off[s], np = peak_off[s + 1] - p0;
    const float* m = masses + p0;
    const float* it = intens + p0;
    float lo, hi;
    tol_bounds(tol, labels[l], lo, hi);
    lo = __fadd_rn(lo, -PROTON);   // lo + offset.unwrap_or_default()
    hi = __fadd_rn(hi, -PROTON);
    const int klo = f32_key(lo), khi = f32_key(hi);
    uint32_t a, b2;
    binary_search_slice(np, [&](uint32_t k) { return f32_key(__ldg(m + k)) < klo; }, [&](uint32_t k) { return f32_key(__ldg(m + k)) <= khi; }, a, b2);
    int best = -1;
    float max_int = 0.0f;
    for (uint32_t idx = a; idx < b2; idx++) {
        const float mm = __ldg(m + idx);
        if (mm >= lo && mm <= hi) {
            const float v = __ldg(it + idx);
            if (v >= max_int) { max_int = v; best = (int)idx; }
        }
    }
    out[j] = best >= 0 ? __ldg(it + best) : 0.0f;
}

// ------------------------------------------------------------------------------------------- index construction
// IonSeries (ion_series.rs:36-85) for every kind of every peptide; one thread per peptide (sequential f32 running sum).
__global__ void k_build_ions(uint32_t n_pep, const uint32_t* seq_off, const uint8_t* seq, const float* mods, const float* nterm, const float* mono,
                             const uint32_t* ion_off, uint32_t n_kinds, DbView kinds_src, float* ions, const float* residue_mass) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pep) return;
    const float Cm = 12.0f, O = 15.994914f, H = 1.007825f, PRO = 1.0072764f, N = 14.003074f;
    const float NH3 = __fadd_rn(__fadd_rn(N, __fmul_rn(H, 2.0f)), PRO);
    const uint32_t o0 = seq_off[p], L = seq_off[p + 1] - o0;
    if (L == 0) return;
    const float nt = isnan(nterm[p]) ? 0.0f : nterm[p];
    const float m = mono[p];
    float* out = ions + ion_off[p];
    for (uint32_t k = 0; k < n_kinds; k++) {
        const uint32_t kind = kinds_src.kinds[k];
        float cum;
        switch (kind) {
            case 0: cum = __fsub_rn(nt, __fadd_rn(Cm, O)); break;
            case 1: cum = nt; break;
            case 2: cum = __fadd_rn(nt, NH3); break;
            case 3: cum = __fadd_rn(__fsub_rn(m, nt), __fadd_rn(__fadd_rn(__fsub_rn(__fadd_rn(Cm, O), NH3), N), H)); break;
            case 4: cum = __fsub_rn(m, nt); break;
            default: cum = __fsub_rn(__fsub_rn(m, nt), NH3); break;
        }
        for (uint32_t i = 0; i + 1 < L; i++) {
            const uint8_t r = seq[o0 + i];
            const float rm = __fadd_rn((r >= 'A' && r <= 'Z') ? residue_mass[r - 'A'] : 0.0f, mods[o0 + i]);
            cum = kind <= 2 ? __fadd_rn(cum, rm) : __fadd_rn(cum, -rm);
            out[k * (L - 1) + i] = cum;
        }
    }
}

// Fragment generation for the index (database.rs:272-297): keep ions with index > min_ion_index.
// Pass 0 (frag_off == nullptr -> counts[p]); pass 1 writes keys (total-order key of mz) and peptide ids.
__global__ void k_gen_fragments(uint32_t n_pep, const uint8_t* pep_len, const uint32_t* ion_off, const float* ions, uint32_t n_kinds, DbView kinds_src,
                                uint32_t min_ion_index, uint32_t* counts, const uint64_t* frag_off, uint32_t* out_key, uint32_t* out_pep) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pep) return;
    const uint32_t L = pep_len[p];
    if (L == 0) { if (counts) counts[p] = 0; return; }
    const float* src = ions + ion_off[p];
    uint64_t w = frag_off ? frag_off[p] : 0;
    uint32_t c = 0;
    for (uint32_t k = 0; k < n_kinds; k++) {
        const uint32_t kind = kinds_src.kinds[k];
        for (uint32_t i = 0; i + 1 < L; i++) {
            const bool keep = kind <= 2 ? (i + 1) > min_ion_index : ((L - 1) - i) > min_ion_index;
            if (!keep) continue;
            if (frag_off) {
                out_key[w] = (uint32_t)f32_key(src[k * (L - 1) + i]) ^ 0x80000000u;  // unsigned order == total_cmp order
                out_pep[w] = p;
                w++;
            }
            c++;
        }
    }
    if (counts) counts[p] = c;
}

// After the global sort by m/z: record bucket minima and form (bucket, peptide) 64-bit keys with the m/z as payload.
__global__ void k_bucket_keys(uint64_t n_frag, uint32_t bucket_shift, const uint32_t* key_sorted, const uint32_t* pep_sorted, uint64_t* key64,
                              uint32_t* mzbits, float* bucket_min) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_frag) return;
    const uint32_t u = key_sorted[i] ^ 0x80000000u;                 // back to the signed total-order key
    const uint32_t bits = u ^ (((uint32_t)((int)u >> 31)) >> 1);    // inverse of f32_key
    mzbits[i] = bits;
    const uint64_t bucket = i >> bucket_shift;
    key64[i] = (bucket << 32) | pep_sorted[i];
    if ((i & ((1ull << bucket_shift) - 1)) == 0) bucket_min[bucket] = __uint_as_float(bits);
}
// Search directories. page_grid[p][g] = #{entries of page p with PeptideIx < g << shift} (g = 0..grid_n), bucket_lut[c] = #{bucket_min < edge(c)}.
__global__ void k_build_page_grid(DbView db, uint32_t grid_shift, uint32_t grid_n, uint16_t* grid) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t total = (uint64_t)db.n_bucket * (grid_n + 1);
    if (j >= total) return;
    const uint32_t page = (uint32_t)(j / (grid_n + 1)), g = (uint32_t)(j - (uint64_t)page * (grid_n + 1));
    const uint64_t pbase = (uint64_t)page * db.bucket_size;
    const uint32_t pn = (uint32_t)(min(pbase + db.bucket_size, db.n_frag) - pbase);
    const uint64_t key64 = (uint64_t)g << grid_shift;
    uint32_t pos = pn;
    if (key64 <= 0xFFFFFFFFull) pos = page_lower_bound(db.frag + pbase, 0, pn, (uint32_t)key64);
    grid[j] = (uint16_t)pos;
}
// *bad |= the array is not ascending / positive / NaN-free (the pep LUT is only used for arrays the reference's binary search is well defined on)
__global__ void k_check_ascending(uint32_t n, const float* a, uint32_t* bad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = a[i];
    if (!(x > 0.0f) || !(x < 3.0e38f) || (i > 0 && !(x >= a[i - 1]))) *bad = 1u;
}
__global__ void k_build_pep_lut(DbView db, float base, float inv_w, uint32_t* lut) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c > PEP_LUT_CELLS) return;
    uint32_t lo = c == PEP_LUT_CELLS ? db.n_pep : 0;
    if (c > 0 && c < PEP_LUT_CELLS && inv_w > 0.0f) {
        const float e = base + (float)c * (1.0f / inv_w);
        uint32_t hi = db.n_pep;
        while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (db.pep_mono[m] < e) lo = m + 1; else hi = m; }
    }
    lut[c] = lo;
}
// ---- secondary (open-search) index: keys (block, m/z) of every fragment, block offsets, per-block m/z LUT
__global__ void k_wide_keys(uint64_t n_frag, const uint2* frag, uint32_t block, uint64_t* key64, uint32_t* pep) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_frag) return;
    const uint2 f = frag[i];
    key64[i] = ((uint64_t)(f.x / block) << 32) | (uint32_t)((uint32_t)f32_key(__uint_as_float(f.y)) ^ 0x80000000u);   // unsigned order == total_cmp order
    pep[i] = f.x;
}
__device__ __forceinline__ uint32_t mz_bits_of_key(uint64_t key) {
    const uint32_t u = (uint32_t)key ^ 0x80000000u;                    // back to the signed total_cmp key ...
    return u ^ (((uint32_t)((int)u >> 31)) >> 1);                       // ... and to the float's bit pattern (f32_key is an involution)
}
__global__ void k_wide_pack(uint64_t n_frag, const uint64_t* key64, const uint32_t* pep, uint2* out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_frag) return;
    out[i] = make_uint2(pep[i], mz_bits_of_key(key64[i]));
}
// the narrow copy: the same sorted keys as two parallel arrays, m/z and PeptideIx relative to its block
__global__ void k_narrow_pack(uint64_t n_frag, const uint64_t* key64, const uint32_t* pep, uint32_t block, float* mz, uint16_t* off) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_frag) return;
    const uint64_t k = key64[i];
    mz[i] = __uint_as_float(mz_bits_of_key(k));
    off[i] = (uint16_t)(pep[i] - (uint32_t)(k >> 32) * block);
}
__global__ void k_wide_block_offsets(uint64_t n_frag, const uint64_t* key64, uint32_t n_block, uint64_t* blk_off) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b > n_block) return;
    uint64_t lo = 0, hi = n_frag;
    const uint64_t want = (uint64_t)b << 32;
    while (lo < hi) { const uint64_t m = (lo + hi) >> 1; if (key64[m] < want) lo = m + 1; else hi = m; }
    blk_off[b] = lo;
}
// Sum of the precursor-window sizes (peptides inside Tolerance::bounds of the peptide's own mass) of `samples` peptides spread evenly over the
// index: the host sizes the blocks of the narrow-search copy by the average (sage_b200.cu: narrow_block_for).
__global__ void k_window_sample(DbView db, Tol ptol, uint32_t samples, unsigned long long* sum) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= samples || db.n_pep == 0) return;
    const uint32_t i = (uint32_t)((uint64_t)k * db.n_pep / samples);
    float lo, hi;
    tol_bounds(ptol, __ldg(db.pep_mono + i), lo, hi);
    const uint32_t a = pep_partition(db, lo, false), b = pep_partition(db, hi, true);
    atomicAdd(sum, (unsigned long long)(b > a ? b - a : 0u));
}
// rng[0] = min, rng[1] = max of the m/z bit patterns. Bit order is value order only for positive floats: an index holding m/z <= 0 yields a
// range the host treats as degenerate (set_mz_cells: no LUT, every search covers the whole block).
__global__ void k_frag_mz_range(uint64_t n_frag, const uint2* frag, uint32_t* rng) {
    uint32_t lo = 0xFFFFFFFFu, hi = 0u;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_frag; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t y = frag[i].y;
        lo = min(lo, y); hi = max(hi, y);
    }
    for (int o = 16; o > 0; o >>= 1) { lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
    if ((threadIdx.x & 31) == 0) { atomicMin(rng, lo); atomicMax(rng + 1, hi); }
}
__global__ void k_wide_lut(WideIndexView w, uint32_t* lut) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t per = (uint64_t)w.cells + 1;
    if (j >= (uint64_t)w.n_block * per) return;
    const uint32_t b = (uint32_t)(j / per), c = (uint32_t)(j - (uint64_t)b * per);
    const uint2* e = w.frag + w.blk_off[b];
    const uint32_t n = (uint32_t)(w.blk_off[b + 1] - w.blk_off[b]);
    uint32_t lo = 0;
    if (c == w.cells) lo = n;
    else if (c > 0) {
        const float edge = w.base + (float)c * (1.0f / w.inv_w);
        uint32_t hi = n;
        while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (__uint_as_float(e[m].y) < edge) lo = m + 1; else hi = m; }
    }
    lut[j] = lo;
}
// One thread per (block, directory cell): #{entries with m/z < edge(c)}, split into the group base (written by the group's first cell) and the
// u16 remainder. A remainder above 65535 (> 65535 entries between two edges of one group: near-degenerate m/z) is clamped, i.e. the walk
// starts earlier than it could; inv_w == 0 (degenerate m/z range) leaves every start at the block start.
__global__ void k_narrow_dir(NarrowIndexView v, uint16_t* dir, uint32_t* grp) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= (uint64_t)v.n_block * v.cells) return;
    const uint32_t b = (uint32_t)(j / v.cells), c = (uint32_t)(j - (uint64_t)b * v.cells);
    const float* m = v.mz + v.blk_off[b];
    const uint32_t n = (uint32_t)(v.blk_off[b + 1] - v.blk_off[b]);
    auto below = [&](uint32_t cc) -> uint32_t {
        if (cc == 0 || !(v.inv_w > 0.0f)) return 0;
        const float edge = v.base + (float)cc * (1.0f / v.inv_w);
        uint32_t lo = 0, hi = n;
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (m[mid] < edge) lo = mid + 1; else hi = mid; }
        return lo;
    };
    const uint32_t g = c / NARROW_GROUP;
    const uint32_t at = below(c), gb = below(g * NARROW_GROUP);
    if (c == g * NARROW_GROUP) grp[(uint64_t)b * (v.cells / NARROW_GROUP) + g] = at;
    dir[j] = (uint16_t)min(at - gb, 65535u);
}

__global__ void k_build_bucket_lut(DbView db, float base, float inv_w, uint32_t* lut) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= BUCKET_LUT_CELLS) return;
    uint32_t lo = 0;
    if (c > 0 && inv_w > 0.0f) {
        const float e = base + (float)c * (1.0f / inv_w);
        uint32_t hi = db.n_bucket;
        while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (db.bucket_min[m] < e) lo = m + 1; else hi = m; }
    }
    lut[c] = lo;
}

// Verifies that an uploaded index is exactly {ions with index > min_ion_index}: per peptide, fragment count and the wrapped sum
// of m/z bit patterns must match what k_gen would emit. acc[2p] = count, acc[2p+1] = sum.
__global__ void k_index_signature(uint64_t n_frag, const uint2* frag, uint32_t n_pep, uint32_t* acc) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_frag) return;
    const uint2 f = frag[i];
    if (f.x >= n_pep) return;
    atomicAdd(acc + 2ull * f.x, 1u);
    atomicAdd(acc + 2ull * f.x + 1, f.y);
}
__global__ void k_index_verify(uint32_t n_pep, const uint8_t* pep_len, const uint32_t* ion_off, const float* ions, uint32_t n_kinds, DbView kinds_src,
                               uint32_t min_ion_index, const uint32_t* acc, uint32_t* mismatch) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pep) return;
    const uint32_t L = pep_len[p];
    const float* src = ions + ion_off[p];
    uint32_t c = 0, sum = 0;
    for (uint32_t k = 0; k < n_kinds; k++)
        for (uint32_t i = 0; i + 1 < L; i++) {
            const bool keep = kinds_src.kinds[k] <= 2 ? (i + 1) > min_ion_index : ((L - 1) - i) > min_ion_index;
            if (keep) { c++; sum += __float_as_uint(src[k * (L - 1) + i]); }
        }
    if (c != acc[2ull * p] || sum != acc[2ull * p + 1]) atomicAdd(mismatch, 1u);
}
__global__ void k_pack_fragments(uint64_t n_frag, const uint64_t* key64, const uint32_t* mzbits, uint2* frag) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_frag) return;
    frag[i] = make_uint2((uint32_t)key64[i], mzbits[i]);
}
__global__ void k_pack_fragments_soa(uint64_t n_frag, const uint32_t* pep, const float* mz, uint2* frag) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_frag) return;
    frag[i] = make_uint2(pep[i], __float_as_uint(mz[i]));
}
__global__ void k_unpack_fragments(uint64_t n_frag, const uint2* frag, uint32_t* pep, float* mz) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_frag) return;
    const uint2 f = frag[i];
    if (pep) pep[i] = f.x;
    if (mz) mz[i] = __uint_as_float(f.y);
}

}  // namespace sb
