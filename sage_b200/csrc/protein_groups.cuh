// protein_groups.cuh — protein grouping on the device: Sage's protein_grouping.rs (ProteinGrouper::build, BipartiteGraph::into_cover,
// ProteinGroupLookup::group_string) and the keys of fdr.rs picked_protein_group. Host orchestration: sage_b200.cu (sage_b200_protein_groups,
// sage_b200_bipartite_cover). Integer-only: every output is exact (DESIGN.md §13).
//
// The cover runs in two phases, by the two facts DESIGN.md §13 proves: an uncovered peptide never loses degree, so every forced pick is made
// by the first trim from the original degrees; after that the connected components are independent, and each runs the greedy alone
// (one warp per small component, one CTA per large one), with Rust's max_by_key tie rule: the last index among equal (remaining, original).
#pragma once
#include <stdint.h>

namespace sb {

constexpr uint32_t PG_NONE = 0xFFFFFFFFu;
constexpr uint32_t PG_LARGE = 512;   // components with more groups than this run on one CTA of PG_CTA threads
constexpr uint32_t PG_CTA = 512;

// ------------------------------------------------------------------------------------------------ ProteinGrouper::build
// The pass's peptide set (protein_grouping.rs annotate_features): label != -1 && peptide_q < threshold. NaN compares false.
__global__ void k_pg_mark(const uint32_t* __restrict__ pep, const uint8_t* __restrict__ label_ok, const float* __restrict__ q, uint32_t n, float threshold,
                          uint8_t* __restrict__ mark) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && label_ok[i] && q[i] < threshold) mark[pep[i]] = 1;
}

__global__ void k_pg_set_len(const uint32_t* __restrict__ set, const uint32_t* __restrict__ poff, uint32_t U, uint32_t* __restrict__ len) {
    const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u < U) len[u] = poff[set[u] + 1] - poff[set[u]];
}

// The (peptide, protein) pairs of the set in scan order (ascending PeptideIx, each list in stored order): key = 2 * id + peptide.decoy, and
// the first position of each key, which numbers the ProteinIx by first encounter.
__global__ void k_pg_flatten(const uint32_t* __restrict__ set, const uint32_t* __restrict__ soff, const uint32_t* __restrict__ poff,
                             const uint32_t* __restrict__ pids, const uint8_t* __restrict__ pdecoy, uint32_t U, uint32_t* __restrict__ pair_key,
                             uint32_t* __restrict__ first) {
    const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= U) return;
    const uint32_t q = set[u], a = poff[q], b = poff[q + 1], o = soff[u], d = pdecoy[q] ? 1u : 0u;
    for (uint32_t j = a; j < b; j++) {
        const uint32_t key = 2 * pids[j] + d, pos = o + (j - a);
        pair_key[pos] = key;
        atomicMin(first + key, pos);
    }
}

__global__ void k_pg_key_present(const uint32_t* __restrict__ first, uint32_t n_keys, uint8_t* __restrict__ flag) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n_keys) flag[k] = first[k] != PG_NONE;
}

__global__ void k_pg_gather_u32(const uint32_t* __restrict__ src, const uint32_t* __restrict__ at, uint32_t n, uint32_t* __restrict__ dst) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[at[i]];
}

// pix_of_key[key of ProteinIx r] = r
__global__ void k_pg_scatter_rank(const uint32_t* __restrict__ key_by_pix, uint32_t P, uint32_t* __restrict__ pix_of_key) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < P) pix_of_key[key_by_pix[r]] = r;
}

__global__ void k_pg_pair_pix(const uint32_t* __restrict__ pair_key, const uint32_t* __restrict__ pix_of_key, uint32_t T, uint32_t* __restrict__ pix) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < T) pix[t] = pix_of_key[pair_key[t]];
}

// Lexicographic order of Vec<u32> (a prefix first) over a CSR: list i is val[off[i] .. off[i+1]).
struct PgLexLess {
    const uint32_t* val;
    const uint32_t* off;
    __device__ bool operator()(uint32_t a, uint32_t b) const {
        const uint32_t oa = off[a], la = off[a + 1] - oa, ob = off[b], lb = off[b + 1] - ob;
        const uint32_t L = la < lb ? la : lb;
        for (uint32_t j = 0; j < L; j++) {
            const uint32_t x = val[oa + j], y = val[ob + j];
            if (x != y) return x < y;
        }
        return la < lb;
    }
};

__device__ __forceinline__ bool pg_lex_equal(const uint32_t* val, const uint32_t* off, uint32_t a, uint32_t b) {
    const uint32_t oa = off[a], la = off[a + 1] - oa, ob = off[b], lb = off[b + 1] - ob;
    if (la != lb) return false;
    for (uint32_t j = 0; j < la; j++)
        if (val[oa + j] != val[ob + j]) return false;
    return true;
}

// Heads of runs of equal lists in lexicographic order: the rank of a run is the meta-peptide (or group) index.
__global__ void k_pg_lex_heads(const uint32_t* __restrict__ sorted, const uint32_t* __restrict__ val, const uint32_t* __restrict__ off, uint32_t n,
                               uint32_t* __restrict__ head) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < n) head[p] = (p == 0 || !pg_lex_equal(val, off, sorted[p - 1], sorted[p])) ? 1u : 0u;
}

// rank_of[sorted[p]] = inclusive head count - 1
__global__ void k_pg_rank_of(const uint32_t* __restrict__ sorted, const uint32_t* __restrict__ incl, uint32_t n, uint32_t* __restrict__ rank_of) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < n) rank_of[sorted[p]] = incl[p] - 1;
}

__global__ void k_pg_csr_len(const uint32_t* __restrict__ rep, const uint32_t* __restrict__ off, uint32_t n, uint32_t* __restrict__ len) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) len[i] = off[rep[i] + 1] - off[rep[i]];
}

// protein_grouping.rs:188-194: every entry of meta-peptide m's list (with multiplicity) gives the pair (ProteinIx, m), sorted later.
__global__ void k_pg_meta_pairs(const uint32_t* __restrict__ rep, const uint32_t* __restrict__ val, const uint32_t* __restrict__ off,
                                const uint32_t* __restrict__ moff, uint32_t M, uint64_t* __restrict__ pair, uint32_t* __restrict__ deg) {
    const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    const uint32_t a = off[rep[m]], b = off[rep[m] + 1], o = moff[m];
    for (uint32_t j = a; j < b; j++) {
        pair[o + (j - a)] = ((uint64_t)val[j] << 32) | m;
        atomicAdd(deg + val[j], 1u);
    }
}

__global__ void k_pg_low32(const uint64_t* __restrict__ pair, uint32_t n, uint32_t* __restrict__ lo) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) lo[i] = (uint32_t)pair[i];
}

// Group members as (group << 32 | name id), sorted later into each group's ascending ids; the group's decoy flag.
__global__ void k_pg_members(const uint32_t* __restrict__ group_of, const uint32_t* __restrict__ key_by_pix, uint32_t P, uint64_t* __restrict__ member,
                             uint32_t* __restrict__ gsize, uint8_t* __restrict__ gdecoy) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= P) return;
    const uint32_t g = group_of[r], key = key_by_pix[r];
    member[r] = ((uint64_t)g << 32) | (key >> 1);
    atomicAdd(gsize + g, 1u);
    gdecoy[g] = (uint8_t)(key & 1u);
}

// protein_grouping.rs:206-212: edges (group, each entry of its evidence list).
__global__ void k_pg_edges(const uint32_t* __restrict__ rep, const uint32_t* __restrict__ ev, const uint32_t* __restrict__ ev_off,
                           const uint32_t* __restrict__ eoff, uint32_t G, uint32_t* __restrict__ el, uint32_t* __restrict__ er) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const uint32_t a = ev_off[rep[g]], b = ev_off[rep[g] + 1], o = eoff[g];
    for (uint32_t j = a; j < b; j++) {
        el[o + (j - a)] = g;
        er[o + (j - a)] = ev[j];
    }
}

// ------------------------------------------------------------------------------------------------ BipartiteGraph::into_cover
__global__ void k_pg_degrees(const uint32_t* __restrict__ el, const uint32_t* __restrict__ er, uint32_t E, uint32_t* __restrict__ ldeg,
                             uint32_t* __restrict__ rdeg) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    atomicAdd(ldeg + el[e], 1u);
    atomicAdd(rdeg + er[e], 1u);
}

// The first trim's forced picks: a right node of degree 1 covers its left node.
__global__ void k_pg_forced(const uint32_t* __restrict__ el, const uint32_t* __restrict__ er, const uint32_t* __restrict__ rdeg, uint32_t E,
                            uint8_t* __restrict__ lcov) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < E && rdeg[er[e]] == 1) lcov[el[e]] = 1;
}

__global__ void k_pg_cover_rights(const uint32_t* __restrict__ el, const uint32_t* __restrict__ er, const uint8_t* __restrict__ lcov, uint32_t E,
                                  uint32_t* __restrict__ rcov) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < E && lcov[el[e]]) rcov[er[e]] = 1;
}

// Remaining degree after the first trim: the edges of an uncovered left node to uncovered right nodes.
__global__ void k_pg_remaining(const uint32_t* __restrict__ ladj, const uint32_t* __restrict__ loff, const uint8_t* __restrict__ lcov,
                               const uint32_t* __restrict__ rcov, uint32_t G, uint32_t* __restrict__ rem, uint8_t* __restrict__ active) {
    const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= G) return;
    uint32_t c = 0;
    if (!lcov[l])
        for (uint32_t k = loff[l]; k < loff[l + 1]; k++) c += rcov[ladj[k]] ? 0u : 1u;
    rem[l] = c;
    active[l] = c > 0;
}

// Lock-free union-find over the remaining edges: nodes 0..G-1 are left, G.. right. A root is hooked under the smaller root by CAS.
__device__ __forceinline__ uint32_t pg_find(uint32_t* parent, uint32_t x) {
    uint32_t p = __ldcg(parent + x);
    while (p != x) {
        x = p;
        p = __ldcg(parent + x);
    }
    return x;
}

__global__ void k_pg_union(const uint32_t* __restrict__ el, const uint32_t* __restrict__ er, const uint8_t* __restrict__ lcov,
                           const uint32_t* __restrict__ rcov, uint32_t E, uint32_t G, uint32_t* parent) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E || lcov[el[e]] || rcov[er[e]]) return;
    uint32_t a = el[e], b = G + er[e];
    while (true) {
        a = pg_find(parent, a);
        b = pg_find(parent, b);
        if (a == b) return;
        if (a < b) { const uint32_t t = a; a = b; b = t; }
        if (atomicCAS(parent + a, a, b) == a) return;
    }
}

__global__ void k_pg_comp_of(uint32_t* parent, const uint32_t* __restrict__ act, uint32_t n_act, uint32_t* __restrict__ comp) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_act) comp[i] = pg_find(parent, act[i]);
}

// The max of (remaining, original, index) over a team, remaining >= 1: Rust's max_by_key keeps the last of equal keys, so the larger index wins.
struct PgBest {
    uint64_t key;   // remaining << 32 | original; 0 = none
    uint32_t idx;
};
__device__ __forceinline__ PgBest pg_better(PgBest a, PgBest b) { return (b.key > a.key || (b.key == a.key && b.idx > a.idx)) ? b : a; }
__device__ __forceinline__ PgBest pg_warp_best(PgBest v) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        PgBest o;
        o.key = __shfl_xor_sync(0xffffffffu, v.key, s);
        o.idx = __shfl_xor_sync(0xffffffffu, v.idx, s);
        v = pg_better(v, o);
    }
    return v;
}

// The greedy of one component over its groups lefts[0..s), ascending: pick the best, cover its uncovered right nodes (claimed once each,
// so parallel edges count once per node), and take one from the remaining degree of every left node at each of their edges.
// TEAM = 32: one warp per component; TEAM = PG_CTA: one CTA.
template <uint32_t TEAM>
__device__ void pg_greedy(const uint32_t* __restrict__ lefts, uint32_t s, const uint32_t* __restrict__ ldeg, const uint32_t* __restrict__ ladj,
                          const uint32_t* __restrict__ loff, const uint32_t* __restrict__ radj, const uint32_t* __restrict__ roff, uint32_t* rem,
                          uint32_t* rcov, uint8_t* __restrict__ lcov, unsigned long long* picks) {
    __shared__ PgBest part[TEAM / 32];
    const uint32_t t = threadIdx.x % TEAM;
    uint32_t n_picks = 0;
    while (true) {
        PgBest b{0, 0};
        for (uint32_t k = t; k < s; k += TEAM) {
            const uint32_t l = lefts[k], r = __ldcg(rem + l);
            if (r) b = pg_better(b, PgBest{((uint64_t)r << 32) | ldeg[l], l});
        }
        b = pg_warp_best(b);
        if (TEAM > 32) {
            if ((t & 31) == 0) part[t >> 5] = b;
            __syncthreads();
            b = part[0];
            for (uint32_t w = 1; w < TEAM / 32; w++) b = pg_better(b, part[w]);
            __syncthreads();
        }
        if (b.key == 0) break;
        const uint32_t l = b.idx;
        for (uint32_t k = loff[l] + t; k < loff[l + 1]; k += TEAM) {
            const uint32_t r = ladj[k];
            if (atomicExch(rcov + r, 1u) == 0u)
                for (uint32_t j = roff[r]; j < roff[r + 1]; j++) atomicSub(rem + radj[j], 1u);
        }
        if (t == 0) lcov[l] = 1;
        n_picks++;
        if (TEAM > 32) __syncthreads(); else __syncwarp();
    }
    if (t == 0) atomicAdd(picks, (unsigned long long)n_picks);
}

__global__ void __launch_bounds__(256) k_pg_greedy_warp(const uint32_t* __restrict__ comp_off, const uint32_t* __restrict__ comp_len, uint32_t n_comp,
                                                        const uint32_t* __restrict__ lefts, const uint32_t* __restrict__ ldeg, const uint32_t* __restrict__ ladj,
                                                        const uint32_t* __restrict__ loff, const uint32_t* __restrict__ radj, const uint32_t* __restrict__ roff,
                                                        uint32_t* rem, uint32_t* rcov, uint8_t* __restrict__ lcov, unsigned long long* picks) {
    const uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
    if (c >= n_comp || comp_len[c] > PG_LARGE) return;
    pg_greedy<32>(lefts + comp_off[c], comp_len[c], ldeg, ladj, loff, radj, roff, rem, rcov, lcov, picks);
}

__global__ void __launch_bounds__(PG_CTA) k_pg_greedy_cta(const uint32_t* __restrict__ large, const uint32_t* __restrict__ comp_off,
                                                          const uint32_t* __restrict__ comp_len, const uint32_t* __restrict__ lefts,
                                                          const uint32_t* __restrict__ ldeg, const uint32_t* __restrict__ ladj, const uint32_t* __restrict__ loff,
                                                          const uint32_t* __restrict__ radj, const uint32_t* __restrict__ roff, uint32_t* rem, uint32_t* rcov,
                                                          uint8_t* __restrict__ lcov, unsigned long long* picks) {
    const uint32_t c = large[blockIdx.x];
    pg_greedy<PG_CTA>(lefts + comp_off[c], comp_len[c], ldeg, ladj, loff, radj, roff, rem, rcov, lcov, picks);
}

__global__ void k_pg_large_flag(const uint32_t* __restrict__ comp_len, uint32_t n_comp, uint8_t* __restrict__ flag) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < n_comp) flag[c] = comp_len[c] > PG_LARGE;
}

// ------------------------------------------------------------------------------------------------ ProteinGroupLookup::group_string
// One thread per row still unannotated: each (id, peptide.decoy) of its peptide -> ProteinIx -> group -> covered? The distinct covered groups
// (global index base + g) are kept ascending in the row's slot of the scratch; a nonempty set annotates the row with this pass.
__global__ void k_pg_lookup(const uint32_t* __restrict__ pep, uint32_t n, const uint32_t* __restrict__ poff, const uint32_t* __restrict__ pids,
                            const uint8_t* __restrict__ pdecoy, const uint64_t* __restrict__ cap_off, const uint32_t* __restrict__ pix_of_key,
                            const uint32_t* __restrict__ group_of, const uint8_t* __restrict__ lcov, uint32_t base, uint8_t pass_no,
                            uint8_t* __restrict__ pass, uint32_t* __restrict__ count, uint32_t* __restrict__ scratch, unsigned long long* annotated) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || pass[i]) return;
    const uint32_t q = pep[i], d = pdecoy[q] ? 1u : 0u;
    uint32_t* out = scratch + cap_off[i];
    uint32_t c = 0;
    for (uint32_t j = poff[q]; j < poff[q + 1]; j++) {
        const uint32_t r = pix_of_key[2 * pids[j] + d];
        if (r == PG_NONE) continue;
        const uint32_t g = group_of[r];
        if (!lcov[g]) continue;
        const uint32_t v = base + g;
        uint32_t k = c;
        while (k > 0 && out[k - 1] > v) k--;
        if (k > 0 && out[k - 1] == v) continue;
        for (uint32_t m = c; m > k; m--) out[m] = out[m - 1];
        out[k] = v;
        c++;
    }
    if (c) {
        pass[i] = pass_no;
        count[i] = c;
        atomicAdd(annotated, 1ull);
    }
}

__global__ void k_pg_fallback(const uint32_t* __restrict__ pep, uint32_t n, const uint32_t* __restrict__ poff, const uint8_t* __restrict__ pass,
                              uint32_t* __restrict__ count, uint32_t* __restrict__ csr_len) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (!pass[i]) count[i] = poff[pep[i] + 1] - poff[pep[i]];
    csr_len[i] = pass[i] ? count[i] : 0u;
}

__global__ void k_pg_compact_rows(const uint64_t* __restrict__ cap_off, const uint64_t* __restrict__ out_off, const uint32_t* __restrict__ scratch,
                                  const uint32_t* __restrict__ csr_len, uint32_t n, uint32_t* __restrict__ row_groups) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (uint32_t k = 0; k < csr_len[i]; k++) row_groups[out_off[i] + k] = scratch[cap_off[i] + k];
}

// ------------------------------------------------------------------------------------------------ picked_protein_group keys
// A group string is equal to another when the sets of (name, tagged) are: tagged = decoy && generate_decoys. Single-name strings (a
// singleton group, or a fallback row of one protein) key as 2 * id + tagged; groups of several names are hashed and grouped exactly.
__device__ __forceinline__ uint64_t pg_mix(uint64_t h, uint64_t x) {
    h ^= x + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
    h *= 0xFF51AFD7ED558CCDull;
    return h ^ (h >> 31);
}

__global__ void k_pg_group_hash(const uint32_t* __restrict__ goff, const uint32_t* __restrict__ members, const uint8_t* __restrict__ gdecoy,
                                uint32_t G, bool gen, uint64_t* __restrict__ hash, uint32_t* __restrict__ idx) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    uint64_t h = pg_mix(0x9E37, (gen && gdecoy[g]) ? 1u : 0u);
    for (uint32_t k = goff[g]; k < goff[g + 1]; k++) h = pg_mix(h, members[k]);
    hash[g] = h;
    idx[g] = g;
}

__device__ __forceinline__ bool pg_group_equal(const uint32_t* goff, const uint32_t* members, const uint8_t* gdecoy, bool gen, uint32_t a, uint32_t b) {
    if ((gen && gdecoy[a]) != (gen && gdecoy[b])) return false;
    const uint32_t oa = goff[a], la = goff[a + 1] - oa, ob = goff[b], lb = goff[b + 1] - ob;
    if (la != lb) return false;
    for (uint32_t k = 0; k < la; k++)
        if (members[oa + k] != members[ob + k]) return false;
    return true;
}

// rep[g] = the first sorted position of g's equal-hash run whose group is equal to g (the pattern of k_picked_group).
__global__ void k_pg_group_rep(const uint32_t* __restrict__ goff, const uint32_t* __restrict__ members, const uint8_t* __restrict__ gdecoy, bool gen,
                               const uint64_t* __restrict__ hash_s, const uint32_t* __restrict__ g_s, uint32_t G, uint32_t* __restrict__ rep) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= G) return;
    const uint64_t h = hash_s[p];
    const uint32_t g = g_s[p];
    uint32_t r = p;
    for (uint32_t q = p; q-- > 0 && hash_s[q] == h;)
        if (pg_group_equal(goff, members, gdecoy, gen, g_s[q], g)) r = q;
    rep[g] = r;
}

// Each row with exactly one group string: its competition key, side (Peptide::decoy) and score, compacted in row order by the caller's select.
__global__ void k_pg_row_keys(const uint32_t* __restrict__ pep, uint32_t n, const uint8_t* __restrict__ pass, const uint32_t* __restrict__ count,
                              const uint64_t* __restrict__ out_off, const uint32_t* __restrict__ row_groups, const uint32_t* __restrict__ goff,
                              const uint32_t* __restrict__ members, const uint8_t* __restrict__ gdecoy, const uint32_t* __restrict__ rep,
                              const uint32_t* __restrict__ poff, const uint32_t* __restrict__ pids, const uint8_t* __restrict__ pdecoy, bool gen,
                              uint32_t n_names, uint32_t* __restrict__ key, uint8_t* __restrict__ side, uint8_t* __restrict__ competes) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t q = pep[i];
    const bool dec = pdecoy[q] != 0;
    competes[i] = count[i] == 1;
    side[i] = dec;
    if (count[i] != 1) return;
    if (!pass[i]) {
        key[i] = 2 * pids[poff[q]] + ((gen && dec) ? 1u : 0u);
        return;
    }
    const uint32_t g = row_groups[out_off[i]];
    const uint32_t t = (gen && gdecoy[g]) ? 1u : 0u;
    key[i] = goff[g + 1] - goff[g] == 1 ? 2 * members[goff[g]] + t : 2 * n_names + rep[g];
}

// Nonzero flags counted into *count.
__global__ void k_pg_count(const uint8_t* __restrict__ flag, uint32_t n, unsigned long long* count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned m = __ballot_sync(0xffffffffu, i < n && flag[i]);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(count, (unsigned long long)__popc(m));
}

__global__ void k_pg_add(uint32_t* __restrict__ v, uint32_t n, uint32_t x) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] += x;
}

__global__ void k_pg_scatter_q(const uint32_t* __restrict__ row, const float* __restrict__ q, uint32_t m, float* __restrict__ out) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < m) out[row[c]] = q[c];
}

__global__ void k_pg_fill(float* __restrict__ v, uint32_t n, float x) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = x;
}

}  // namespace sb
