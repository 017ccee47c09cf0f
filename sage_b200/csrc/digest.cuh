// digest.cuh — FASTA -> peptide table on the device: Sage's enzyme.rs (cleavage sites, missed-cleavage and semi-enzymatic windows,
// per-protein de-duplication, group_digests), peptide.rs:258-388 (Peptide::try_from, apply, reverse) and database.rs:162-258
// (Parameters::digest, reorder_peptides). Host orchestration (FASTA parsing, the parameter normalisation, the stage order): sage_b200.cu
// (sage_b200_digest_create). DESIGN.md §14 states the exactness contract and the tie argument.
//
// Layout: a window is (protein, start, length, missed, semi, position) in generation order; a group is one (sequence, position, decoy) of
// group_digests, held as its reference window; a form is one modified peptide of a group, held compactly as (group, chosen variable sites,
// reversed) until the output kernel writes its residues and modifications.
#pragma once
#include <stdint.h>

#include "picked.cuh"   // picked_mix, picked_pos: the 64-bit key mix and the reversed-interior index of Peptide::reverse

namespace sb {

constexpr float DG_H2O = 18.010565f;   // mass.rs:5
constexpr uint32_t DG_KMAX = 8;        // the largest max_variable_mods the compact form holds
enum { DG_POS_NTERM = 0, DG_POS_CTERM = 1, DG_POS_FULL = 2, DG_POS_INTERNAL = 3 };   // enzyme.rs:64-71 Position
enum { DG_SPEC_PEP_N = 0, DG_SPEC_PEP_C = 1, DG_SPEC_PROT_N = 2, DG_SPEC_PROT_C = 3, DG_SPEC_RESIDUE = 4 };   // ModificationSpecificity
enum { DG_SITE_N = 0, DG_SITE_C = 1, DG_SITE_SEQ = 2 };   // peptide.rs ModificationSite

// mass.rs:64-76
__constant__ float c_dg_mono[26] = {71.03711f, 0.0f,      103.00919f, 115.02694f, 129.04259f, 147.0684f, 57.02146f,  137.05891f, 113.08406f,
                                    0.0f,      128.09496f, 113.08406f, 131.0405f,  114.04293f, 237.14774f, 97.05276f, 128.05858f, 156.1011f,
                                    87.03203f, 101.04768f, 150.95363f, 99.06841f,  186.07932f, 0.0f,       163.06332f, 0.0f};

struct DgWin {
    uint32_t start;   // global residue index of the window's first residue
    uint32_t prot;    // protein index in parse order
    uint16_t len;
    uint8_t missed;
    uint8_t flags;    // bit 0: semi-enzymatic; bits 1-2: Position
};

struct DgForm {
    uint32_t group;
    uint8_t n;                 // chosen variable sites
    uint8_t rev;               // Peptide::reverse applied
    uint16_t sel[DG_KMAX];     // indices into the group's site list, ascending
};

// A mod spec as the device reads it: kind (DG_SPEC_*), residue (-1 = None) and mass.
struct DgSpec {
    int32_t kind, residue;
    float mass;
};

struct DgParams {
    uint32_t cleave, restrict_;   // A..Z bit masks of the cleave class and of `restrict`
    uint32_t min_len, max_len, missed;
    uint8_t has_enzyme, dollar, c_terminal, semi, generate_decoys;
    uint32_t kmax;                // max_variable_mods, at least 1
    float min_mass, max_mass;
    uint32_t n_static, n_var;
    const DgSpec* statics;        // Builder order: by spec, one mass per spec
    const DgSpec* vars;           // stable-sorted by spec, one entry per (spec, mass)
};

// Everything the form-level device functions read.
struct DgView {
    const uint8_t* res;           // residues of every protein, concatenated
    const uint32_t* prot_off;     // [P + 1]
    const DgWin* win;
    const uint32_t* grp_win;      // reference window of each group
    const uint8_t* grp_meta;      // Position | decoy << 2
    const uint32_t* site_off;     // [G + 1] into site_code / site_mass
    const uint32_t* site_code;    // kind << 16 | residue index
    const float* site_mass;
    const DgForm* forms;
    const float* form_mono;
    DgParams p;
};

__device__ __forceinline__ float dg_residue_mass(uint8_t c) { return (c >= 'A' && c <= 'Z') ? c_dg_mono[c - 'A'] : 0.0f; }

// ------------------------------------------------------------------------------------------------ cleavage sites (enzyme.rs:186-240)
// One warp per protein: a ballot over the residues marks the positions where a site is cut (try_site's `restrict` test applied), the lanes'
// counts are scanned and the cut positions are written in order. Pass 1 (cuts == nullptr) only counts.
__global__ void k_dg_sites(const uint8_t* __restrict__ res, const uint32_t* __restrict__ prot_off, uint32_t P, DgParams p,
                           uint32_t* __restrict__ n_cuts, const uint32_t* __restrict__ cut_off, uint32_t* __restrict__ cuts) {
    const uint32_t prot = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (prot >= P) return;
    const uint32_t o = prot_off[prot], n = prot_off[prot + 1] - o;
    if (!p.has_enzyme) {   // the non-specific digest has no sites
        if (!cuts && lane == 0) n_cuts[prot] = 0;
        return;
    }
    uint32_t count = 0, base = cuts ? cut_off[prot] : 0;
    for (uint32_t c0 = 0; c0 < n; c0 += 32) {
        const uint32_t i = c0 + lane;
        bool cut = false;
        uint32_t right = 0;
        if (i < n) {
            if (p.dollar) {   // regex "$": one empty match at the end
                cut = i == n - 1;
                right = n;
            } else {
                const uint8_t b = res[o + i];
                if (b >= 'A' && b <= 'Z' && ((p.cleave >> (b - 'A')) & 1u)) {
                    right = p.c_terminal ? i + 1 : i;
                    cut = true;
                    if (right < n) {
                        const uint8_t r = res[o + right];
                        if (r >= 'A' && r <= 'Z' && ((p.restrict_ >> (r - 'A')) & 1u)) cut = false;
                    }
                }
            }
        }
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, cut);
        if (cuts && cut) cuts[base + count + __popc(m & ((1u << lane) - 1u))] = right;
        count += __popc(m);
    }
    if (!cuts && lane == 0) n_cuts[prot] = count;
}

// ------------------------------------------------------------------------------------------------ windows (enzyme.rs:242-342)
// Every window of one protein in generation order: the base sites, the missed-cleavage windows (cleavage = 1..=1+missed over all base
// sites), then the semi-enzymatic sub-windows of each of those; or, without an enzyme, every (start, len) of min_len..=max_len. visit(start,
// end, missed, semi) is called for each; the length filter is the caller's.
template <class F>
__device__ void dg_for_windows(const DgParams& p, const uint32_t* cuts, uint32_t k, uint32_t n, F visit) {
    if (!p.has_enzyme) {
        for (uint32_t len = p.min_len; len <= p.max_len; len++)
            if (n >= len)
                for (uint32_t i = 0; i + len <= n; i++) visit(i, i + len, 0u, false);
        return;
    }
    const uint32_t m = k + 1;   // base sites: (0, c0), (c0, c1), ..., (c_{k-1}, n)
    auto s_of = [&](uint32_t j) { return j == 0 ? 0u : cuts[j - 1]; };
    auto e_of = [&](uint32_t j) { return j == k ? n : cuts[j]; };
    auto l1 = [&](auto f) {
        for (uint32_t j = 0; j < m; j++) f(s_of(j), e_of(j), 0u);
        if (p.missed > 0)
            for (uint32_t c = 1; c <= 1 + p.missed; c++)
                if (m >= c)
                    for (uint32_t w = 0; w + c <= m; w++) f(s_of(w), e_of(w + c - 1), c - 1);
    };
    l1([&](uint32_t s, uint32_t e, uint32_t miss) { visit(s, e, miss, false); });
    if (p.semi)
        l1([&](uint32_t s, uint32_t e, uint32_t miss) {
            for (uint32_t cut = s; cut < e; cut++) {
                visit(s, cut, miss, true);
                visit(cut, e, miss, true);
            }
        });
}

// One thread per protein. Pass 1 (out == nullptr) counts the windows that pass the length filter; pass 2 writes them at win_off[prot].
__global__ void k_dg_windows(const uint32_t* __restrict__ prot_off, const uint32_t* __restrict__ cut_off, const uint32_t* __restrict__ cuts, uint32_t P,
                             DgParams p, uint64_t* __restrict__ n_win, const uint64_t* __restrict__ win_off, DgWin* __restrict__ out) {
    const uint32_t prot = blockIdx.x * blockDim.x + threadIdx.x;
    if (prot >= P) return;
    const uint32_t o = prot_off[prot], n = prot_off[prot + 1] - o;
    const uint32_t c0 = cut_off[prot], k = cut_off[prot + 1] - c0;
    uint64_t at = out ? win_off[prot] : 0, count = 0;
    dg_for_windows(p, cuts + c0, k, n, [&](uint32_t s, uint32_t e, uint32_t miss, bool semi) {
        if (s > e || e > n) return;
        const uint32_t len = e - s;
        if (len < p.min_len || len > p.max_len || len == 0) return;
        if (out) {
            const uint32_t pos = s == 0 ? (e == n ? DG_POS_FULL : DG_POS_NTERM) : (e == n ? DG_POS_CTERM : DG_POS_INTERNAL);
            out[at++] = DgWin{o + s, prot, (uint16_t)len, (uint8_t)miss, (uint8_t)((semi ? 1u : 0u) | (pos << 1))};
        }
        count++;
    });
    if (!out) n_win[prot] = count;
}

// ------------------------------------------------------------------------------------------------ per-protein `seen` and group_digests
__device__ __forceinline__ uint64_t dg_hash(const uint8_t* s, uint32_t L, bool rev) {
    uint64_t h = picked_mix(0x5A6E, L);
    for (uint32_t j = 0; j < L; j++) h = picked_mix(h, s[picked_pos(j, L, rev)]);
    return h;
}

__global__ void k_dg_hash(const uint8_t* __restrict__ res, const DgWin* __restrict__ win, uint32_t W, uint64_t* __restrict__ hash, uint32_t* __restrict__ idx) {
    const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= W) return;
    const DgWin x = win[w];
    hash[w] = dg_hash(res + x.start, x.len, false);
    idx[w] = w;
}

__global__ void k_dg_run_start(const uint64_t* __restrict__ hash_s, uint32_t W, uint32_t* __restrict__ rs) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < W) rs[q] = (q == 0 || hash_s[q] != hash_s[q - 1]) ? q : 0u;
}

// Exact classes after the sort by hash: the window at sorted position q takes the first position of its equal-hash run (rs = inclusive max
// scan of the run heads) whose residues equal its own. Without a collision that is the run's head, found at the first comparison.
__global__ void k_dg_class(const uint8_t* __restrict__ res, const DgWin* __restrict__ win, const uint32_t* __restrict__ idx_s, const uint32_t* __restrict__ rs,
                           uint32_t W, uint32_t* __restrict__ cls) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= W) return;
    const DgWin x = win[idx_s[q]];
    uint32_t c = q;
    for (uint32_t r = rs[q]; r < q; r++) {
        const DgWin y = win[idx_s[r]];
        if (y.len != x.len) continue;
        uint32_t j = 0;
        while (j < x.len && res[x.start + j] == res[y.start + j]) j++;
        if (j == x.len) {
            c = r;
            break;
        }
    }
    cls[q] = c;
}

// After the stable sort by class, each class lists its windows in (protein, generation) order: the first window of each (class, protein)
// is the one the protein's `seen` set keeps. Its group key is (class, Position, decoy); group_digests' stable sort puts the lowest protein first.
__global__ void k_dg_seen(const DgWin* __restrict__ win, const uint32_t* __restrict__ cls_s, const uint32_t* __restrict__ idx_s, const uint8_t* __restrict__ prot_decoy,
                          uint32_t W, uint8_t* __restrict__ keep, uint64_t* __restrict__ key) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= W) return;
    const DgWin x = win[idx_s[q]];
    keep[q] = (q == 0 || cls_s[q] != cls_s[q - 1] || win[idx_s[q - 1]].prot != x.prot) ? 1 : 0;
    key[q] = ((uint64_t)cls_s[q] << 3) | ((uint64_t)((x.flags >> 1) & 3u) << 1) | (prot_decoy[x.prot] ? 1u : 0u);
}

__global__ void k_dg_heads64(const uint64_t* __restrict__ key, uint32_t n, uint32_t* __restrict__ head) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < n) head[q] = (q == 0 || key[q] != key[q - 1]) ? 1u : 0u;
}

// Per group: its reference window and (Position, decoy); the class's flag "holds a target group" (the `targets` set without generate_decoys).
__global__ void k_dg_groups(const uint64_t* __restrict__ key_s, const uint32_t* __restrict__ idx_s, const uint32_t* __restrict__ grp_start, uint32_t G,
                            uint32_t* __restrict__ grp_win, uint8_t* __restrict__ grp_meta, uint32_t* __restrict__ grp_cls, uint8_t* __restrict__ cls_target) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const uint32_t q = grp_start[g];
    const uint64_t k = key_s[q];
    grp_win[g] = idx_s[q];
    grp_meta[g] = (uint8_t)(((k >> 1) & 3u) | ((k & 1u) << 2));
    grp_cls[g] = (uint32_t)(k >> 3);
    if (!(k & 1u)) cls_target[k >> 3] = 1;
}

// ------------------------------------------------------------------------------------------------ Peptide::try_from, apply (peptide.rs:156-388)
// Per group: whether Peptide::try_from accepts the sequence, its base mass (H2O + residues, a sequential f32 sum), its variable-mod site
// count, its form count 1 + sum_{n=1..kmax} C(sites, n) (0 when rejected), and with generate_decoys whether its reversed sequence is a target.
__device__ __forceinline__ uint64_t dg_binom(uint32_t s, uint32_t n) {   // C(s, n), saturating at 2^62
    if (n > s) return 0;
    uint64_t r = 1;
    for (uint32_t i = 1; i <= n; i++) {
        const uint64_t f = s - n + i;
        if (r > (1ull << 62) / f) return 1ull << 62;
        r = r * f / i;
    }
    return r;
}

// push_resi (peptide.rs:156-208) for one variable spec over a forward sequence; site(code) is called per site in order.
template <class F>
__device__ void dg_var_sites(const DgSpec& t, const uint8_t* s, uint32_t L, uint32_t pos, F site) {
    const bool nt = pos == DG_POS_NTERM || pos == DG_POS_FULL, ct = pos == DG_POS_CTERM || pos == DG_POS_FULL;
    const int first = s[0], last = s[L - 1];
    switch (t.kind) {
        case DG_SPEC_PROT_N:
            if (!nt) break;
            // fallthrough
        case DG_SPEC_PEP_N:
            if (t.residue < 0) site(DG_SITE_N << 16);
            else if (t.residue == first) site(DG_SITE_SEQ << 16);
            break;
        case DG_SPEC_PROT_C:
            if (!ct) break;
            // fallthrough
        case DG_SPEC_PEP_C:
            if (t.residue < 0) site(DG_SITE_C << 16);
            else if (t.residue == last) site((DG_SITE_SEQ << 16) | (L - 1));
            break;
        default:
            for (uint32_t i = 0; i < L; i++)
                if (s[i] == t.residue) site((DG_SITE_SEQ << 16) | i);
    }
}

__global__ void k_dg_group_info(const uint8_t* __restrict__ res, const DgWin* __restrict__ win, const uint32_t* __restrict__ grp_win,
                                const uint8_t* __restrict__ grp_meta, uint32_t G, DgParams p, const uint64_t* __restrict__ hash_s,
                                const uint32_t* __restrict__ idx_s, uint32_t W, float* __restrict__ grp_base, uint32_t* __restrict__ n_sites,
                                uint64_t* __restrict__ n_forms, uint8_t* __restrict__ rev_target, uint32_t* __restrict__ overflow) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const DgWin x = win[grp_win[g]];
    const uint8_t* s = res + x.start;
    const uint32_t L = x.len, pos = grp_meta[g] & 3u;
    float mass = DG_H2O;
    bool ok = true;
    for (uint32_t j = 0; j < L; j++) {
        const uint8_t c = s[j];
        const float m = dg_residue_mass(c);
        if (c >= 128 || m == 0.0f) {
            ok = false;
            break;
        }
        mass += m;
    }
    grp_base[g] = mass;
    uint32_t S = 0;
    for (uint32_t v = 0; ok && v < p.n_var; v++) dg_var_sites(p.vars[v], s, L, pos, [&](uint32_t) { S++; });
    if (S > 0xFFFFu) atomicOr(overflow, 1u);   // DgForm holds site indices as u16
    n_sites[g] = ok ? S : 0;
    uint64_t F = 0;
    if (ok) {
        F = 1;
        if (p.n_var)
            for (uint32_t k = 1; k <= p.kmax; k++) F = min((unsigned long long)(F + dg_binom(S, k)), 1ull << 62);
    }
    n_forms[g] = F;
    uint8_t rt = 0;
    if (ok && p.generate_decoys) {   // targets.contains(reversed sequence): every window's sequence is a target here
        const uint64_t h = dg_hash(s, L, true);
        uint32_t lo = 0, hi = W;
        while (lo < hi) {
            const uint32_t mid = lo + (hi - lo) / 2;
            if (hash_s[mid] < h) lo = mid + 1; else hi = mid;
        }
        for (uint32_t q = lo; q < W && hash_s[q] == h && !rt; q++) {
            const DgWin y = win[idx_s[q]];
            if (y.len != L) continue;
            uint32_t j = 0;
            while (j < L && res[y.start + j] == s[picked_pos(j, L, true)]) j++;
            rt = j == L;
        }
    }
    rev_target[g] = rt;
}

__global__ void k_dg_site_fill(const uint8_t* __restrict__ res, const DgWin* __restrict__ win, const uint32_t* __restrict__ grp_win,
                               const uint8_t* __restrict__ grp_meta, const uint32_t* __restrict__ site_off, uint32_t G, DgParams p,
                               uint32_t* __restrict__ site_code, float* __restrict__ site_mass) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    uint32_t at = site_off[g];
    if (site_off[g + 1] == at) return;
    const DgWin x = win[grp_win[g]];
    for (uint32_t v = 0; v < p.n_var; v++)
        dg_var_sites(p.vars[v], res + x.start, x.len, grp_meta[g] & 3u, [&](uint32_t code) {
            site_code[at] = code;
            site_mass[at++] = p.vars[v].mass;
        });
}

// One form's modifications, n-terminal and c-terminal masses (NaN = None) as apply + the static mods leave them (peptide.rs:136-255), at
// residue j of the FORWARD sequence. Variable sites are applied first, in combination order; a static mod then fills what is still 0.0.
struct DgFormRef {
    const uint8_t* s;   // forward sequence
    uint32_t L, pos, site0;
    const DgForm* f;
};

__device__ __forceinline__ DgFormRef dg_form_ref(const DgView& V, uint32_t form) {
    const DgForm* f = V.forms + form;
    const uint32_t g = f->group;
    const DgWin x = V.win[V.grp_win[g]];
    return DgFormRef{V.res + x.start, x.len, (uint32_t)(V.grp_meta[g] & 3u), V.site_off[g], f};
}

__device__ float dg_mod_at(const DgView& V, const DgFormRef& r, uint32_t j) {
    float v = 0.0f;
    for (uint32_t i = 0; i < r.f->n; i++) {
        const uint32_t code = V.site_code[r.site0 + r.f->sel[i]];
        if ((code >> 16) == DG_SITE_SEQ && (code & 0xFFFFu) == j && v == 0.0f) v += V.site_mass[r.site0 + r.f->sel[i]];
    }
    const bool nt = r.pos == DG_POS_NTERM || r.pos == DG_POS_FULL, ct = r.pos == DG_POS_CTERM || r.pos == DG_POS_FULL;
    const int c = r.s[j];
    for (uint32_t i = 0; i < V.p.n_static; i++) {
        const DgSpec t = V.p.statics[i];
        switch (t.kind) {
            case DG_SPEC_PROT_N:
                if (!nt) break;
                // fallthrough
            case DG_SPEC_PEP_N:
                if (t.residue >= 0 && j == 0 && c == t.residue && v == 0.0f) v += t.mass;
                break;
            case DG_SPEC_PROT_C:
                if (!ct) break;
                // fallthrough
            case DG_SPEC_PEP_C:
                if (t.residue >= 0 && j == r.L - 1 && c == t.residue && v == 0.0f) v += t.mass;
                break;
            default:
                if (c == t.residue && v == 0.0f) v = t.mass;
        }
    }
    return v;
}

__device__ void dg_terms(const DgView& V, const DgFormRef& r, float& nterm, float& cterm) {
    const float none = __int_as_float(0x7FC00000);
    nterm = cterm = none;
    for (uint32_t i = 0; i < r.f->n; i++) {
        const uint32_t code = V.site_code[r.site0 + r.f->sel[i]];
        const float m = V.site_mass[r.site0 + r.f->sel[i]];
        if ((code >> 16) == DG_SITE_N && nterm != nterm) nterm = 0.0f + m;
        if ((code >> 16) == DG_SITE_C && cterm != cterm) cterm = 0.0f + m;
    }
    const bool nt = r.pos == DG_POS_NTERM || r.pos == DG_POS_FULL, ct = r.pos == DG_POS_CTERM || r.pos == DG_POS_FULL;
    for (uint32_t i = 0; i < V.p.n_static; i++) {
        const DgSpec t = V.p.statics[i];
        if (t.residue >= 0) continue;
        if ((t.kind == DG_SPEC_PEP_N || (t.kind == DG_SPEC_PROT_N && nt)) && nterm != nterm) nterm = 0.0f + t.mass;
        if ((t.kind == DG_SPEC_PEP_C || (t.kind == DG_SPEC_PROT_C && ct)) && cterm != cterm) cterm = 0.0f + t.mass;
    }
}

// One thread per (group, combination rank): rank 0 is the unmodified peptide, then the combinations of 1..kmax sites in itertools'
// lexicographic order. A form survives no_duplicates (peptide.rs:321-333) and the inclusive mass filter; it then yields its reversed
// row (generate_decoys, unless the reversal is a target) before its forward row (unless a decoy whose sequence is a target). Pass 1
// (out == nullptr) writes the row count; pass 2 writes the rows at row_off[rank].
__global__ void k_dg_expand(DgView V, const uint64_t* __restrict__ form_off, uint32_t G, uint32_t T, const float* __restrict__ grp_base,
                            const uint32_t* __restrict__ grp_cls, const uint8_t* __restrict__ cls_target, const uint8_t* __restrict__ rev_target,
                            uint32_t* __restrict__ rows, const uint32_t* __restrict__ row_off, DgForm* __restrict__ out, float* __restrict__ out_mono) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= T) return;
    uint32_t lo = 0, hi = G;   // the group: last g with form_off[g] <= r
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (form_off[mid] <= r) lo = mid; else hi = mid;
    }
    const uint32_t g = lo, S = V.site_off[g + 1] - V.site_off[g];
    uint64_t t = r - form_off[g];
    DgForm f{};
    f.group = g;
    if (t > 0) {
        t -= 1;
        uint32_t n = 1;
        for (;; n++) {
            const uint64_t c = dg_binom(S, n);
            if (t < c) break;
            t -= c;
        }
        uint32_t x = 0;
        for (uint32_t i = 0; i < n; i++)
            for (;; x++) {
                const uint64_t c = dg_binom(S - x - 1, n - i - 1);
                if (t < c) {
                    f.sel[i] = (uint16_t)x++;
                    break;
                }
                t -= c;
            }
        f.n = (uint8_t)n;
        const uint32_t s0 = V.site_off[g];
        int nn = 0, cc = 0;
        for (uint32_t a = 0; a < n; a++) {
            const uint32_t ca = V.site_code[s0 + f.sel[a]];
            nn += (ca >> 16) == DG_SITE_N;
            cc += (ca >> 16) == DG_SITE_C;
            for (uint32_t b = a + 1; b < n; b++)
                if (V.site_code[s0 + f.sel[b]] == ca) nn = 2;
        }
        if (nn > 1 || cc > 1) {
            if (!out) rows[r] = 0;
            return;
        }
    }
    DgView W = V;
    W.forms = &f;
    const DgFormRef ref = dg_form_ref(W, 0);
    float sum = 0.0f;   // modification_mass (peptide.rs:129-133): the modifications in order, then nterm, then cterm
    for (uint32_t j = 0; j < ref.L; j++) sum += dg_mod_at(V, ref, j);
    float nterm, cterm;
    dg_terms(V, ref, nterm, cterm);
    sum = sum + (nterm == nterm ? nterm : 0.0f);
    sum = sum + (cterm == cterm ? cterm : 0.0f);
    const float mono = grp_base[g] + sum;
    uint32_t count = 0;
    bool rev = false, fwd = false;
    if (mono >= V.p.min_mass && mono <= V.p.max_mass) {
        const bool decoy = (V.grp_meta[g] >> 2) & 1u;
        rev = V.p.generate_decoys && !(!decoy && rev_target[g]);   // Peptide::reverse flips decoy: a target's reversal is a decoy
        fwd = !decoy || !cls_target[grp_cls[g]];
        count = (rev ? 1u : 0u) + (fwd ? 1u : 0u);
    }
    if (!out) {
        rows[r] = count;
        return;
    }
    uint32_t at = row_off[r];
    if (rev) {
        f.rev = 1;
        out[at] = f;
        out_mono[at++] = mono;
    }
    if (fwd) {
        f.rev = 0;
        out[at] = f;
        out_mono[at] = mono;
    }
}

// ------------------------------------------------------------------------------------------------ reorder_peptides (database.rs:221-258)
__global__ void k_dg_mono_key(const float* __restrict__ mono, uint32_t N, uint32_t* __restrict__ key, uint32_t* __restrict__ idx) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    key[i] = f32_ukey(mono[i]);   // total_cmp order
    idx[i] = i;
}

// Rows of equal-mono runs of two or more: they need initial_sort.
__global__ void k_dg_in_run(const uint32_t* __restrict__ key_s, uint32_t N, uint8_t* __restrict__ flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) flag[i] = ((i > 0 && key_s[i] == key_s[i - 1]) || (i + 1 < N && key_s[i] == key_s[i + 1])) ? 1 : 0;
}

__device__ __forceinline__ int dg_cmp_opt(float a, float b) {   // Option<f32>::partial_cmp with NaN = None: None < Some
    const bool na = a != a, nb = b != b;
    if (na || nb) return na == nb ? 0 : (na ? -1 : 1);
    return a < b ? -1 : (a > b ? 1 : 0);
}

// Peptide::initial_sort (peptide.rs:34-52) of two rows: sequence bytes, modifications by partial_cmp, length, nterm, cterm.
__device__ int dg_initial_sort(const DgView& V, uint32_t a, uint32_t b) {
    const DgFormRef ra = dg_form_ref(V, a), rb = dg_form_ref(V, b);
    const bool va = ra.f->rev, vb = rb.f->rev;
    const uint32_t n = min(ra.L, rb.L);
    for (uint32_t j = 0; j < n; j++) {
        const uint8_t x = ra.s[picked_pos(j, ra.L, va)], y = rb.s[picked_pos(j, rb.L, vb)];
        if (x != y) return x < y ? -1 : 1;
    }
    if (ra.L != rb.L) return ra.L < rb.L ? -1 : 1;
    for (uint32_t j = 0; j < n; j++) {
        const float x = dg_mod_at(V, ra, picked_pos(j, ra.L, va)), y = dg_mod_at(V, rb, picked_pos(j, rb.L, vb));
        if (x < y) return -1;
        if (x > y) return 1;
        if (!(x == y)) return 0;
    }
    float na, ca, nb, cb;
    dg_terms(V, ra, na, ca);
    dg_terms(V, rb, nb, cb);
    const int c = dg_cmp_opt(na, nb);
    return c ? c : dg_cmp_opt(ca, cb);
}

// The merge-sort order of the rows of equal-mono runs: mono (total_cmp), then initial_sort; the sort is stable, so full ties keep the
// row order, which is the reference's (DESIGN.md §14).
struct DgRowLess {
    DgView V;
    __device__ bool operator()(uint32_t a, uint32_t b) const {
        const uint32_t ka = f32_ukey(V.form_mono[a]), kb = f32_ukey(V.form_mono[b]);
        if (ka != kb) return ka < kb;
        return dg_initial_sort(V, a, b) < 0;
    }
};

__global__ void k_dg_u64_to_u32(const uint64_t* __restrict__ a, uint64_t n, uint32_t* __restrict__ b) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) b[i] = (uint32_t)a[i];
}

__global__ void k_dg_scatter(const uint32_t* __restrict__ pos, const uint32_t* __restrict__ val, uint32_t M, uint32_t* __restrict__ dst) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < M) dst[pos[i]] = val[i];
}

// reorder_peptides' merge test of adjacent rows: mono, sequence, modifications, nterm and cterm equal under IEEE ==.
__device__ bool dg_row_equal(const DgView& V, uint32_t a, uint32_t b) {
    if (!(V.form_mono[a] == V.form_mono[b])) return false;
    const DgFormRef ra = dg_form_ref(V, a), rb = dg_form_ref(V, b);
    if (ra.L != rb.L) return false;
    const bool va = ra.f->rev, vb = rb.f->rev;
    for (uint32_t j = 0; j < ra.L; j++)
        if (ra.s[picked_pos(j, ra.L, va)] != rb.s[picked_pos(j, rb.L, vb)]) return false;
    for (uint32_t j = 0; j < ra.L; j++)
        if (!(dg_mod_at(V, ra, picked_pos(j, ra.L, va)) == dg_mod_at(V, rb, picked_pos(j, rb.L, vb)))) return false;
    float na, ca, nb, cb;
    dg_terms(V, ra, na, ca);
    dg_terms(V, rb, nb, cb);
    const bool ne = (na != na && nb != nb) || na == nb, ce = (ca != ca && cb != cb) || ca == cb;
    return ne && ce;
}

__global__ void k_dg_merge_heads(DgView V, const uint32_t* __restrict__ order, uint32_t N, uint32_t* __restrict__ head) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) head[i] = (i == 0 || !dg_row_equal(V, order[i - 1], order[i])) ? 1u : 0u;
}

// Per peptide (rows [first[k], first[k + 1]) of the sorted order): residue count and protein-reference count.
__global__ void k_dg_pep_counts(DgView V, const uint32_t* __restrict__ order, const uint32_t* __restrict__ first, uint32_t n_pep,
                                const uint32_t* __restrict__ grp_start, uint64_t* __restrict__ n_res, uint64_t* __restrict__ n_ref) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_pep) return;
    uint32_t refs = 0;
    for (uint32_t i = first[k]; i < first[k + 1]; i++) {
        const uint32_t g = V.forms[order[i]].group;
        refs += grp_start[g + 1] - grp_start[g];
    }
    n_ref[k] = refs;
    n_res[k] = V.win[V.grp_win[V.forms[order[first[k]]].group]].len;
}

// The output row of each peptide: the first row's residues, modifications, terminals, mass, missed cleavages and semi flag; decoy is the
// AND over the merged rows; protein ids concatenated in row order (sorted per peptide afterwards).
__global__ void k_dg_export(DgView V, const uint32_t* __restrict__ order, const uint32_t* __restrict__ first, uint32_t n_pep,
                            const uint32_t* __restrict__ grp_start, const uint32_t* __restrict__ idx3, const uint32_t* __restrict__ prot_name,
                            const uint32_t* __restrict__ res_off, const uint32_t* __restrict__ ref_off, uint8_t* __restrict__ o_seq, float* __restrict__ o_mods,
                            float* __restrict__ o_nterm, float* __restrict__ o_cterm, float* __restrict__ o_mono, uint8_t* __restrict__ o_decoy,
                            uint8_t* __restrict__ o_missed, uint8_t* __restrict__ o_semi, uint32_t* __restrict__ o_ids) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_pep) return;
    const uint32_t r0 = order[first[k]];
    const DgFormRef r = dg_form_ref(V, r0);
    const bool rev = r.f->rev;
    const uint32_t o = res_off[k];
    for (uint32_t j = 0; j < r.L; j++) {
        const uint32_t src = picked_pos(j, r.L, rev);
        o_seq[o + j] = r.s[src];
        o_mods[o + j] = dg_mod_at(V, r, src);
    }
    float nt, ct;
    dg_terms(V, r, nt, ct);
    o_nterm[k] = nt;
    o_cterm[k] = ct;
    o_mono[k] = V.form_mono[r0];
    const DgWin w = V.win[V.grp_win[r.f->group]];
    o_missed[k] = w.missed;
    o_semi[k] = w.flags & 1u;
    bool decoy = true;
    uint32_t at = ref_off[k];
    for (uint32_t i = first[k]; i < first[k + 1]; i++) {
        const DgForm& f = V.forms[order[i]];
        const bool gd = (V.grp_meta[f.group] >> 2) & 1u;
        decoy = decoy && (f.rev ? !gd : gd);
        for (uint32_t q = grp_start[f.group]; q < grp_start[f.group + 1]; q++) o_ids[at++] = prot_name[V.win[idx3[q]].prot];
    }
    o_decoy[k] = decoy ? 1 : 0;
}

}  // namespace sb
