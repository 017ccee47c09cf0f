// lfq_oracle.cpp — CPU restatement of sage's label-free quantification (crates/sage/src/lfq.rs, isotopes.rs, mass.rs composition), the
// checker of the device path in sage_b200/csrc/lfq.cuh. TEST INFRASTRUCTURE ONLY.
//
// Written in the reference's structure (a map from (PrecursorId, decoy) to a Grid created by the first entry that reaches it) and in its
// association order; built with -ffp-contract=off and the host libm (expf, exp, pow, acos), so every f32/f64 operation is rounded as rustc
// emits it. Where the reference's order is unspecified (DashMap / rayon), the order is the one the device path defines (DESIGN.md §9):
//   * ranges before sorting: ascending (PeptideIx, charge, isotope, forward before decoy); both sorts stable;
//   * each grid cell sums its contributions in (add_ms1 call, spectrum, peak, entry, lo before hi) order.
// Tracing is single-threaded in that order; integration may use threads (grids are independent).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <thread>
#include <tuple>
#include <vector>

namespace {

constexpr float RT_TOL = 0.0050f;   // lfq.rs:15
constexpr size_t K_WIDTH = 10;      // lfq.rs:17
constexpr size_t GRID_SIZE = 100;   // lfq.rs:21
constexpr size_t N_ISOTOPES = 3;    // lfq.rs:23
constexpr float NEUTRON = 1.00335f; // mass.rs:7
constexpr size_t BIN_SIZE = 16 * 1024;
constexpr double PI = 3.141592653589793;

struct Params {   // == sage_b200_lfq_params
    int32_t peak_scoring, integration;
    double spectral_angle;
    float ppm_tolerance, mobility_pct_tolerance, peptide_q_value;
    uint8_t combine_charge_states, min_charge, max_charge;
};

struct Range {   // == sage_b200_lfq_range (PrecursorRange, lfq.rs:70-82)
    float rt, mass_lo, mass_hi, mobility_lo, mobility_hi;
    uint32_t peptide, file_id;
    uint8_t charge, isotope, decoy, pad;
};
static_assert(sizeof(Range) == 32, "Range layout");

struct Alignment { float max_rt, slope, intercept; };

// f32::total_cmp
int32_t total_key(float x) {
    int32_t b;
    memcpy(&b, &x, 4);
    return b ^ (int32_t)(((uint32_t)(b >> 31)) >> 1);
}
bool total_less(float a, float b) { return total_key(a) < total_key(b); }

// Tolerance::bounds (mass.rs:21-35)
void ppm_bounds(float lo, float hi, float c, float& out_lo, float& out_hi) {
    const float dl = c * lo / 1000000.0f, dh = c * hi / 1000000.0f;
    out_lo = c + dl;
    out_hi = c + dh;
}
void pct_bounds(float lo, float hi, float c, float& out_lo, float& out_hi) {
    const float dl = c * lo / 100.0f, dh = c * hi / 100.0f;
    out_lo = c + dl;
    out_hi = c + dh;
}

// composition (mass.rs:78-104)
void composition(uint8_t aa, uint32_t& c, uint32_t& s) {
    switch (aa) {
        case 'A': c = 3; s = 0; break;
        case 'R': c = 6; s = 0; break;
        case 'N': c = 4; s = 0; break;
        case 'D': c = 4; s = 0; break;
        case 'C': c = 3; s = 1; break;
        case 'E': c = 5; s = 0; break;
        case 'Q': c = 5; s = 0; break;
        case 'G': c = 2; s = 0; break;
        case 'H': c = 6; s = 0; break;
        case 'I': c = 6; s = 0; break;
        case 'L': c = 6; s = 0; break;
        case 'K': c = 6; s = 0; break;
        case 'M': c = 5; s = 1; break;
        case 'F': c = 9; s = 0; break;
        case 'P': c = 5; s = 0; break;
        case 'S': c = 3; s = 0; break;
        case 'T': c = 4; s = 0; break;
        case 'W': c = 11; s = 0; break;
        case 'Y': c = 9; s = 0; break;
        case 'V': c = 5; s = 0; break;
        case 'U': c = 3; s = 0; break;
        case 'O': c = 12; s = 0; break;
        default: c = 0; s = 0; break;
    }
}

// isotopes.rs:2-10
void convolve4(const float* a, const float* b, float* out) {
    out[0] = a[0] * b[0];
    out[1] = a[0] * b[1] + a[1] * b[0];
    out[2] = a[0] * b[2] + a[1] * b[1] + a[2] * b[0];
    out[3] = a[0] * b[3] + a[1] * b[2] + a[2] * b[1] + a[3] * b[0];
}
float powi(float x, int k) {   // f32::powi for k = 0..3
    float r = 1.0f;
    bool first = true;
    while (k) {
        if (k & 1) { r = first ? x : r * x; first = false; }
        k >>= 1;
        if (k) x = x * x;
    }
    return r;
}
// isotopes.rs:12-21
void carbon_isotopes(uint16_t count, float* c13) {
    const float lambda = (float)count * 0.011f;
    const float fact[4] = {1, 1, 2, 6};
    for (int k = 0; k < 4; k++) c13[k] = powi(lambda, k) * expf(-lambda) / fact[k];
}
// isotopes.rs:23-41
void sulfur_isotopes(uint16_t count, float* out) {
    const float lambda33 = (float)count * 0.0076f, lambda35 = (float)count * 0.044f;
    float s33[4];
    const float s35[4] = {powi(lambda35, 0) * expf(-lambda35), 0.0f, powi(lambda35, 1) * expf(-lambda35), 0.0f};
    const float fact[4] = {1, 1, 2, 6};
    for (int k = 0; k < 4; k++) s33[k] = powi(lambda33, k) * expf(-lambda33) / fact[k];
    convolve4(s33, s35, out);
}
// isotopes.rs:43-50
void peptide_isotopes(uint16_t carbons, uint16_t sulfurs, float* out3) {
    float c[4], s[4], cs[4];
    carbon_isotopes(carbons, c);
    sulfur_isotopes(sulfurs, s);
    convolve4(c, s, cs);
    const float mx = std::fmax(std::fmax(cs[0], cs[1]), cs[2]);
    for (int i = 0; i < 4; i++) cs[i] /= mx;
    for (int i = 0; i < 3; i++) out3[i] = cs[i];
}

// gaussian_kernel (lfq.rs:614-628)
std::vector<double> gaussian_kernel(double sigma, size_t len) {
    const double step = 2.0 / (double)(len - 1);
    const double constant = 1.0 / (sigma * std::sqrt(2.0 * PI));
    std::vector<double> k(len);
    for (size_t i = 0; i < len; i++) {
        const double x = (double)i * step - 1.0, xs = x / sigma;
        k[i] = constant * std::exp(-0.5 * (xs * xs));
    }
    double sum = 0.0;
    for (double v : k) sum += v;
    for (double& v : k) v /= sum;
    return k;
}

// convolve (lfq.rs:632-646), as written
std::vector<double> convolve(const double* slice, size_t len, const std::vector<double>& kernel) {
    const size_t n = kernel.size() - kernel.size() / 2;
    std::vector<double> out(len);
    for (size_t idx = 0; idx < len; idx++) {
        const size_t ks = kernel.size() > n + idx ? kernel.size() - (n + idx) : 0;
        const size_t ws = idx > n - 1 ? idx - (n - 1) : 0;
        const size_t m = std::min(len - ws, kernel.size() - ks);
        double acc = 0.0;
        for (size_t t = 0; t < m; t++) acc = acc + slice[ws + t] * kernel[ks + t];
        out[idx] = acc;
    }
    return out;
}

// binary_search_slice (database.rs:549-561) with a total_cmp key
template <class Key>
std::pair<size_t, size_t> binary_search_slice(size_t n, Key key, float low, float high) {
    const int32_t kl = total_key(low), kh = total_key(high);
    size_t lo = 0, hi = n;
    while (lo < hi) { size_t mid = lo + (hi - lo) / 2; if (total_key(key(mid)) < kl) lo = mid + 1; else hi = mid; }
    const size_t left = lo == 0 ? 0 : lo - 1;
    lo = left; hi = n;
    while (lo < hi) { size_t mid = lo + (hi - lo) / 2; if (total_key(key(mid)) <= kh) lo = mid + 1; else hi = mid; }
    return {left, lo};
}

// Grid (lfq.rs:307-323)
struct Grid {
    float rt_min, rt_step;
    size_t files, reference_file_id;
    float distribution[N_ISOTOPES];
    std::vector<double> matrix;   // [files * N_ISOTOPES][GRID_SIZE]
};

using Key = std::tuple<uint32_t, uint8_t, uint8_t>;   // (PeptideIx, charge or 0 for PrecursorId::Combined, decoy)

struct Oracle {
    Params p;
    size_t n_files;
    std::vector<Alignment> align;
    std::vector<Range> ranges;
    std::vector<float> min_rts;
    std::vector<uint32_t> seq_off;
    std::vector<uint8_t> seq;
    std::map<Key, Grid> scores;
};

// Grid::add_entry (lfq.rs:538-550)
void add_entry(Grid& g, float spectrum_rt, size_t isotope, size_t file_id, float intensity) {
    const float x = std::floor((spectrum_rt - g.rt_min) / g.rt_step);
    size_t bin_lo = !(x > 0.0f) ? 0 : (x >= 18446744073709551615.0f ? SIZE_MAX : (size_t)x);   // `as usize` saturates
    bin_lo = std::min(bin_lo, GRID_SIZE - 1);
    const size_t bin_hi = std::min(bin_lo + 1, GRID_SIZE - 1);
    const float bin_lo_rt = (float)bin_lo * g.rt_step + g.rt_min;
    const float interp = (spectrum_rt - bin_lo_rt) / g.rt_step;
    g.matrix[(file_id * N_ISOTOPES + isotope) * GRID_SIZE + bin_lo] += (double)((1.0f - interp) * intensity);
    g.matrix[(file_id * N_ISOTOPES + isotope) * GRID_SIZE + bin_hi] += (double)(interp * intensity);
}

struct Result {
    bool present = false;
    uint32_t rt = 0;
    double spectral_angle = 0.0, score = 0.0, margin = INFINITY;
    std::vector<double> areas;
};

// relative distance of two compared values; only comparisons whose outcome can move with acos() count (DESIGN.md §9). Two exact zeros are
// not a near-tie: a score or spectral value that is exactly 0 does not come from acos (a zero rt factor, or no signal in the column).
void note(double& margin, double a, double b) {
    const double d = std::fabs(a - b), m = std::max(std::fabs(a), std::fabs(b));
    if (m > 0.0) margin = std::min(margin, d / m);
}

// summarize_traces (lfq.rs:558-610) + Traces::integrate (lfq.rs:447-509)
Result integrate_grid(const Grid& grid, const Params& s, const std::vector<double>& k) {
    const size_t F = grid.files, C = GRID_SIZE;
    std::vector<double> sa(F * C, 0.0), dot(F * C, 0.0);
    const double ss_dist = (double)std::sqrt(grid.distribution[0] * grid.distribution[0] + grid.distribution[1] * grid.distribution[1] +
                                             grid.distribution[2] * grid.distribution[2]);
    for (size_t file = 0; file < F; file++) {
        std::vector<double> ssi(C, 0.0);
        for (size_t iso = 0; iso < N_ISOTOPES; iso++) {
            const std::vector<double> conv = convolve(grid.matrix.data() + (file * N_ISOTOPES + iso) * C, C, k);
            for (size_t col = 0; col < C; col++) {
                sa[file * C + col] += conv[col] * (double)grid.distribution[iso];
                ssi[col] += conv[col] * conv[col];
            }
        }
        for (size_t col = 0; col < C; col++) {
            const double d = sa[file * C + col];
            const double sim = ssi[col] > 0.0 ? d / (std::sqrt(ssi[col]) * ss_dist) : 0.0;
            sa[file * C + col] = 1.0 - 2.0 * std::acos(sim) / PI;
            dot[file * C + col] = d;
        }
    }
    // find_time_warps (lfq.rs:361-385) against the reference file, then apply_time_warps (lfq.rs:388-400)
    std::vector<long> warps(F, 0);
    const double* ref = dot.data() + grid.reference_file_id * C;
    for (size_t row = 0; row < F; row++) {
        const double* run = dot.data() + row * C;
        long best_off = 0;
        double best = 0.0;
        for (long off = -75; off <= 75; off++) {
            double d = 0.0;
            for (size_t i = 0; i < C; i++) {
                const long j = (long)i + off;
                if (j >= 0 && j < (long)C) d += ref[i] * run[j];
            }
            if (d >= best) { best_off = off; best = d; }
        }
        warps[row] = best_off;
    }
    for (std::vector<double>* m : {&sa, &dot})
        for (size_t row = 0; row < F; row++) {
            std::vector<double> shifted(C, 0.0);
            for (size_t i = 0; i < C; i++) {
                const long j = (long)i + warps[row];
                if (j >= 0 && j < (long)C) shifted[i] = (*m)[row * C + j];
            }
            std::copy(shifted.begin(), shifted.end(), m->begin() + row * C);
        }
    // scores (lfq.rs:402-437); acos_dep[col]: the column's spectral value depends on acos (some dot product is non-zero)
    std::vector<double> spectral(C), intensity(C), scores(C);
    std::vector<bool> acos_dep(C, false);
    double mx = 0.0;
    for (size_t col = 0; col < C; col++) {
        double summed = 1.0, weighted = 0.0;
        for (size_t f = 0; f < F; f++) {
            weighted += sa[f * C + col] * dot[f * C + col];
            summed += dot[f * C + col];
            if (dot[f * C + col] != 0.0) acos_dep[col] = true;
        }
        spectral[col] = weighted / summed;
        intensity[col] = summed;
        mx = std::fmax(mx, summed);
    }
    const long center = (long)C / 2;
    for (size_t col = 0; col < C; col++) {
        const double rt = 1.0 - ((double)std::labs((long)col - center) / (double)center);
        const double sp = spectral[col];
        switch (s.peak_scoring) {
            case 0: scores[col] = std::pow(rt, 0.33); break;
            case 1: scores[col] = sp; break;
            case 2: scores[col] = std::sqrt(intensity[col] / mx); break;
            default: scores[col] = sp * (sp * sp) * std::pow(rt, 0.33) * std::sqrt(intensity[col] / mx); break;
        }
    }
    const bool score_dep = s.peak_scoring == 1 || s.peak_scoring == 3;
    Result r;
    double best = 0.0;
    size_t brt = 0;
    bool best_dep = false;
    for (size_t col = 0; col < C; col++) {
        const bool sa_ok = spectral[col] >= s.spectral_angle;
        if (sa_ok && ((score_dep && acos_dep[col]) || best_dep)) note(r.margin, scores[col], best);
        if (scores[col] > best && acos_dep[col]) note(r.margin, spectral[col], s.spectral_angle);
        if (scores[col] > best && sa_ok) { best = scores[col]; brt = col; best_dep = score_dep && acos_dep[col]; }
    }
    if (best == 0.0) return r;
    size_t left = brt > 0 ? brt - 1 : 0, right = brt + 1;
    const double threshold = best * 0.50;
    const size_t llim = brt > C / 5 ? brt - C / 5 : 0, rlim = std::min(C - 1, brt + 20);
    auto edge = [&](size_t i) {   // the walk's tests at i
        if (score_dep && (acos_dep[i] || best_dep)) note(r.margin, scores[i], threshold);
        if (acos_dep[i]) note(r.margin, spectral[i], s.spectral_angle);
    };
    while (left > llim) {
        edge(left);
        if (!(scores[left] >= threshold && spectral[left] >= s.spectral_angle)) break;
        left -= 1;
    }
    while (right < rlim) {
        edge(right);
        if (!(scores[right] >= threshold && spectral[right] >= s.spectral_angle)) break;
        right += 1;
    }
    r.areas.resize(F);
    for (size_t f = 0; f < F; f++) {
        if (s.integration == 1) {
            double a = 0.0;
            for (size_t i = left; i < right; i++) a += dot[f * C + i];
            r.areas[f] = a;
        } else {
            r.areas[f] = dot[f * C + brt];
        }
    }
    double summed = 1.0, weighted = 0.0;
    for (size_t f = 0; f < F; f++) {
        weighted += sa[f * C + brt] * dot[f * C + brt];
        summed += dot[f * C + brt];
    }
    r.present = true;
    r.rt = (uint32_t)brt;
    r.score = best;
    r.spectral_angle = weighted / summed;
    return r;
}

}  // namespace

extern "C" {

void lo_peptide_isotopes(uint16_t carbons, uint16_t sulfurs, float* out3) { peptide_isotopes(carbons, sulfurs, out3); }

// build_feature_map (lfq.rs:94-193)
void* lo_create(const Params* p, uint64_t n, const uint32_t* peptide_idx, const float* peptide_q, const int32_t* label, const float* aligned_rt,
                const float* calcmass, const uint32_t* file_id, const float* ims, uint64_t n_files, const float* alignments, uint64_t n_peptides,
                const uint32_t* seq_off, const uint8_t* seq) {
    Oracle* o = new Oracle();
    o->p = *p;
    o->n_files = n_files;
    for (uint64_t f = 0; f < n_files; f++) o->align.push_back({alignments[3 * f], alignments[3 * f + 1], alignments[3 * f + 2]});
    o->seq_off.assign(seq_off, seq_off + n_peptides + 1);
    o->seq.assign(seq, seq + seq_off[n_peptides]);
    std::map<uint32_t, Range> map;   // ordered: the pre-sort order is ascending PeptideIx
    for (uint64_t i = 0; i < n; i++) {
        if (!(peptide_q[i] <= p->peptide_q_value && label[i] == 1)) continue;
        if (map.count(peptide_idx[i])) continue;
        Range r{};
        pct_bounds(-p->mobility_pct_tolerance, p->mobility_pct_tolerance, ims[i], r.mobility_lo, r.mobility_hi);
        r.rt = aligned_rt[i];
        r.mass_lo = calcmass[i];
        r.mass_hi = 0.0f;
        r.peptide = peptide_idx[i];
        r.file_id = file_id[i];
        map[peptide_idx[i]] = r;
    }
    for (const auto& kv : map) {
        const Range& range = kv.second;
        for (uint32_t charge = p->min_charge; charge <= p->max_charge; charge++)
            for (uint32_t isotope = 0; isotope < N_ISOTOPES; isotope++) {
                const float mass = (range.mass_lo + (float)isotope * NEUTRON) / (float)charge;
                Range fwd = range;
                ppm_bounds(-p->ppm_tolerance, p->ppm_tolerance, mass, fwd.mass_lo, fwd.mass_hi);
                fwd.charge = (uint8_t)charge;
                fwd.isotope = (uint8_t)isotope;
                fwd.decoy = 0;
                Range rev = fwd;
                ppm_bounds(-p->ppm_tolerance, p->ppm_tolerance, mass + 11.06f, rev.mass_lo, rev.mass_hi);
                rev.rt = std::fmax(fwd.rt - RT_TOL * 2.0f, 0.0f);
                rev.decoy = 1;
                o->ranges.push_back(fwd);
                o->ranges.push_back(rev);
            }
    }
    std::stable_sort(o->ranges.begin(), o->ranges.end(), [](const Range& a, const Range& b) { return total_less(a.rt, b.rt); });
    for (size_t c = 0; c < o->ranges.size(); c += BIN_SIZE) {
        const size_t e = std::min(c + BIN_SIZE, o->ranges.size());
        o->min_rts.push_back(o->ranges[c].rt);
        std::stable_sort(o->ranges.begin() + c, o->ranges.begin() + e, [](const Range& a, const Range& b) { return total_less(a.mass_lo, b.mass_lo); });
    }
    return o;
}

void lo_destroy(void* h) { delete (Oracle*)h; }
uint64_t lo_n_ranges(void* h) { return ((Oracle*)h)->ranges.size(); }
uint64_t lo_n_pages(void* h) { return ((Oracle*)h)->min_rts.size(); }
uint64_t lo_n_grids(void* h) { return ((Oracle*)h)->scores.size(); }

void lo_export_map(void* h, void* ranges, float* min_rts) {
    Oracle* o = (Oracle*)h;
    if (ranges) memcpy(ranges, o->ranges.data(), sizeof(Range) * o->ranges.size());
    if (min_rts) memcpy(min_rts, o->min_rts.data(), 4 * o->min_rts.size());
}

// the grids in (id, decoy) order: keys [n][3] (peptide, charge, decoy) and matrices [n][files * 3 * 100]
void lo_export_grids(void* h, uint32_t* keys, double* matrices) {
    Oracle* o = (Oracle*)h;
    size_t i = 0;
    for (const auto& kv : o->scores) {
        keys[3 * i] = std::get<0>(kv.first);
        keys[3 * i + 1] = std::get<1>(kv.first);
        keys[3 * i + 2] = std::get<2>(kv.first);
        if (matrices) memcpy(matrices + i * kv.second.matrix.size(), kv.second.matrix.data(), 8 * kv.second.matrix.size());
        i++;
    }
}

// the tracing loop of FeatureMap::quantify (lfq.rs:239-287) over one batch, spectra and peaks in order
void lo_add_ms1(void* h, uint64_t n, const uint64_t* peak_off, const float* masses, const float* intensities, const uint32_t* file_id, const float* sst,
                const float* mobilities) {
    Oracle* o = (Oracle*)h;
    const std::vector<double> unused;
    for (uint64_t s = 0; s < n; s++) {
        const Alignment a = o->align[file_id[s]];
        const float rt = (sst[s] / a.max_rt) * a.slope + a.intercept;
        // rt_slice (lfq.rs:205-221)
        const auto pages = binary_search_slice(o->min_rts.size(), [&](size_t i) { return o->min_rts[i]; }, rt - RT_TOL, rt + RT_TOL);
        const float min_rt = rt - RT_TOL, max_rt = rt + RT_TOL;
        for (uint64_t pk = peak_off[s]; pk < peak_off[s + 1]; pk++) {
            const float mass = masses[pk], intensity = intensities[pk];
            // Query::mass_lookup (lfq.rs:649-675) / mass_mobility_lookup (lfq.rs:677-686)
            for (size_t page = pages.first; page < pages.second; page++) {
                const size_t left_idx = page * BIN_SIZE, right_idx = std::min(left_idx + BIN_SIZE, o->ranges.size());
                const Range* slice = o->ranges.data() + left_idx;
                const auto inner = binary_search_slice(right_idx - left_idx, [&](size_t i) { return slice[i].mass_lo; }, mass - 0.1f, mass + 0.1f);
                for (size_t i = inner.first; i < inner.second; i++) {
                    const Range& e = slice[i];
                    if (!(e.rt <= max_rt && e.rt >= min_rt && mass >= e.mass_lo && mass <= e.mass_hi)) continue;
                    if (mobilities && !(e.mobility_hi >= mobilities[pk] && e.mobility_lo <= mobilities[pk])) continue;
                    // add_entry closure (lfq.rs:244-265)
                    const Key key{e.peptide, o->p.combine_charge_states ? (uint8_t)0 : e.charge, e.decoy};
                    auto it = o->scores.find(key);
                    if (it == o->scores.end()) {
                        Grid g;
                        uint32_t carbon = 0, sulfur = 0;
                        for (uint32_t r = o->seq_off[e.peptide]; r < o->seq_off[e.peptide + 1]; r++) {
                            uint32_t c, su;
                            composition(o->seq[r], c, su);
                            carbon += c;
                            sulfur += su;
                        }
                        peptide_isotopes((uint16_t)carbon, (uint16_t)sulfur, g.distribution);
                        // Grid::new (lfq.rs:513-535)
                        g.rt_step = (RT_TOL * 2.0f) / (float)GRID_SIZE;
                        g.rt_min = e.rt - RT_TOL;
                        g.files = o->n_files;
                        g.reference_file_id = e.file_id;
                        g.matrix.assign(GRID_SIZE * o->n_files * N_ISOTOPES, 0.0);
                        it = o->scores.emplace(key, std::move(g)).first;
                    }
                    add_entry(it->second, rt, e.isotope, file_id[s], intensity);
                }
            }
        }
    }
}

// summarize_traces + integrate for every grid, in (id, decoy) order, with `threads` workers. Returns the number of grids (rows of the outputs);
// present[i] == 0 where integrate returned None. margin[i]: smallest relative gap of an acos-dependent decision of grid i (inf: none).
uint64_t lo_integrate(void* h, int threads, uint32_t* keys, uint8_t* present, uint32_t* rt, double* spectral_angle, double* score, double* areas,
                      double* margin) {
    Oracle* o = (Oracle*)h;
    std::vector<const std::pair<const Key, Grid>*> items;
    for (const auto& kv : o->scores) items.push_back(&kv);
    const std::vector<double> k = gaussian_kernel(0.5, K_WIDTH);
    const size_t n = items.size(), F = o->n_files;
    auto work = [&](size_t a, size_t b) {
        for (size_t i = a; i < b; i++) {
            const Result r = integrate_grid(items[i]->second, o->p, k);
            keys[3 * i] = std::get<0>(items[i]->first);
            keys[3 * i + 1] = std::get<1>(items[i]->first);
            keys[3 * i + 2] = std::get<2>(items[i]->first);
            present[i] = r.present;
            rt[i] = r.rt;
            spectral_angle[i] = r.spectral_angle;
            score[i] = r.score;
            margin[i] = r.margin;
            for (size_t f = 0; f < F; f++) areas[i * F + f] = r.present ? r.areas[f] : 0.0;
        }
    };
    const size_t T = (size_t)std::max(1, threads);
    std::vector<std::thread> pool;
    for (size_t t = 0; t < T; t++) pool.emplace_back(work, n * t / T, n * (t + 1) / T);
    for (auto& th : pool) th.join();
    return n;
}

}  // extern "C"
