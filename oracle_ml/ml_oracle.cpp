// ml_oracle.cpp — CPU restatement of Sage's PSM rescoring, the authority the device path (sage_b200/csrc/fdr.cuh) is tested against.
//
// Restates, from the reference sources (crates/sage/src/ml/ and crates/sage-cli/src/runner.rs):
//   linear_discriminant.rs:63-231   LinearDiscriminantAnalysis::train / score, score_psms
//   kde.rs:14-169                   Kde, Builder::build, Estimator::posterior_error
//   gauss.rs:26-165, matrix.rs      Gauss::solve with its eps ladder, on a row-major matrix
//   ml/mod.rs:24-32                 mean, std
//   qvalue.rs:8-36                  spectrum_q_value
//   runner.rs:280-291               spectrum_fdr: score_psms, the heuristic fallback, the descending sort
// with host libm (exp, log1p, log10, log1pf, pow, sqrt) and -ffp-contract=off, in the orders DESIGN.md §10 defines where the reference leaves
// them to rayon: Kde::pdf folds chunks of KDE_CHUNK samples from 0.0 and adds the chunk sums in order from -0.0; the unstable sort breaks ties
// by input row. f64 Sum starts from -0.0 (the neutral element of current Rust's `impl Sum for f64`). Shares no code with the library.
//
// Also restates the runner's predict_rt stage (runner.rs:513-531), the authority for sage_b200/csrc/rt.cuh:
//   retention_alignment.rs  global_alignment
//   regression.rs           LinearRegression::fit
//   retention_model.rs      RetentionModel::embed / fit / predict
//   mobility_model.rs       MobilityModel::embed / fit / predict
// in the orders DESIGN.md §11 defines: poisson ties by input row, ordered maps (ascending PeptideIx, ascending file), fit chunks of RT_CHUNK
// training rows merged in order.
//
// Also restates fdr.rs:16-287 (Competition::assign_q_value, picked_peptide, picked_protein, picked_precursor) with real key strings:
// Peptide::reverse and Display (peptide.rs:307-318, 390-406) written out with Rust's shortest round-trip f32 formatting, and
// insertion-ordered maps, in the definitions of DESIGN.md §12.
//
// Also restates protein_grouping.rs (generate_protein_groups, the literal BipartiteGraph loop) and fdr.rs:192-226 (picked_protein_group)
// with real name strings, in the definitions of DESIGN.md §13.
#include <algorithm>
#include <charconv>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <regex>
#include <set>
#include <string>
#include <unordered_map>
#include <thread>
#include <vector>

namespace {

constexpr uint64_t KDE_CHUNK = 4096;
constexpr int D = 20;

// The Feature fields rescoring reads, laid out as the search returns them (128 bytes per row).
struct Row {
    uint32_t spectrum, peptide_idx, peptide_len, rank;
    int32_t label;
    float expmass, calcmass;
    uint32_t charge;
    float rt, ims, delta_mass, isotope_error, average_ppm;
    uint32_t pad0;
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
static_assert(sizeof(Row) == 128, "Feature row layout");

double rust_sum(const double* x, uint64_t n) {   // Iterator::sum::<f64>()
    double s = -0.0;
    for (uint64_t i = 0; i < n; i++) s += x[i];
    return s;
}

struct Kde {   // kde.rs:14-49
    std::vector<double> sample;
    double bandwidth = 0, constant = 0;
    Kde(std::vector<double> s, double bw_factor) : sample(std::move(s)) {
        const double n = (double)sample.size();
        const double mean = rust_sum(sample.data(), sample.size()) / n;   // ml/mod.rs:24-26
        double acc = 0.0;
        for (double x : sample) acc = acc + (x - mean) * (x - mean);      // ml/mod.rs:28-32 (powi(2) is x * x)
        const double sigma = std::sqrt(acc / n);
        bandwidth = (sigma * std::pow((4.0 / 3.0) / n, 1.0 / 5.0)) * bw_factor;
        constant = std::sqrt(2.0 * M_PI) * bandwidth * n;
    }
    double pdf(double x) const {
        double total = -0.0;
        for (uint64_t c0 = 0; c0 < sample.size(); c0 += KDE_CHUNK) {
            double acc = 0.0;
            const uint64_t c1 = std::min<uint64_t>(sample.size(), c0 + KDE_CHUNK);
            for (uint64_t i = c0; i < c1; i++) {
                const double u = (x - sample[i]) / bandwidth;
                acc = acc + std::exp(-0.5 * (u * u));
            }
            total += acc;
        }
        return total / constant;
    }
};

struct Estimator {   // kde.rs:139-169
    std::vector<double> bins;
    double min_score = 0, score_step = 0;
    double posterior_error(double score) const {
        const double t = std::floor((score - min_score) / score_step);
        uint64_t lo = !(t >= 0.0) ? 0 : (t >= 18446744073709551616.0 ? UINT64_MAX : (uint64_t)t);   // `as usize` saturates
        const uint64_t last = bins.empty() ? 0 : bins.size() - 1;
        lo = std::min(last, lo);
        const uint64_t hi = std::min(last, lo + 1);
        const double lower = bins[lo], upper = bins[hi];
        const double lo_score = (double)lo * score_step + min_score;
        const double linear = (score - lo_score) / score_step;
        return lower + (upper - lower) * linear;
    }
};

Estimator kde_build(const double* scores, const uint8_t* decoy, uint64_t n, uint64_t bins, bool monotonic, double bw_factor, int threads) {
    std::vector<double> d, t;
    for (uint64_t i = 0; i < n; i++) (decoy[i] ? d : t).push_back(scores[i]);
    const double pi = (double)d.size() / (double)n;
    const Kde kd(std::move(d), bw_factor), kt(std::move(t), bw_factor);
    Estimator e;
    double mn = 1.7976931348623157e308, mx = -1.7976931348623157e308;
    for (uint64_t i = 0; i < n; i++) { mn = std::fmin(mn, scores[i]); mx = std::fmax(mx, scores[i]); }
    e.min_score = mn;
    e.score_step = (mx - mn) / (double)(bins - 1);
    e.bins.assign(bins, 0.0);
    auto work = [&](int w) {   // bins are independent; each one is evaluated in the defined order
        for (uint64_t b = (uint64_t)w; b < bins; b += (uint64_t)threads) {
            const double score = (double)b * e.score_step + mn;
            const double dec = kd.pdf(score) * pi;
            const double tar = kt.pdf(score) * (1.0 - pi);
            e.bins[b] = dec / (tar + dec);
        }
    };
    std::vector<std::thread> pool;
    for (int w = 0; w < threads; w++) pool.emplace_back(work, w);
    for (auto& th : pool) th.join();
    if (monotonic) {
        double acc = e.bins.back();
        for (uint64_t i = bins; i-- > 0;) { acc = std::fmax(acc, e.bins[i]); e.bins[i] = acc; }
    }
    return e;
}

struct Mat {   // matrix.rs (row-major)
    int rows, cols;
    std::vector<double> a;
    Mat(int r, int c) : rows(r), cols(c), a((size_t)r * c, 0.0) {}
    double& at(int i, int j) { return a[(size_t)i * cols + j]; }
};

bool solve_inner(Mat l, Mat r, double eps, std::vector<double>* x) {   // gauss.rs:27-40
    const int m = l.rows, n = l.cols;
    for (int i = 0; i < n; i++) l.at(i, i) += eps;
    int h = 0, k = 0;
    while (h < m && k < n) {   // echelon, gauss.rs:85-124
        std::pair<int, double> best(0, -1.7976931348623157e308);
        for (int i = h; i < m; i++)
            if (l.at(i, k) >= best.second) best = {i, l.at(i, k)};
        const int i = best.first;
        if (l.at(i, k) == 0.0) { k++; continue; }
        if (h != i) {
            for (int c = 0; c < l.cols; c++) std::swap(l.at(h, c), l.at(i, c));
            for (int c = 0; c < r.cols; c++) std::swap(r.at(h, c), r.at(i, c));
        }
        for (int i2 = h + 1; i2 < m; i2++) {
            const double f = l.at(i2, k) / l.at(h, k);
            l.at(i2, k) = 0.0;
            for (int j = k + 1; j < n; j++) l.at(i2, j) -= l.at(h, j) * f;
            for (int j = 0; j < r.cols; j++) r.at(i2, j) -= r.at(h, j) * f;
        }
        h++;
        k++;
    }
    for (int i = l.rows - 1; i >= 0; i--) {   // reduce, gauss.rs:127-143
        for (int j = 0; j < l.cols; j++) {
            const double x0 = l.at(i, j);
            if (x0 == 0.0) continue;
            for (int c = j; c < l.cols; c++) l.at(i, c) /= x0;
            for (int c = 0; c < r.cols; c++) r.at(i, c) /= x0;
            break;
        }
    }
    for (int i = l.rows - 1; i >= 0; i--) {   // backfill, gauss.rs:146-164
        for (int j = 0; j < l.cols; j++) {
            if (l.at(i, j) == 0.0) continue;
            for (int k2 = 0; k2 < i; k2++) {
                const double f = l.at(k2, j) / l.at(i, j);
                for (int c = 0; c < l.cols; c++) l.at(k2, c) -= l.at(i, c) * f;
                for (int c = 0; c < r.cols; c++) r.at(k2, c) -= r.at(i, c) * f;
            }
            break;
        }
    }
    for (int i = 0; i < n; i++)   // left_solved, gauss.rs:66-83
        for (int j = 0; j < n; j++) {
            const double v = l.at(i, j);
            if (i == j) { if (v != 1.0 && v != 0.0) return false; }
            else if (v > 1e-8) return false;
        }
    *x = r.a;
    return true;
}

// LinearDiscriminantAnalysis::train (linear_discriminant.rs:63-124) over a row-major [n][dim] matrix. Returns 1 when a solution was found (coef
// and eps filled), 0 for None (an empty class or every eps failing).
int lda_train(const double* X, const uint8_t* decoy, uint64_t n, int dim, double* coef, double* eps_out) {
    std::vector<double> sum(2 * dim, 0.0), mean(2 * dim);
    uint64_t count[2] = {0, 0};
    for (uint64_t i = 0; i < n; i++) {
        const int c = decoy[i] ? 0 : 1;
        for (int j = 0; j < dim; j++) sum[c * dim + j] += X[i * dim + j];
        count[c]++;
    }
    if (count[0] == 0 || count[1] == 0) return 0;
    for (int c = 0; c < 2; c++)
        for (int j = 0; j < dim; j++) mean[c * dim + j] = sum[c * dim + j] / (double)count[c];
    std::vector<Mat> S(2, Mat(dim, dim));
    std::vector<double> cen(dim);
    for (uint64_t i = 0; i < n; i++) {
        const int c = decoy[i] ? 0 : 1;
        for (int j = 0; j < dim; j++) cen[j] = X[i * dim + j] - mean[c * dim + j];
        for (int j = 0; j < dim; j++)
            for (int k = 0; k < dim; k++) S[c].at(j, k) += cen[j] * cen[k];
    }
    Mat sw(dim, dim), rhs(dim, 1);
    for (int c = 0; c < 2; c++)
        for (size_t e = 0; e < sw.a.size(); e++) sw.a[e] += S[c].a[e] / (double)count[c];
    for (int j = 0; j < dim; j++) rhs.a[j] = mean[dim + j] - mean[j];
    std::vector<double> x;
    for (double eps = 1e-8; eps <= 1.0; eps *= 10.0)   // Gauss::solve, gauss.rs:42-51
        if (solve_inner(sw, rhs, eps, &x)) {
            std::copy(x.begin(), x.end(), coef);
            *eps_out = eps;
            return 1;
        }
    return 0;
}

double clamp_sqrt(double v) {   // f64::clamp(0.001, 0.999).sqrt()
    if (v < 0.001) v = 0.001;
    if (v > 0.999) v = 0.999;
    return std::sqrt(v);
}

}  // namespace

namespace {

constexpr uint64_t RT_CHUNK = 1024;
const char VALID_AA[] = "ACDEFGHIKLMNPQRSTVWYUO";   // mass.rs:59-62
constexpr size_t N_AA = 22;
constexpr int RT_D = 22 * 3 + 3, IMS_D = 22 * 4 + 12;

struct AaMap {   // retention_model.rs:64-67: letters outside VALID_AA keep the map's initial 0
    size_t m[26];
    AaMap() {
        for (size_t& v : m) v = 0;
        for (size_t i = 0; i < N_AA; i++) m[VALID_AA[i] - 'A'] = i;
    }
};
const AaMap AA;

// retention_model.rs:42-59
void rt_embed(const uint8_t* seq, size_t len, float mono, double* e) {
    const size_t NT = N_AA, CT = N_AA * 2, LEN = RT_D - 3, MASS = RT_D - 2, ICPT = RT_D - 1;
    std::fill(e, e + RT_D, 0.0);
    const size_t cterm = len >= 3 ? len - 3 : 0;
    for (size_t i = 0; i < len; i++) {
        const size_t idx = AA.m[seq[i] - 'A'];
        e[idx] += 1.0;
        if (i == 0 || i == 1) e[NT + idx] += 1.0;
        else if (i == cterm || i == cterm + 1) e[CT + idx] += 1.0;
    }
    e[LEN] = (double)len;
    e[MASS] = std::log1p((double)mono);
    e[ICPT] = 1.0;
}

bool contains(const size_t* set, size_t n, size_t x) {
    for (size_t i = 0; i < n; i++)
        if (set[i] == x) return true;
    return false;
}

// mobility_model.rs:97-149, the group constants as letter offsets compared with the VALID_AA position, as written
void ims_embed(const uint8_t* seq, size_t len, float mono, uint8_t charge, double* e) {
    const size_t F = IMS_D, PCT = N_AA, NT = N_AA * 2, CT = N_AA * 3;
    const size_t BULKY[6] = {'L' - 'A', 'V' - 'A', 'I' - 'A', 'F' - 'A', 'W' - 'A', 'Y' - 'A'};
    const size_t UC_POLAR[4] = {'S' - 'A', 'T' - 'A', 'N' - 'A', 'Q' - 'A'};
    const size_t POSITIVE[3] = {'R' - 'A', 'K' - 'A', 'H' - 'A'};
    const size_t NEGATIVE[2] = {'D' - 'A', 'E' - 'A'};
    const size_t TINY[3] = {'G' - 'A', 'A' - 'A', 'S' - 'A'};
    const size_t BRANCHED[3] = {'L' - 'A', 'I' - 'A', 'V' - 'A'};
    std::fill(e, e + IMS_D, 0.0);
    const size_t cterm = len >= 3 ? len - 3 : 0;
    const double pep_length = (double)len;
    for (size_t i = 0; i < len; i++) {
        const size_t idx = AA.m[seq[i] - 'A'];
        e[idx] += 1.0;
        if (i == 0 || i == 1) e[NT + idx] += 1.0;
        else if (i > cterm) e[CT + idx] += 1.0;
        if (contains(BULKY, 6, idx)) e[F - 9] += 1.0;
        if (contains(UC_POLAR, 4, idx)) e[F - 10] += 1.0;
        if (contains(POSITIVE, 3, idx)) e[F - 8] += 1.0;
        if (contains(NEGATIVE, 2, idx)) e[F - 7] += 1.0;
        if (contains(TINY, 3, idx)) e[F - 11] += 1.0;
        if (contains(BRANCHED, 3, idx)) e[F - 12] += 1.0;
    }
    for (size_t idx = 0; idx < N_AA; idx++) e[PCT + idx] = e[idx] / pep_length;
    const double z = (double)charge;
    e[F - 5] = z;
    e[F - 6] = 1. / z;
    e[F - 3] = (double)len;
    e[F - 2] = (double)mono / 1000.0;
    e[F - 4] = ((double)mono / z) / 1000.0;
    e[F - 1] = 1.0;
}

struct Fit {
    bool ok = false;
    std::vector<double> beta;
    double r2 = 0, eps = 0;
};

// regression.rs:72-117 over items 0..n (already filtered), embed(i, row) and target(i). The rayon fold/reduce is chunks of RT_CHUNK items, each
// from Acc::zero, merged as ((0 + A_0) + A_1) + ...; the SSE sum is chunk sums from -0.0 added in order from -0.0. Chunks run on `threads`.
template <class Embed, class Target>
Fit linreg_fit(uint64_t n, int d, Embed embed, Target target, int threads) {
    Fit out;
    if (n == 0) return out;
    const uint64_t chunks = (n + RT_CHUNK - 1) / RT_CHUNK;
    const size_t acc_len = (size_t)d * d + d + 2;
    std::vector<double> part(chunks * acc_len, 0.0);
    auto run = [&](auto&& body) {
        std::vector<std::thread> pool;
        for (int w = 0; w < threads; w++)
            pool.emplace_back([&, w]() {
                for (uint64_t c = (uint64_t)w; c < chunks; c += (uint64_t)threads) body(c);
            });
        for (auto& t : pool) t.join();
    };
    run([&](uint64_t c) {   // Acc::add_row over the chunk, the full d x d product as written
        double* acc = &part[c * acc_len];
        double *cov = acc, *b = acc + (size_t)d * d;
        std::vector<double> row(d);
        for (uint64_t i = c * RT_CHUNK; i < std::min(n, (c + 1) * RT_CHUNK); i++) {
            embed(i, row.data());
            const double y = target(i);
            for (int j = 0; j < d; j++) {
                const double rj = row[j];
                b[j] += rj * y;
                for (int k = 0; k < d; k++) cov[(size_t)j * d + k] += rj * row[k];
            }
            acc[acc_len - 2] += y;
            acc[acc_len - 1] += y * y;
        }
    });
    std::vector<double> tot(acc_len, 0.0);
    for (uint64_t c = 0; c < chunks; c++)
        for (size_t a = 0; a < acc_len; a++) tot[a] += part[c * acc_len + a];
    const double nf = (double)n, y_mean = tot[acc_len - 2] / nf, y_var = tot[acc_len - 1] - nf * y_mean * y_mean;
    Mat cov(d, d), rhs(d, 1);
    std::copy(tot.begin(), tot.begin() + (size_t)d * d, cov.a.begin());
    std::copy(tot.begin() + (size_t)d * d, tot.begin() + (size_t)d * d + d, rhs.a.begin());
    std::vector<double> beta;
    for (double eps = 1e-8; eps <= 1.0; eps *= 10.0)   // Gauss::solve
        if (solve_inner(cov, rhs, eps, &beta)) {
            out.ok = true;
            out.eps = eps;
            break;
        }
    if (!out.ok) return out;
    std::vector<double> csse(chunks);
    run([&](uint64_t c) {
        std::vector<double> row(d);
        double s = -0.0;
        for (uint64_t i = c * RT_CHUNK; i < std::min(n, (c + 1) * RT_CHUNK); i++) {
            embed(i, row.data());
            double pred = -0.0;
            for (int j = 0; j < d; j++) pred += row[j] * beta[j];
            const double diff = pred - target(i);
            s += diff * diff;
        }
        csse[c] = s;
    });
    double sse = -0.0;
    for (double v : csse) sse += v;
    out.r2 = 1.0 - sse / y_var;
    out.beta = beta;
    return out;
}

double rust_min(double a, double b) {   // f64::min; -0.0 kept over +0.0
    if (std::isnan(a)) return b;
    if (std::isnan(b)) return a;
    if (a < b) return a;
    if (b < a) return b;
    return std::signbit(a) ? a : b;
}

uint32_t ceil_as_u32(float rt) {   // `rt.ceil() as u32`, saturating
    const float c = std::ceil(rt);
    if (!(c >= 0.0f)) return 0;
    if (c >= 4294967296.0f) return UINT32_MAX;
    return (uint32_t)c;
}

}  // namespace

extern "C" {

int mo_kde_build(const double* scores, const uint8_t* decoy, uint64_t n, uint64_t bins, int monotonic, double bw_factor, int threads, double* out_bins,
                 double* min_score, double* score_step) {
    const Estimator e = kde_build(scores, decoy, n, bins, monotonic != 0, bw_factor, std::max(1, threads));
    std::copy(e.bins.begin(), e.bins.end(), out_bins);
    *min_score = e.min_score;
    *score_step = e.score_step;
    return 0;
}

int mo_lda_train(const double* X, const uint8_t* decoy, uint64_t n, int dim, double* coef, double* eps) {
    return lda_train(X, decoy, n, dim, coef, eps);
}

double mo_lda_score(const double* coef, const double* row, int dim) {   // LinearDiscriminantAnalysis::score
    double s = -0.0;
    for (int j = 0; j < dim; j++) s += coef[j] * row[j];
    return s;
}

// runner.rs:280-291. kind 0 = Ppm, 2 = Da. Any of the three columns may be NULL (Feature defaults). Outputs as sage_b200_spectrum_fdr; features
// (optional, [n][20]) receives the LDA feature rows. Returns the wall time in seconds.
double mo_spectrum_fdr(int kind, float lo, float hi, const void* rows_v, uint64_t n, const float* aligned_rt, const float* delta_rt, const float* delta_ims,
                       int threads, float* disc, float* pep, float* q, uint32_t* order, uint64_t* passing, int32_t* fitted, double* coef, double* eps,
                       double* features) {
    const auto t0 = std::chrono::steady_clock::now();
    const Row* rows = (const Row*)rows_v;
    threads = std::max(1, threads);
    *passing = 0;
    *fitted = 0;
    std::fill(coef, coef + D, 0.0);
    *eps = 0.0;
    std::vector<uint8_t> decoy(n);
    for (uint64_t i = 0; i < n; i++) decoy[i] = rows[i].label == -1;
    bool ok = false;
    if (n) {
        // score_psms, linear_discriminant.rs:133-231
        auto mass_error = [&](const Row& r) { return kind == 0 ? (double)r.delta_mass : (double)(float)(r.expmass - r.calcmass); };
        const double bw_adjust = kind == 0 ? 2.0 : 0.1;
        const float span = std::ceil(std::fmax(hi - lo, kind == 0 ? 100.0f : 1000.0f));
        std::vector<double> dm(n);
        for (uint64_t i = 0; i < n; i++) dm[i] = mass_error(rows[i]);
        const Estimator mass_model = kde_build(dm.data(), decoy.data(), n, (uint64_t)std::fabs(span), false, bw_adjust, threads);
        std::vector<double> X(n * D);
        for (uint64_t i = 0; i < n; i++) {
            const Row& r = rows[i];
            double* x = &X[i * D];
            double poisson = std::log1p(-r.poisson);
            if (!std::isfinite(poisson)) poisson = 3.5;
            x[0] = r.rank; x[1] = r.charge;
            x[2] = std::log1p(r.hyperscore); x[3] = std::log1p(r.delta_next); x[4] = std::log1p(r.delta_best);
            x[5] = mass_model.posterior_error(mass_error(r));
            x[6] = r.isotope_error; x[7] = r.average_ppm; x[8] = poisson;
            x[9] = std::log1p((double)r.matched_intensity_pct); x[10] = r.matched_peaks;
            x[11] = std::log1p((double)r.longest_b); x[12] = std::log1p((double)r.longest_y);
            x[13] = (double)r.longest_y / (double)r.peptide_len;
            x[14] = std::log1p((double)r.peptide_len); x[15] = r.missed_cleavages;
            x[16] = aligned_rt ? aligned_rt[i] : r.rt;
            x[17] = r.ims;
            x[18] = clamp_sqrt(delta_rt ? delta_rt[i] : 0.999f);
            x[19] = clamp_sqrt(delta_ims ? delta_ims[i] : 0.999f);
        }
        if (features) std::copy(X.begin(), X.end(), features);
        if (lda_train(X.data(), decoy.data(), n, D, coef, eps)) {
            ok = true;
            for (int j = 0; j < D; j++) ok = ok && std::isfinite(coef[j]);
        }
        if (ok) {
            std::vector<double> scores(n);
            for (uint64_t i = 0; i < n; i++) scores[i] = mo_lda_score(coef, &X[i * D], D);
            const Estimator kde = kde_build(scores.data(), decoy.data(), n, 1000, true, 1.0, threads);
            for (uint64_t i = 0; i < n; i++) {
                disc[i] = (float)scores[i];
                float p = (float)std::log10(kde.posterior_error(scores[i]));
                if (std::isinf(p)) p = -324.0f;
                pep[i] = p;
            }
        }
    }
    if (!ok) {   // runner.rs:284-287; posterior_error keeps its default 1.0
        for (uint64_t i = 0; i < n; i++) {
            disc[i] = log1pf((float)(-rows[i].poisson)) + rows[i].longest_y_pct / 3.0f;
            pep[i] = 1.0f;
        }
    }
    *fitted = ok;
    // par_sort_unstable_by(|a, b| b.discriminant_score.total_cmp(&a.discriminant_score)), ties by input row
    auto total_key = [&](uint64_t i) {
        int32_t b;
        memcpy(&b, &disc[i], 4);
        return b ^ (int32_t)((uint32_t)(b >> 31) >> 1);
    };
    std::vector<uint32_t> idx(n);
    for (uint64_t i = 0; i < n; i++) idx[i] = (uint32_t)i;
    std::stable_sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return total_key(a) > total_key(b); });
    // spectrum_q_value, qvalue.rs:8-36
    std::vector<float> qs(n);
    int32_t dec = 1, tar = 0;
    for (uint64_t p = 0; p < n; p++) {
        if (rows[idx[p]].label == -1) dec++;
        else tar++;
        qs[p] = (float)dec / (float)tar;
    }
    float q_min = 1.0f;
    uint64_t pass = 0;
    for (uint64_t p = n; p-- > 0;) {
        q_min = std::fmin(q_min, qs[p]);
        q[idx[p]] = q_min;
        if (q_min <= 0.01f) pass++;
    }
    *passing = pass;
    std::copy(idx.begin(), idx.end(), order);
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}


// RetentionModel::embed (model 0, charge ignored) or MobilityModel::embed (model 1) of one peptide into out[69] / out[100].
void mo_rt_embed(int model, const uint8_t* seq, uint64_t len, float mono, uint32_t charge, double* out) {
    if (model == 0) rt_embed(seq, len, mono, out);
    else ims_embed(seq, len, mono, (uint8_t)charge, out);
}

// LinearRegression::fit on a given row-major [n][d] matrix and targets: 1 with beta[d], r2 and eps, or 0 for None.
int mo_linreg_fit(const double* X, const double* y, uint64_t n, int d, int threads, double* beta, double* r2, double* eps) {
    const Fit f = linreg_fit(n, d, [&](uint64_t i, double* row) { std::copy(X + i * d, X + (i + 1) * d, row); }, [&](uint64_t i) { return y[i]; },
                             std::max(1, threads));
    if (!f.ok) return 0;
    std::copy(f.beta.begin(), f.beta.end(), beta);
    *r2 = f.r2;
    *eps = f.eps;
    return 1;
}

// runner.rs:513-531 predict_rt. Peptides: off[n_pep + 1], seq, mono. cols: aligned_rt, predicted_rt, delta_rt_model, predicted_ims,
// delta_ims_model, spectrum_q (indexed like the rows, each [n]). align[n_files][3] = max_rt, slope, intercept. stats = training rows, matrix rows
// kept. fitted / r2 / eps: [2] (RT, mobility). Returns the wall time in seconds.
double mo_predict_rt(const uint32_t* off, const uint8_t* seq, const float* mono, const void* rows_v, const uint32_t* file_id, uint64_t n, uint64_t n_files,
                     int threads, float* aligned_rt, float* predicted_rt, float* delta_rt, float* predicted_ims, float* delta_ims, float* spectrum_q, float* align,
                     uint64_t* stats, int32_t* fitted, double* r2, double* eps, double* rt_beta, double* ims_beta) {
    const auto t0 = std::chrono::steady_clock::now();
    const Row* rows = (const Row*)rows_v;
    threads = std::max(1, threads);
    // par_sort_unstable_by(|a, b| a.poisson.total_cmp(&b.poisson)), ties by input row
    auto total_key = [&](uint64_t i) {
        int64_t b;
        memcpy(&b, &rows[i].poisson, 8);
        return b ^ (int64_t)((uint64_t)(b >> 63) >> 1);
    };
    std::vector<uint32_t> order(n);
    for (uint64_t i = 0; i < n; i++) order[i] = (uint32_t)i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return total_key(a) < total_key(b); });
    // spectrum_q_value over that order
    std::vector<float> qs(n), q(n);
    int32_t dec = 1, tar = 0;
    for (uint64_t p = 0; p < n; p++) {
        if (rows[order[p]].label == -1) dec++;
        else tar++;
        qs[p] = (float)dec / (float)tar;
    }
    float q_min = 1.0f;
    for (uint64_t p = n; p-- > 0;) {
        q_min = std::fmin(q_min, qs[p]);
        q[order[p]] = q_min;
    }
    if (spectrum_q) std::copy(q.begin(), q.end(), spectrum_q);
    std::vector<uint32_t> train;   // the training filter, in poisson order
    for (uint64_t p = 0; p < n; p++)
        if (rows[order[p]].label == 1 && q[order[p]] <= 0.01f) train.push_back(order[p]);

    // global_alignment
    std::vector<uint32_t> max_u(n_files, 0);
    for (uint64_t i = 0; i < n; i++) max_u[file_id[i]] = std::max(max_u[file_id[i]], ceil_as_u32(rows[i].rt));
    std::vector<double> max_rt(n_files);
    for (uint64_t f = 0; f < n_files; f++) max_rt[f] = (double)max_u[f];
    std::map<uint32_t, std::map<uint64_t, double>> rts;
    for (uint32_t r : train) {
        auto& files = rts[rows[r].peptide_idx];
        auto it = files.find(file_id[r]);
        if (it == files.end()) files[file_id[r]] = (double)rows[r].rt;
        else it->second = rust_min(it->second, (double)rows[r].rt);
    }
    std::vector<std::vector<double>> mat;
    for (auto& [pep, files] : rts) {
        std::vector<double> v(n_files, NAN);
        double sum = 0.0, len = 0.0;
        for (auto& [f, rt0] : files) {
            const double rt = rt0 / max_rt[f];
            v[f] = rt;
            sum += rt;
            len += 1.0;
        }
        if (std::isnormal(sum / len)) mat.push_back(std::move(v));
    }
    std::vector<double> mean_rts(mat.size());
    for (size_t r = 0; r < mat.size(); r++) {
        uint64_t len = 0;
        double sum = 0.0;
        for (double x : mat[r])
            if (std::isfinite(x)) { len++; sum += x; }
        mean_rts[r] = sum / (double)len;
    }
    std::vector<float> al(3 * n_files);
    for (uint64_t f = 0; f < n_files; f++) {
        uint64_t len = 0;
        double dot = 0.0, sum_x = 0.0, sum_y = 0.0;
        for (size_t r = 0; r < mat.size(); r++) {
            const double x = mat[r][f], y = mean_rts[r];
            if (!std::isfinite(x)) continue;
            len++;
            dot += x * y;
            sum_x += x;
            sum_y += y;
        }
        const double x_mean = sum_x / (double)len, y_mean = sum_y / (double)len;
        const double ssxy = dot - (double)len * x_mean * y_mean;
        double sx2 = 1E-8;
        for (size_t r = 0; r < mat.size(); r++)
            if (std::isfinite(mat[r][f])) sx2 += (mat[r][f] - x_mean) * (mat[r][f] - x_mean);
        double slope = ssxy / sx2, intercept = y_mean - slope * x_mean;
        if (!std::isfinite(slope)) slope = 1.0;
        if (!std::isfinite(intercept)) intercept = 0.0;
        al[3 * f] = (float)max_rt[f];
        al[3 * f + 1] = (float)slope;
        al[3 * f + 2] = (float)intercept;
    }
    std::copy(al.begin(), al.end(), align);
    for (uint64_t i = 0; i < n; i++) {
        const float* a = &al[3 * file_id[i]];
        aligned_rt[i] = (rows[i].rt / a[0]) * a[1] + a[2];
    }
    stats[0] = train.size();
    stats[1] = mat.size();

    // retention_model::predict, mobility_model::predict
    auto pep_of = [&](uint32_t r, const uint8_t** s, uint64_t* len) {
        const uint32_t p = rows[r].peptide_idx;
        *s = seq + off[p];
        *len = off[p + 1] - off[p];
        return p;
    };
    for (int model = 0; model < 2; model++) {
        const int d = model == 0 ? RT_D : IMS_D;
        auto embed_row = [&](uint32_t r, double* e) {
            const uint8_t* s;
            uint64_t len;
            const uint32_t p = pep_of(r, &s, &len);
            if (model == 0) rt_embed(s, len, mono[p], e);
            else ims_embed(s, len, mono[p], (uint8_t)rows[r].charge, e);
        };
        const Fit fit = linreg_fit(
            train.size(), d, [&](uint64_t i, double* e) { embed_row(train[i], e); },
            [&](uint64_t i) { return model == 0 ? (double)aligned_rt[train[i]] : (double)rows[train[i]].ims; }, threads);
        float* pred = model == 0 ? predicted_rt : predicted_ims;
        float* delta = model == 0 ? delta_rt : delta_ims;
        fitted[model] = fit.ok;
        r2[model] = fit.ok ? fit.r2 : 0.0;
        eps[model] = fit.ok ? fit.eps : 0.0;
        double* beta_out = model == 0 ? rt_beta : ims_beta;
        std::fill(beta_out, beta_out + d, 0.0);
        if (!fit.ok) {
            std::fill(pred, pred + n, 0.0f);
            std::fill(delta, delta + n, 0.999f);
            continue;
        }
        std::copy(fit.beta.begin(), fit.beta.end(), beta_out);
        std::vector<double> e(d);
        const double hi = model == 0 ? 1.0 : 2.0;
        for (uint64_t i = 0; i < n; i++) {   // predict_peptide: fold from 0.0, then clamp (NaN passes) as f32
            embed_row((uint32_t)i, e.data());
            double v = 0.0;
            for (int j = 0; j < d; j++) v = v + e[j] * fit.beta[j];
            if (v < 0.0) v = 0.0;
            if (v > hi) v = hi;
            const float bounded = (float)v;
            pred[i] = bounded;
            delta[i] = std::fabs((model == 0 ? aligned_rt[i] : rows[i].ims) - bounded);
        }
    }
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ fdr.rs (picked FDR)
namespace {

std::string fmt_plus(float x) {   // `{:+}` of an f32: shortest round-trip, positional, signed; NaN prints "NaN"
    if (std::isnan(x)) return "NaN";
    if (std::isinf(x)) return x > 0 ? "+inf" : "-inf";
    char buf[128];
    auto r = std::to_chars(buf, buf + sizeof buf, x, std::chars_format::fixed);
    std::string s(buf, r.ptr);
    return std::signbit(x) ? s : "+" + s;
}

struct PepTable {
    const uint32_t* off;
    const uint8_t* seq;
    const float* mods;
    const float* nterm;
    const float* cterm;   // NULL = None everywhere
    const uint8_t* decoy;
};

std::string display(const PepTable& T, uint32_t i, bool reversed) {   // impl Display for Peptide, of the peptide or of its reverse()
    const uint32_t a = T.off[i], L = T.off[i + 1] - a;
    std::string s(T.seq + a, T.seq + a + L);
    std::vector<float> m(T.mods + a, T.mods + a + L);
    const uint32_t n = L == 0 ? 0 : L - 1;
    if (reversed && n > 1) {
        std::reverse(s.begin() + 1, s.begin() + n);
        std::reverse(m.begin() + 1, m.begin() + n);
    }
    std::string out;
    if (!std::isnan(T.nterm[i])) out += "[" + fmt_plus(T.nterm[i]) + "]-";
    for (uint32_t k = 0; k < L; k++) {
        out += s[k];
        if (m[k] != 0.0f) out += "[" + fmt_plus(m[k]) + "]";   // NaN != 0.0 holds
    }
    if (T.cterm && !std::isnan(T.cterm[i])) out += "-[" + fmt_plus(T.cterm[i]) + "]";
    return out;
}

struct Comp {
    float forward = -3.40282347e+38f, reverse = -3.40282347e+38f;
    bool has_f = false, has_r = false;
    std::string fix, rix;
};

// An insertion-ordered map: entries in the order their key first appears.
struct CompMap {
    std::unordered_map<std::string, size_t> at;
    std::vector<Comp> entries;
    Comp& entry(const std::string& key) {
        auto it = at.find(key);
        if (it != at.end()) return entries[it->second];
        at.emplace(key, entries.size());
        entries.emplace_back();
        return entries.back();
    }
};

float fmax_rust(float acc, float v) { return v > acc ? v : acc; }
float fmin_q(float a, float b) {   // DESIGN.md §12: NaN ignored, -0.0 below +0.0
    if (std::isnan(a)) return b;
    if (std::isnan(b)) return a;
    if (a < b) return a;
    if (b < a) return b;
    return std::signbit(a) ? a : b;
}
int64_t total_key(float x) {
    int32_t b;
    memcpy(&b, &x, 4);
    return (int64_t)(b ^ ((b >> 31) & 0x7FFFFFFF));
}

struct QRow {
    std::string ix;
    bool decoy;
    float score, q;
};

// fdr.rs:87-111 over rows in pre-sort order; pep_of(row) gives each sorted row's PEP.
template <class Pep>
uint64_t q_tail(std::vector<QRow>& rows, Pep pep_of, float threshold) {
    std::stable_sort(rows.begin(), rows.end(), [](const QRow& a, const QRow& b) { return total_key(b.score) < total_key(a.score); });
    float decoy = 1.0f, target = 0.0f;
    for (QRow& r : rows) {
        decoy += pep_of(r);
        if (!r.decoy) target += 1.0f;
        r.q = decoy / target;
    }
    float q_min = 1.0f;
    uint64_t passing = 0;
    for (size_t k = rows.size(); k-- > 0;) {
        q_min = fmin_q(q_min, rows[k].q);
        rows[k].q = q_min;
        if (q_min <= threshold && !rows[k].decoy) passing++;
    }
    return passing;
}

// Competition::assign_q_value (fdr.rs:59-120)
uint64_t assign_q_value(const CompMap& map, int threads, std::unordered_map<std::string, float>* out) {
    const size_t m = map.entries.size();
    std::vector<double> score(m);
    std::vector<uint8_t> dec(m);
    for (size_t e = 0; e < m; e++) {
        const Comp& c = map.entries[e];
        score[e] = (double)(c.reverse > c.forward ? c.reverse : c.forward);
        dec[e] = c.reverse >= c.forward;
    }
    std::vector<QRow> rows;
    for (const Comp& c : map.entries) {
        if (c.has_f) rows.push_back({c.fix, false, c.forward, 1.0f});
        if (c.has_r) rows.push_back({c.rix, true, c.reverse, 1.0f});
    }
    if (m == 0) return 0;
    const Estimator est = kde_build(score.data(), dec.data(), m, 1000, true, 1.0, threads);
    const uint64_t passing = q_tail(rows, [&](const QRow& r) { return (float)est.posterior_error((double)r.score); }, 0.01f);
    for (const QRow& r : rows) (*out)[r.ix] = r.q;   // later rows overwrite
    return passing;
}

}  // namespace

extern "C" {

// picked_peptide then picked_protein. Proteins of peptide i: names [prot_off[i], prot_off[i+1]) of the list whose name k is
// chars[name_off[k] .. name_off[k+1]). Returns 0, or -1 for two distinct peptides on one side with one key (clash[0..1]).
int mo_picked_fdr(const uint32_t* off, const uint8_t* seq, const float* mods, const float* nterm, const float* cterm, const uint8_t* decoy,
                  const uint32_t* prot_off, const uint64_t* name_off, const char* chars, const char* decoy_tag, int generate_decoys,
                  const uint32_t* pep_idx, const float* disc, uint64_t n, int threads, float* peptide_q, float* protein_q, uint64_t* passing,
                  uint64_t* entries, uint32_t* clash) {
    const PepTable T{off, seq, mods, nterm, cterm, decoy};
    std::unordered_map<uint32_t, std::string> keys;
    CompMap pm;
    for (uint64_t i = 0; i < n; i++) {   // fdr.rs:125-144
        const uint32_t p = pep_idx[i];
        auto it = keys.find(p);
        if (it == keys.end()) it = keys.emplace(p, display(T, p, generate_decoys && decoy[p])).first;
        Comp& e = pm.entry(it->second);
        const std::string ix = std::to_string(p);
        std::string& side_ix = decoy[p] ? e.rix : e.fix;
        bool& has = decoy[p] ? e.has_r : e.has_f;
        if (has && side_ix != ix) {
            clash[0] = (uint32_t)std::stoul(side_ix);
            clash[1] = p;
            return -1;
        }
        float& sc = decoy[p] ? e.reverse : e.forward;
        sc = fmax_rust(sc, disc[i]);
        side_ix = ix;
        has = true;
    }
    std::unordered_map<std::string, float> pq;
    passing[0] = assign_q_value(pm, threads, &pq);
    entries[0] = pm.entries.size();
    for (uint64_t i = 0; i < n; i++) peptide_q[i] = pq.at(std::to_string(pep_idx[i]));   // fdr.rs:148-150

    auto name = [&](uint32_t k) { return std::string(chars + name_off[k], chars + name_off[k + 1]); };
    auto proteins = [&](uint32_t p) {   // Peptide::proteins(decoy_tag, generate_decoys), peptide.rs:81-96
        std::string s;
        for (uint32_t k = prot_off[p]; k < prot_off[p + 1]; k++) {
            if (k > prot_off[p]) s += ";";
            s += (decoy[p] && generate_decoys) ? std::string(decoy_tag) + name(k) : name(k);
        }
        return s;
    };
    CompMap rm;
    for (uint64_t i = 0; i < n; i++) {   // fdr.rs:160-177: the key is the protein list, here of length 1
        const uint32_t p = pep_idx[i];
        if (prot_off[p + 1] - prot_off[p] != 1) continue;
        Comp& e = rm.entry(name(prot_off[p]));
        if (decoy[p]) { e.reverse = fmax_rust(e.reverse, disc[i]); e.rix = proteins(p); e.has_r = true; }
        else { e.forward = fmax_rust(e.forward, disc[i]); e.fix = proteins(p); e.has_f = true; }
    }
    std::unordered_map<std::string, float> rq;
    passing[1] = assign_q_value(rm, threads, &rq);
    entries[1] = rm.entries.size();
    for (uint64_t i = 0; i < n; i++) {   // fdr.rs:181-187
        const uint32_t p = pep_idx[i];
        protein_q[i] = prot_off[p + 1] - prot_off[p] == 1 ? rq.at(proteins(p)) : 1.0f;
    }
    return 0;
}

// picked_precursor (fdr.rs:228-287) over the rows in the given order.
uint64_t mo_picked_precursor(const double* score, const uint8_t* decoy, uint64_t n, float* q) {
    std::vector<QRow> rows(n);
    for (uint64_t i = 0; i < n; i++) rows[i] = {std::to_string(i), decoy[i] != 0, (float)score[i], 1.0f};
    // `decoy += 1.0` on decoy rows and `target += 1.0` on target rows: the tail's sum with PEP 1 / 0 (+0.0 leaves an f32 as it is)
    const uint64_t passing = q_tail(rows, [](const QRow& r) { return r.decoy ? 1.0f : 0.0f; }, 0.05f);
    for (const QRow& r : rows) q[std::stoull(r.ix)] = r.q;
    return passing;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ protein_grouping.rs, fdr.rs:192-226
// generate_protein_groups and picked_protein_group with real name strings and the reference's order of steps: ordered maps where the reference
// sorts, the literal BipartiteGraph loop (trim to a fixpoint, add the largest, repeat), Peptide::proteins for the fallback.
namespace {

using ProteinKey = std::pair<std::string, bool>;

// BipartiteGraph (protein_grouping.rs), literally.
struct Bipartite {
    std::vector<std::pair<uint32_t, uint32_t>> edges;
    std::vector<uint32_t> original, left_degree, right_degree;
    std::vector<uint8_t> left_cover, right_cover;
    uint64_t picks = 0;
    Bipartite(std::vector<std::pair<uint32_t, uint32_t>> e, size_t n_left, size_t n_right)
        : edges(std::move(e)), left_degree(n_left, 0), right_degree(n_right, 0), left_cover(n_left, 0), right_cover(n_right, 0) {
        for (auto [l, r] : edges) {
            left_degree[l]++;
            right_degree[r]++;
        }
        original = left_degree;
    }
    void trim() {
        size_t prev = 0;
        while (prev != edges.size()) {
            prev = edges.size();
            for (auto [l, r] : edges)
                if (right_degree[r] == 1) left_cover[l] = 1;
            std::vector<std::pair<uint32_t, uint32_t>> kept;
            for (auto [l, r] : edges) {
                if (left_cover[l]) {
                    right_cover[r] = 1;
                    left_degree[l]--;
                    right_degree[r]--;
                } else {
                    kept.push_back({l, r});
                }
            }
            edges.swap(kept);
            kept.clear();
            for (auto [l, r] : edges) {
                if (right_cover[r]) {
                    left_degree[l]--;
                    right_degree[r]--;
                } else {
                    kept.push_back({l, r});
                }
            }
            edges.swap(kept);
        }
    }
    void add_largest() {   // max_by_key over (remaining, original): the last of equal maxima
        size_t best = 0;
        for (size_t i = 1; i < left_degree.size(); i++)
            if (std::make_pair(left_degree[i], original[i]) >= std::make_pair(left_degree[best], original[best])) best = i;
        left_cover[best] = 1;
        picks++;
    }
    std::vector<uint8_t> into_cover() {
        while (!edges.empty()) {
            trim();
            if (!edges.empty()) add_largest();
        }
        return left_cover;
    }
};

struct GroupingInput {
    const uint32_t* prot_off;
    const uint64_t* name_off;
    const char* chars;
    const uint8_t* decoy;
    std::string name(uint32_t k) const { return std::string(chars + name_off[k], chars + name_off[k + 1]); }
};

std::string format_name(const ProteinKey& k, const std::string& tag, bool generate_decoys) {
    return k.second && generate_decoys ? tag + k.first : k.first;
}

// annotate_features at one threshold: rows with an empty string are unannotated. Appends the pass's group table lines
// ("<covered> <decoy> <sorted names joined by />") and writes [peptides, meta peptides, groups, covered, greedy picks, annotated] to stats.
void annotate(const GroupingInput& in, const uint32_t* pep_idx, const int32_t* label, const float* peptide_q, uint64_t n, float threshold,
              const std::string& tag, bool generate_decoys, std::vector<std::string>& groups_of_row, std::vector<uint32_t>& num,
              std::vector<uint8_t>& pass, uint8_t pass_no, std::string& table, uint64_t* stats) {
    std::set<uint32_t> peptides;
    for (uint64_t i = 0; i < n; i++)
        if (label[i] != -1 && peptide_q[i] < threshold) peptides.insert(pep_idx[i]);
    // ProteinGrouper::build
    std::map<ProteinKey, uint32_t> protein_index;
    std::vector<ProteinKey> proteins;
    std::set<std::vector<uint32_t>> meta_peptides;
    for (uint32_t p : peptides) {
        std::vector<uint32_t> list;
        for (uint32_t k = in.prot_off[p]; k < in.prot_off[p + 1]; k++) {
            ProteinKey key{in.name(k), in.decoy[p] != 0};
            auto it = protein_index.find(key);
            if (it == protein_index.end()) {
                it = protein_index.emplace(key, (uint32_t)proteins.size()).first;
                proteins.push_back(key);
            }
            list.push_back(it->second);
        }
        std::sort(list.begin(), list.end());
        meta_peptides.insert(list);
    }
    std::map<uint32_t, std::vector<size_t>> prot_to_metapeps;
    size_t i_meta = 0;
    for (const auto& mp : meta_peptides) {
        for (uint32_t prot : mp) prot_to_metapeps[prot].push_back(i_meta);
        i_meta++;
    }
    std::map<std::vector<size_t>, std::vector<uint32_t>> evidence_to_group;
    for (const auto& [prot, metas] : prot_to_metapeps) evidence_to_group[metas].push_back(prot);
    std::vector<std::vector<uint32_t>> groups;
    std::vector<std::pair<uint32_t, uint32_t>> edges;
    for (const auto& [metas, group] : evidence_to_group) {
        for (size_t m : metas) edges.push_back({(uint32_t)groups.size(), (uint32_t)m});
        groups.push_back(group);
    }
    // into_group_map
    Bipartite graph(edges, groups.size(), meta_peptides.size());
    const std::vector<uint8_t> cover = graph.into_cover();
    std::map<ProteinKey, std::vector<uint32_t>> protein_to_groups;
    std::vector<std::string> group_str(groups.size());
    uint64_t covered = 0;
    for (size_t g = 0; g < groups.size(); g++) {
        std::vector<std::string> fmt, raw;
        for (uint32_t ix : groups[g]) {
            fmt.push_back(format_name(proteins[ix], tag, generate_decoys));
            raw.push_back(proteins[ix].first);
        }
        std::sort(fmt.begin(), fmt.end());
        std::sort(raw.begin(), raw.end());
        for (size_t k = 0; k < fmt.size(); k++) group_str[g] += (k ? "/" : "") + fmt[k];
        table += std::to_string((int)cover[g]) + " " + std::to_string((int)proteins[groups[g][0]].second) + " ";
        for (size_t k = 0; k < raw.size(); k++) table += (k ? "/" : "") + raw[k];
        table += "\n";
        if (!cover[g]) continue;
        covered++;
        for (uint32_t ix : groups[g]) protein_to_groups[proteins[ix]].push_back((uint32_t)g);
    }
    // the lookup of every row still unannotated
    uint64_t annotated = 0;
    for (uint64_t i = 0; i < n; i++) {
        if (pass[i]) continue;
        const uint32_t p = pep_idx[i];
        std::set<uint32_t> group_set;
        for (uint32_t k = in.prot_off[p]; k < in.prot_off[p + 1]; k++) {
            auto it = protein_to_groups.find({in.name(k), in.decoy[p] != 0});
            if (it != protein_to_groups.end()) group_set.insert(it->second.begin(), it->second.end());
        }
        if (group_set.empty()) continue;
        std::vector<std::string> strs;
        for (uint32_t g : group_set) strs.push_back(group_str[g]);
        std::sort(strs.begin(), strs.end());
        std::string s;
        for (size_t k = 0; k < strs.size(); k++) s += (k ? ";" : "") + strs[k];
        num[i] = (uint32_t)std::count(s.begin(), s.end(), ';') + 1;
        groups_of_row[i] = s;
        pass[i] = pass_no;
        annotated++;
    }
    stats[0] = peptides.size();
    stats[1] = meta_peptides.size();
    stats[2] = groups.size();
    stats[3] = covered;
    stats[4] = graph.picks;
    stats[5] = annotated;
}

std::string g_grouping_text;

}  // namespace

extern "C" {

// generate_protein_groups then picked_protein_group. Names as for mo_picked_fdr. Writes num / pass / q per row, and to stats: pass 1's then
// pass 2's [peptides, meta peptides, groups, covered, greedy picks, annotated], passing, entries. Returns the length of the text kept for
// mo_grouping_text: each row's protein_groups string, then pass 1's and pass 2's group table lines, each line ended by '\n'.
uint64_t mo_protein_groups(const uint32_t* prot_off, const uint64_t* name_off, const char* chars, const uint8_t* decoy, const uint32_t* pep_idx,
                           const int32_t* label, const float* peptide_q, const float* disc, uint64_t n, int protein_grouping, int has_threshold,
                           float threshold, int generate_decoys, const char* decoy_tag, int threads, uint32_t* num, uint8_t* pass, float* q,
                           uint64_t* stats) {
    const GroupingInput in{prot_off, name_off, chars, decoy};
    const std::string tag(decoy_tag);
    std::vector<std::string> strs(n);
    std::vector<uint32_t> count(n, 0);
    std::vector<uint8_t> row_pass(n, 0);
    std::string tables[2];
    std::fill(stats, stats + 14, 0);
    if (protein_grouping) {
        if (has_threshold) {
            float t = threshold;   // f32::clamp(0.0, 1.0): NaN stays NaN
            if (t < 0.0f) t = 0.0f;
            if (t > 1.0f) t = 1.0f;
            annotate(in, pep_idx, label, peptide_q, n, t, tag, generate_decoys, strs, count, row_pass, 1, tables[0], stats);
        }
        annotate(in, pep_idx, label, peptide_q, n, 1.0f, tag, generate_decoys, strs, count, row_pass, 2, tables[1], stats + 6);
    }
    for (uint64_t i = 0; i < n; i++) {   // the fallback: Peptide::proteins(decoy_tag, generate_decoys)
        if (row_pass[i]) continue;
        const uint32_t p = pep_idx[i];
        std::string s;
        for (uint32_t k = prot_off[p]; k < prot_off[p + 1]; k++) s += (k > prot_off[p] ? ";" : "") + format_name({in.name(k), decoy[p] != 0}, tag, generate_decoys);
        strs[i] = s;
        count[i] = prot_off[p + 1] - prot_off[p];
    }
    // picked_protein_group: key and Ix are the string
    CompMap map;
    for (uint64_t i = 0; i < n; i++) {
        if (count[i] != 1) continue;
        Comp& e = map.entry(strs[i]);
        if (decoy[pep_idx[i]]) { e.reverse = fmax_rust(e.reverse, disc[i]); e.rix = strs[i]; e.has_r = true; }
        else { e.forward = fmax_rust(e.forward, disc[i]); e.fix = strs[i]; e.has_f = true; }
    }
    std::unordered_map<std::string, float> scores;
    stats[12] = assign_q_value(map, threads, &scores);
    stats[13] = map.entries.size();
    g_grouping_text.clear();
    for (uint64_t i = 0; i < n; i++) {
        num[i] = count[i];
        pass[i] = row_pass[i];
        q[i] = count[i] == 1 ? scores.at(strs[i]) : 1.0f;
        g_grouping_text += strs[i] + "\n";
    }
    g_grouping_text += tables[0] + tables[1];
    return g_grouping_text.size();
}

void mo_grouping_text(char* dst) { memcpy(dst, g_grouping_text.data(), g_grouping_text.size()); }

// BipartiteGraph::new(edges, n_left, n_right).into_cover(), literally. Returns the number of add_largest picks.
uint64_t mo_bipartite_cover(const uint32_t* left, const uint32_t* right, uint64_t n_edges, uint64_t n_left, uint64_t n_right, uint8_t* cover) {
    std::vector<std::pair<uint32_t, uint32_t>> edges(n_edges);
    for (uint64_t k = 0; k < n_edges; k++) edges[k] = {left[k], right[k]};
    Bipartite graph(std::move(edges), n_left, n_right);
    const std::vector<uint8_t> c = graph.into_cover();
    std::copy(c.begin(), c.end(), cover);
    return graph.picks;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ result files (runner.rs writers)
// The text of matched_fragments.sage.tsv and tmt.tsv with digits from std::to_chars (libstdc++'s shortest round-trip, closest, ties to even)
// laid out as ryu::Buffer::format and Rust's `{:+}` do, and csv-core's QuoteStyle::Necessary, in the definitions of DESIGN.md §17. Shares
// no code with sage_b200/csrc/write.cuh. (fmt_plus above takes std::to_chars' fixed form, which for |x| >= 2^24 can be the exact integer
// rather than Rust's shortest digits padded with zeros: the writer uses wo_plus.)
namespace {

// to_chars' shortest scientific form of |x|: its digits into d (returns their count) and the exponent of the last digit into k
template <class T>
int wo_digits(T x, char* d, int& k) {
    char b[64];
    auto r = std::to_chars(b, b + sizeof b, std::fabs(x), std::chars_format::scientific);
    int n = 0, i = 0;
    for (; b[i] != 'e'; i++)
        if (b[i] != '.') d[n++] = b[i];
    int e = 0;
    std::from_chars(b + i + 1 + (b[i + 1] == '+'), r.ptr, e);
    k = e - (n - 1);
    return n;
}

// ryu::Buffer::format of x into o (at least 64 bytes); returns the length
template <class T>
int wo_ryu_buf(T x, char* o) {
    const int T_ = sizeof(T) == 8 ? 16 : 13;
    auto put = [&](const char* s) { int n = (int)std::strlen(s); std::memcpy(o, s, n); return n; };
    if (std::isnan(x)) return put("NaN");
    if (std::isinf(x)) return put(x > 0 ? "inf" : "-inf");
    if (x == 0) return put(std::signbit(x) ? "-0.0" : "0.0");
    char d[32];
    int k, p = 0;
    const int len = wo_digits(x, d, k), kk = len + k;
    if (std::signbit(x)) o[p++] = '-';
    if (0 <= k && kk <= T_) {
        std::memcpy(o + p, d, len), p += len;
        for (int i = 0; i < k; i++) o[p++] = '0';
        o[p++] = '.', o[p++] = '0';
    } else if (0 < kk && kk <= T_) {
        std::memcpy(o + p, d, kk), p += kk;
        o[p++] = '.';
        std::memcpy(o + p, d + kk, len - kk), p += len - kk;
    } else if (-5 < kk && kk <= 0) {
        o[p++] = '0', o[p++] = '.';
        for (int i = 0; i < -kk; i++) o[p++] = '0';
        std::memcpy(o + p, d, len), p += len;
    } else {
        o[p++] = d[0];
        if (len > 1) {
            o[p++] = '.';
            std::memcpy(o + p, d + 1, len - 1), p += len - 1;
        }
        o[p++] = 'e';
        p = (int)(std::to_chars(o + p, o + 64, kk - 1).ptr - o);
    }
    return p;
}

// Rust's `{:+}` of an f32 into o (at least 64 bytes); returns the length
int wo_plus_buf(float x, char* o) {
    if (std::isnan(x)) return std::memcpy(o, "NaN", 3), 3;
    int p = 0;
    o[p++] = std::signbit(x) ? '-' : '+';
    if (std::isinf(x)) return std::memcpy(o + p, "inf", 3), p + 3;
    if (x == 0) return o[p++] = '0', p;
    char d[32];
    int k;
    const int len = wo_digits(x, d, k), kk = len + k;
    if (k >= 0) {
        std::memcpy(o + p, d, len), p += len;
        for (int i = 0; i < k; i++) o[p++] = '0';
    } else if (kk > 0) {
        std::memcpy(o + p, d, kk), p += kk;
        o[p++] = '.';
        std::memcpy(o + p, d + kk, len - kk), p += len - kk;
    } else {
        o[p++] = '0', o[p++] = '.';
        for (int i = 0; i < -kk; i++) o[p++] = '0';
        std::memcpy(o + p, d, len), p += len;
    }
    return p;
}

template <class T>
std::string wo_ryu(T x) {
    char o[64];
    return std::string(o, wo_ryu_buf(x, o));
}
std::string wo_plus(float x) {
    char o[64];
    return std::string(o, wo_plus_buf(x, o));
}

std::string wo_field(const char* s, size_t n) {   // csv-core QuoteStyle::Necessary, delimiter '\t'
    std::string f(s, n);
    if (f.find_first_of("\t\"\r\n") == std::string::npos) return f;
    std::string q = "\"";
    for (char c : f) {
        if (c == '"') q += '"';
        q += c;
    }
    return q + "\"";
}

struct WoFragment {
    int32_t kind, charge, ordinal;
    float intensity, mz_calculated, mz_experimental;
};

std::string g_wo_text;

// rec(i) -> record i's text; records split over `threads` host threads and joined in order
template <class F>
void wo_records(uint64_t n, int threads, F rec) {
    threads = std::max(1, threads);
    std::vector<std::string> part(threads);
    std::vector<std::thread> th;
    for (int t = 0; t < threads; t++)
        th.emplace_back([&, t] {
            for (uint64_t i = n * t / threads; i < n * (t + 1) / threads; i++) part[t] += rec(i);
        });
    for (auto& x : th) x.join();
    for (auto& p : part) g_wo_text += p;
}

std::string wo_header(const std::vector<std::string>& f) {
    std::string h;
    for (size_t i = 0; i < f.size(); i++) h += (i ? "\t" : "") + wo_field(f[i].data(), f[i].size());
    return h + "\n";
}

}  // namespace

extern "C" {

// Per-block FNV-1a 64 of formatted values, each followed by '\n': format 0 ryu f32 (bits first + i), 1 `{:+}` f32, 2 ryu f64 values[i].
void mo_format_hashes(int format, uint64_t first, const double* values, uint64_t n, uint64_t block, uint64_t* hashes, int threads) {
    const uint64_t nb = n / block;
    std::vector<std::thread> th;
    threads = std::max(1, threads);
    for (int t = 0; t < threads; t++)
        th.emplace_back([&, t] {
            for (uint64_t b = t; b < nb; b += threads) {
                uint64_t h = 0xcbf29ce484222325ull;
                for (uint64_t i = b * block; i < (b + 1) * block; i++) {
                    char s[72];
                    int n;
                    if (format == 2) n = wo_ryu_buf(values[i], s);
                    else {
                        const uint32_t u = (uint32_t)(first + i);
                        float x;
                        std::memcpy(&x, &u, 4);
                        n = format == 0 ? wo_ryu_buf(x, s) : wo_plus_buf(x, s);
                    }
                    s[n++] = '\n';
                    for (int c = 0; c < n; c++) h = (h ^ (unsigned char)s[c]) * 0x100000001b3ull;
                }
                hashes[b] = h;
            }
        });
    for (auto& x : th) x.join();
}

// One value's text: format 0 ryu f32, 1 `{:+}` f32, 2 ryu f64, 3 csv field of the bytes s[0..n). Returns the length written to out.
uint64_t mo_format_one(int format, double x, const char* s, uint64_t n, char* out) {
    std::string r = format == 0 ? wo_ryu((float)x) : format == 1 ? wo_plus((float)x) : format == 2 ? wo_ryu(x) : wo_field(s, n);
    std::memcpy(out, r.data(), r.size());
    return r.size();
}

// matched_fragments.sage.tsv; returns the size, the text is taken with mo_take_text
uint64_t mo_write_fragments(const uint64_t* psm_id, const uint32_t* frag_offset, const uint32_t* frag_count, uint64_t n_rows, const WoFragment* fr, int threads) {
    g_wo_text = wo_header({"psm_id", "fragment_type", "fragment_ordinals", "fragment_charge", "fragment_mz_calculated", "fragment_mz_experimental",
                           "fragment_intensity"});
    wo_records(n_rows, threads, [&](uint64_t i) {
        std::string r;
        for (uint32_t k = 0; k < frag_count[i]; k++) {
            const WoFragment& f = fr[frag_offset[i] + k];
            r += std::to_string(psm_id[i]) + "\t" + "abcxyz"[f.kind] + "\t" + std::to_string(f.ordinal) + "\t" + std::to_string(f.charge) + "\t" +
                 wo_ryu(f.mz_calculated) + "\t" + wo_ryu(f.mz_experimental) + "\t" + wo_ryu(f.intensity) + "\n";
        }
        return r;
    });
    return g_wo_text.size();
}

// tmt.tsv
uint64_t mo_write_tmt(const uint64_t* file_off, const char* file_bytes, const uint64_t* spec_off, const char* spec_bytes, const uint32_t* file_id,
                      const uint32_t* spec, const float* injection, const float* peaks, uint64_t n, uint64_t n_channels, int user_labels, int threads) {
    std::vector<std::string> h = {"filename", "scannr", "ion_injection_time"};
    for (uint64_t c = 0; c < n_channels; c++) h.push_back((user_labels ? "user_" : "tmt_") + std::to_string(c + 1));
    g_wo_text = wo_header(h);
    wo_records(n, threads, [&](uint64_t i) {
        std::string r = wo_field(file_bytes + file_off[file_id[i]], file_off[file_id[i] + 1] - file_off[file_id[i]]) + "\t" +
                        wo_field(spec_bytes + spec_off[spec[i]], spec_off[spec[i] + 1] - spec_off[spec[i]]) + "\t" + wo_ryu(injection[i]);
        for (uint64_t c = 0; c < n_channels; c++) r += "\t" + wo_ryu(peaks[i * n_channels + c]);
        return r + "\n";
    });
    return g_wo_text.size();
}

// The peptide table and names the results / pin / lfq writers read.
struct WoTable {
    const uint32_t* res_off;
    const uint8_t* seq;
    const float* mods;
    const float* nterm;
    const float* cterm;   // NULL = None
    const uint8_t* decoy;
    const uint8_t* semi;  // NULL = 0
    const uint32_t* prot_off;
    const uint32_t* prot_ids;
    const uint64_t* name_off;
    const char* name_bytes;
    const char* tag;
    int generate_decoys;
};

// The post-search columns of results / pin; NULL = Feature's default.
struct WoColumns {
    const float *discriminant, *posterior, *spectrum_q, *peptide_q, *protein_q, *protein_group_q, *aligned_rt, *predicted_rt, *delta_rt, *predicted_ims,
        *delta_ims;
    const uint32_t* num_groups;
    const uint8_t* group_pass;   // NULL: no groups
    const uint64_t* row_group_off;
    const uint32_t* row_groups;
    const uint64_t* group_off;
    const uint32_t* group_members;
    const uint8_t* group_decoy;
};

static std::string wo_name(const WoTable& t, uint32_t id) { return std::string(t.name_bytes + t.name_off[id], t.name_bytes + t.name_off[id + 1]); }
static std::string wo_display(const WoTable& t, uint32_t p) {   // impl Display for Peptide with Rust's `{:+}`
    std::string out;
    if (!std::isnan(t.nterm[p])) out += "[" + wo_plus(t.nterm[p]) + "]-";
    for (uint32_t r = t.res_off[p]; r < t.res_off[p + 1]; r++) {
        out += (char)t.seq[r];
        if (t.mods[r] != 0.0f) out += "[" + wo_plus(t.mods[r]) + "]";
    }
    if (t.cterm && !std::isnan(t.cterm[p])) out += "-[" + wo_plus(t.cterm[p]) + "]";
    return out;
}
static std::string wo_proteins(const WoTable& t, uint32_t p) {   // Peptide::proteins
    std::string out;
    for (uint32_t k = t.prot_off[p]; k < t.prot_off[p + 1]; k++) {
        if (k > t.prot_off[p]) out += ";";
        out += (t.decoy[p] && t.generate_decoys ? std::string(t.tag) : std::string()) + wo_name(t, t.prot_ids[k]);
    }
    return out;
}
static std::string wo_groups(const WoTable& t, const WoColumns& c, uint64_t i, uint32_t p) {
    if (!c.group_pass) return "";
    if (!c.group_pass[i]) return wo_proteins(t, p);
    std::vector<std::string> gs;
    for (uint64_t k = c.row_group_off[i]; k < c.row_group_off[i + 1]; k++) {
        const uint32_t g = c.row_groups[k];
        std::vector<std::string> names;
        for (uint64_t m = c.group_off[g]; m < c.group_off[g + 1]; m++)
            names.push_back((c.group_decoy[g] && t.generate_decoys ? std::string(t.tag) : std::string()) + wo_name(t, c.group_members[m]));
        std::sort(names.begin(), names.end());
        std::string s;
        for (size_t j = 0; j < names.size(); j++) s += (j ? "/" : "") + names[j];
        gs.push_back(s);
    }
    std::sort(gs.begin(), gs.end());
    std::string out;
    for (size_t j = 0; j < gs.size(); j++) out += (j ? ";" : "") + gs[j];
    return out;
}
static float wo_opt(const float* a, uint64_t i, float d) { return a ? a[i] : d; }
static std::string wo_str(const uint64_t* off, const char* bytes, uint32_t i) { return std::string(bytes + off[i], bytes + off[i + 1]); }

static const std::vector<std::string> kResultsHeader = {"psm_id", "peptide", "proteins", "protein_groups", "num_proteins", "num_protein_groups", "filename",
    "scannr", "rank", "label", "expmass", "calcmass", "charge", "peptide_len", "missed_cleavages", "semi_enzymatic", "isotope_error", "precursor_ppm",
    "fragment_ppm", "hyperscore", "delta_next", "delta_best", "rt", "aligned_rt", "predicted_rt", "delta_rt_model", "ion_mobility", "predicted_mobility",
    "delta_mobility", "matched_peaks", "longest_b", "longest_y", "longest_y_pct", "matched_intensity_pct", "scored_candidates", "poisson",
    "sage_discriminant_score", "posterior_error", "spectrum_q", "peptide_q", "protein_q", "protein_group_q", "ms2_intensity"};
static const std::vector<std::string> kPinHeader = {"SpecId", "Label", "ScanNr", "ExpMass", "CalcMass", "FileName", "retentiontime", "ion_mobility", "rank",
    "z=2", "z=3", "z=4", "z=5", "z=6", "z=other", "peptide_len", "missed_cleavages", "semi_enzymatic", "isotope_error", "ln(precursor_ppm)", "fragment_ppm",
    "ln(hyperscore)", "ln(delta_next)", "ln(delta_best)", "aligned_rt", "predicted_rt", "sqrt(delta_rt_model)", "predicted_mobility",
    "sqrt(delta_mobility)", "matched_peaks", "longest_b", "longest_y", "longest_y_pct", "ln(matched_intensity_pct)", "scored_candidates", "ln(-poisson)",
    "posterior_error", "Peptide", "Proteins"};

// results.sage.tsv (pin = 0) or results.sage.pin (pin = 1); std::regex gives the pin's ScanNr
uint64_t mo_write_results(int pin, const Row* rows, const uint64_t* psm_id, const uint32_t* file_id, const uint32_t* spec, uint64_t n, const uint64_t* file_off,
                          const char* file_bytes, const uint64_t* spec_off, const char* spec_bytes, const WoTable* tab, const WoColumns* cols, int threads) {
    const WoTable& t = *tab;
    const WoColumns& c = *cols;
    g_wo_text = wo_header(pin ? kPinHeader : kResultsHeader);
    const std::regex scan_re("scan=([0-9]+)");
    wo_records(n, threads, [&](uint64_t i) {
        const Row& r = rows[i];
        const uint32_t p = r.peptide_idx;
        const std::string fname = wo_field(file_bytes + file_off[file_id[i]], file_off[file_id[i] + 1] - file_off[file_id[i]]);
        const std::string sid = wo_str(spec_off, spec_bytes, spec[i]);
        const std::string pep = wo_display(t, p), prots = wo_proteins(t, p);
        std::vector<std::string> f;
        auto I = [&](int64_t v) { f.push_back(std::to_string(v)); };
        const int semi = t.semi ? t.semi[p] : 0;
        const float aligned = wo_opt(c.aligned_rt, i, r.rt), pred_rt = wo_opt(c.predicted_rt, i, 0.0f), drt = wo_opt(c.delta_rt, i, 0.999f);
        const float pred_ims = wo_opt(c.predicted_ims, i, 0.0f), dims = wo_opt(c.delta_ims, i, 0.999f), post = wo_opt(c.posterior, i, 1.0f);
        if (!pin) {
            I((int64_t)psm_id[i]);
            f.push_back(wo_field(pep.data(), pep.size()));
            f.push_back(wo_field(prots.data(), prots.size()));
            const std::string g = wo_groups(t, c, i, p);
            f.push_back(wo_field(g.data(), g.size()));
            I(t.prot_off[p + 1] - t.prot_off[p]);
            I(c.num_groups ? c.num_groups[i] : 0);
            f.push_back(fname);
            f.push_back(wo_field(sid.data(), sid.size()));
            I(r.rank); I(r.label);
            f.push_back(wo_ryu(r.expmass)); f.push_back(wo_ryu(r.calcmass));
            I(r.charge); I(r.peptide_len); I(r.missed_cleavages); I(semi);
            f.push_back(wo_ryu(r.isotope_error)); f.push_back(wo_ryu(r.delta_mass)); f.push_back(wo_ryu(r.average_ppm));
            f.push_back(wo_ryu(r.hyperscore)); f.push_back(wo_ryu(r.delta_next)); f.push_back(wo_ryu(r.delta_best));
            f.push_back(wo_ryu(r.rt)); f.push_back(wo_ryu(aligned)); f.push_back(wo_ryu(pred_rt)); f.push_back(wo_ryu(drt));
            f.push_back(wo_ryu(r.ims)); f.push_back(wo_ryu(pred_ims)); f.push_back(wo_ryu(dims));
            I(r.matched_peaks); I(r.longest_b); I(r.longest_y);
            f.push_back(wo_ryu(r.longest_y_pct)); f.push_back(wo_ryu(r.matched_intensity_pct));
            I(r.scored_candidates);
            f.push_back(wo_ryu(r.poisson));
            f.push_back(wo_ryu(wo_opt(c.discriminant, i, 0.0f))); f.push_back(wo_ryu(post)); f.push_back(wo_ryu(wo_opt(c.spectrum_q, i, 1.0f)));
            f.push_back(wo_ryu(wo_opt(c.peptide_q, i, 1.0f))); f.push_back(wo_ryu(wo_opt(c.protein_q, i, 1.0f)));
            f.push_back(wo_ryu(wo_opt(c.protein_group_q, i, 1.0f))); f.push_back(wo_ryu(r.ms2_intensity));
        } else {
            std::string scannr = sid;
            for (auto it = std::sregex_iterator(sid.begin(), sid.end(), scan_re); it != std::sregex_iterator(); ++it) scannr = (*it)[1].str();
            I((int64_t)psm_id[i]); I(r.label);
            f.push_back(wo_field(scannr.data(), scannr.size()));
            f.push_back(wo_ryu(r.expmass)); f.push_back(wo_ryu(r.calcmass));
            f.push_back(fname);
            f.push_back(wo_ryu(r.rt)); f.push_back(wo_ryu(r.ims));
            I(r.rank);
            for (uint32_t z = 2; z <= 6; z++) I(r.charge == z ? 1 : 0);
            I((r.charge < 2 || r.charge > 6) ? r.charge : 0);
            I(r.peptide_len); I(r.missed_cleavages); I(semi);
            f.push_back(wo_ryu(r.isotope_error));
            f.push_back(wo_ryu(log1pf(std::fabs(r.delta_mass))));
            f.push_back(wo_ryu(r.average_ppm));
            f.push_back(wo_ryu(std::log1p(r.hyperscore))); f.push_back(wo_ryu(std::log1p(r.delta_next))); f.push_back(wo_ryu(std::log1p(r.delta_best)));
            f.push_back(wo_ryu(aligned)); f.push_back(wo_ryu(pred_rt));
            const float cl = std::isnan(drt) ? drt : std::min(std::max(drt, 0.001f), 1.0f);
            f.push_back(wo_ryu(std::sqrt(cl)));
            f.push_back(wo_ryu(pred_ims)); f.push_back(wo_ryu(dims));
            I(r.matched_peaks); I(r.longest_b); I(r.longest_y);
            f.push_back(wo_ryu(r.longest_y_pct)); f.push_back(wo_ryu(log1pf(r.matched_intensity_pct)));
            I(r.scored_candidates);
            f.push_back(wo_ryu(std::log1p(-r.poisson)));
            f.push_back(wo_ryu(post));
            f.push_back(wo_field(pep.data(), pep.size()));
            f.push_back(wo_field(prots.data(), prots.size()));
        }
        std::string rec;
        for (size_t k = 0; k < f.size(); k++) rec += (k ? "\t" : "") + f[k];
        return rec + "\n";
    });
    return g_wo_text.size();
}

// lfq.tsv over sage_b200_lfq_integrate's rows (peptide u32, charge u8, decoy u8, 16 more bytes, spectral_angle f64, score f64)
struct WoLfqRow {
    uint32_t peptide;
    uint8_t charge, decoy;
    uint16_t pad0;
    uint32_t rt, pad1;
    double spectral_angle, score;
};
uint64_t mo_write_lfq(const WoLfqRow* rows, const double* areas, const float* q, uint64_t n, const uint64_t* file_off, const char* file_bytes, uint64_t n_files,
                      const WoTable* tab, int threads) {
    const WoTable& t = *tab;
    std::vector<std::string> h = {"peptide", "charge", "proteins", "q_value", "score", "spectral_angle"};
    for (uint64_t k = 0; k < n_files; k++) h.push_back(wo_str(file_off, file_bytes, (uint32_t)k));
    g_wo_text = wo_header(h);
    wo_records(n, threads, [&](uint64_t i) {
        const WoLfqRow& r = rows[i];
        if (r.decoy) return std::string();
        const std::string pep = wo_display(t, r.peptide), prots = wo_proteins(t, r.peptide);
        std::string rec = wo_field(pep.data(), pep.size()) + "\t" + std::to_string(r.charge ? (int)r.charge : -1) + "\t" + wo_field(prots.data(), prots.size()) +
                          "\t" + wo_ryu(q[i]) + "\t" + wo_ryu(r.score) + "\t" + wo_ryu(r.spectral_angle);
        for (uint64_t k = 0; k < n_files; k++) rec += "\t" + wo_ryu(areas[i * n_files + k]);
        return rec + "\n";
    });
    return g_wo_text.size();
}

void mo_take_text(char* out) { std::memcpy(out, g_wo_text.data(), g_wo_text.size()); }

}  // extern "C"
