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
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
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

}  // extern "C"
