"""An independent numpy restatement of sage's PSM rescoring and RT / mobility prediction, written from crates/sage/src/ml/ (kde.rs, mod.rs,
gauss.rs, matrix.rs, linear_discriminant.rs, qvalue.rs, retention_alignment.rs, regression.rs, retention_model.rs, mobility_model.rs) and
crates/sage-cli/src/runner.rs (cited as file:line). TEST INFRASTRUCTURE ONLY: it shares no code with the CPU oracle (oracle_ml/) or the device
kernels, so a misreading of the Rust that those two share shows up as a difference here.

Where the Rust leaves an order to rayon, a DashMap or a HashMap, this module uses the orders DESIGN.md §10 and §11 define:
- Kde::pdf: chunks of KDE_CHUNK samples in sample order, each folded from +0.0, the chunk sums added in order from -0.0;
- LinearRegression::fit: chunks of RT_CHUNK training rows in poisson order, each accumulator from 0.0, merged as ((0 + A0) + A1) + ...; the SSE
  as chunk sums from -0.0 added in order from -0.0;
- both unstable sorts are stable (ties by input row); peptides in ascending PeptideIx, files in ascending order;
- f64::min over a (peptide, file)'s RTs keeps -0.0 over +0.0; a `Sum` of f64 starts from -0.0, a `fold(0.0, ..)` from +0.0.

Every f32 / f64 operation is one numpy or Python operation (one IEEE rounding, no contraction). Folds whose association matters are explicit
loops, vectorised only across independent sums (never np.sum, which is pairwise, nor Python's sum, which compensates since 3.12). exp, log1p,
log10, log1pf and pow are the C library's: Python's math.exp for the KDE's exp (it calls libm, and its arguments there are <= 0 or NaN, which
never raise), ctypes calls of libm for everything else (math.log1p / math.log10 raise where libm returns -inf or NaN). numpy's own exp / log are
not libm's and are not used.
"""
from __future__ import annotations

import ctypes
import ctypes.util
import math

import numpy as np

f32, f64 = np.float32, np.float64
KDE_CHUNK = 4096                      # DESIGN.md §10
RT_CHUNK = 1024                       # DESIGN.md §11
FEATURES = 20                         # linear_discriminant.rs:19
VALID_AA = b"ACDEFGHIKLMNPQRSTVWYUO"   # mass.rs:59-62
PPM, DA = 0, 2                        # sage_b200.api.Tolerance kinds
F64_MAX = 1.7976931348623157e308

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
for _name in ("exp", "log1p", "log10"):
    getattr(_libm, _name).restype = ctypes.c_double
    getattr(_libm, _name).argtypes = [ctypes.c_double]
_libm.pow.restype, _libm.pow.argtypes = ctypes.c_double, [ctypes.c_double, ctypes.c_double]
_libm.log1pf.restype, _libm.log1pf.argtypes = ctypes.c_float, [ctypes.c_float]


def _per_unique(fn, x, dtype):
    """fn (a libm function through ctypes) on every element, called once per distinct value."""
    x = np.asarray(x, dtype)
    u, inv = np.unique(x.ravel(), return_inverse=True)
    return np.array([fn(float(v)) for v in u], dtype)[inv].reshape(x.shape)


def log1p(x):
    return _per_unique(_libm.log1p, x, f64)


def log10(x):
    return _per_unique(_libm.log10, x, f64)


def log1pf(x):
    return _per_unique(_libm.log1pf, x, f32)


def exp(x):
    """libm exp of every element. math.exp raises above ~709.78, where libm returns inf: those go through ctypes."""
    x = np.asarray(x, f64)
    flat = x.ravel()
    big = flat > 709.0
    out = np.fromiter(map(math.exp, np.where(big, 0.0, flat).tolist()), f64, len(flat))
    if big.any():
        out[big] = [_libm.exp(v) for v in flat[big].tolist()]
    return out.reshape(x.shape)


def div(a, b):
    """IEEE a / b (Python floats raise on a zero divisor)."""
    with np.errstate(all="ignore"):
        return float(f64(a) / f64(b))


def rust_max(acc, x):
    """f64::max(acc, x): the other operand when one is NaN."""
    if math.isnan(acc):
        return x
    if math.isnan(x):
        return acc
    return x if x > acc else acc


def rust_min_plain(acc, x):
    """f64::min(acc, x) where the sign of a zero cannot matter."""
    if math.isnan(acc):
        return x
    if math.isnan(x):
        return acc
    return x if x < acc else acc


def rust_min(acc, x):
    """f64::min(acc, x) as DESIGN.md §11 defines it: the other operand when one is NaN, -0.0 kept over +0.0."""
    if math.isnan(acc):
        return x
    if math.isnan(x):
        return acc
    if x < acc:
        return x
    if acc < x:
        return acc
    return acc if math.copysign(1.0, acc) < 0 else x


def total_key32(x):
    """f32::total_cmp as a signed integer key."""
    b = np.asarray(x, f32).view(np.int32).astype(np.int64)
    return b ^ ((b >> 31) & 0x7FFFFFFF)


def total_key64(x):
    """f64::total_cmp as a signed integer key."""
    b = np.asarray(x, f64).view(np.int64)
    return b ^ ((b >> 63).astype(np.uint64) >> np.uint64(1)).astype(np.int64)


# ---------------------------------------------------------------------------------------------------- ml/mod.rs, kde.rs
def mean(xs) -> float:
    """mod.rs:24-26: `iter().sum::<f64>()` (from -0.0) / len."""
    s = -0.0
    for v in xs:
        s += v
    return div(s, len(xs))


def std(xs) -> float:
    """mod.rs:28-32: fold from 0.0 of (x - mean).powi(2) (x * x), / len, sqrt."""
    m = mean(xs)
    acc = 0.0
    for v in xs:
        d = v - m
        acc = acc + d * d
    return math.sqrt(div(acc, len(xs)))


class Kde:
    """kde.rs:14-49."""

    def __init__(self, sample, bw_adjust):
        self.sample = np.asarray(sample, f64)
        n = len(self.sample)
        sigma = std(self.sample.tolist())
        self.bandwidth = bw_adjust(sigma * _libm.pow(div(4.0 / 3.0, n), 1.0 / 5.0))   # kde.rs:22-25
        self.constant = math.sqrt(2.0 * math.pi) * self.bandwidth * n                  # kde.rs:26

    def pdf(self, x):
        """kde.rs:38-48 at every point of x: Σ exp(-0.5 * ((x - xi) / h)²) over the sample in KDE_CHUNK chunks (DESIGN.md §10), / constant."""
        x = np.asarray(x, f64)
        total = np.full(len(x), -0.0)
        with np.errstate(all="ignore"):
            for c0 in range(0, len(self.sample), KDE_CHUNK):
                s = self.sample[c0:c0 + KDE_CHUNK]
                u = (x[None, :] - s[:, None]) / self.bandwidth
                k = exp(-0.5 * (u * u))                                                # kde.rs:34-36, powi(2) is u * u
                acc = np.zeros(len(x))
                for row in k:                                                          # the fold, sample by sample
                    acc = acc + row
                total = total + acc
            return total / self.constant


class Estimator:
    """kde.rs:139-169."""

    def __init__(self, bins, min_score, score_step):
        self.bins, self.min_score, self.score_step = np.asarray(bins, f64), min_score, score_step

    def posterior_error(self, score):
        score = np.asarray(score, f64)
        last = len(self.bins) - 1                                                      # bins.len().saturating_sub(1); bins >= 100 here
        with np.errstate(all="ignore"):
            t = np.floor((score - self.min_score) / self.score_step)
            # `as usize` saturates (NaN and negatives to 0, past the range to usize::MAX), then .min(last)
            lo = np.where(~(t >= 0), 0, np.minimum(t, last)).astype(np.int64)
            hi = np.minimum(last, lo + 1)
            lower, upper = self.bins[lo], self.bins[hi]
            lo_score = lo.astype(f64) * self.score_step + self.min_score
            linear = (score - lo_score) / self.score_step
            return lower + (upper - lower) * linear


def kde_build(scores, decoy, bins=1000, monotonic=True, bw_adjust=lambda x: x):
    """Builder::build (kde.rs:83-136): (bins, min_score, score_step)."""
    scores = np.asarray(scores, f64)
    decoy = np.asarray(decoy, bool)
    d, t = scores[decoy], scores[~decoy]
    pi = div(len(d), len(scores))
    kd, kt = Kde(d, bw_adjust), Kde(t, bw_adjust)
    mn, mx = F64_MAX, -F64_MAX
    for s in scores.tolist():                                                          # kde.rs:104-109
        mn, mx = rust_min_plain(mn, s), rust_max(mx, s)
    step = div(mx - mn, bins - 1)
    with np.errstate(all="ignore"):
        x = np.arange(bins, dtype=f64) * step + mn
        dec = kd.pdf(x) * pi
        tar = kt.pdf(x) * (1.0 - pi)
        out = dec / (tar + dec)
    if monotonic:                                                                      # kde.rs:122-129
        acc = float(out[-1])
        for i in range(bins - 1, -1, -1):
            acc = rust_max(acc, float(out[i]))
            out[i] = acc
    return out, mn, step


# ---------------------------------------------------------------------------------------------------- matrix.rs, gauss.rs
def gauss_solve_inner(left, right, eps):
    """gauss.rs:27-40 on copies of the row-major matrices (numpy [rows, cols]); the solution as a flat vector, or None."""
    l, r = np.array(left, f64), np.array(right, f64)
    m, n = l.shape
    with np.errstate(all="ignore"):
        for i in range(n):                                                             # fill_zero, gauss.rs:59-63
            l[i, i] += eps
        h = k = 0
        while h < m and k < n:                                                         # echelon, gauss.rs:85-124
            best_i, best_v = 0, -F64_MAX
            for i in range(h, m):
                if l[i, k] >= best_v:
                    best_i, best_v = i, l[i, k]
            i = best_i
            if l[i, k] == 0.0:
                k += 1
                continue
            if h != i:
                l[[h, i]] = l[[i, h]]
                r[[h, i]] = r[[i, h]]
            for i2 in range(h + 1, m):
                factor = l[i2, k] / l[h, k]
                l[i2, k] = 0.0
                l[i2, k + 1:n] -= l[h, k + 1:n] * factor
                r[i2, :] -= r[h, :] * factor
            h += 1
            k += 1
        for i in range(m - 1, -1, -1):                                                 # reduce, gauss.rs:127-143
            for j in range(n):
                x = l[i, j]
                if x == 0.0:
                    continue
                l[i, j:] /= x
                r[i, :] /= x
                break
        for i in range(m - 1, -1, -1):                                                 # backfill, gauss.rs:146-164
            for j in range(n):
                if l[i, j] == 0.0:
                    continue
                for k2 in range(i):
                    factor = l[k2, j] / l[i, j]
                    l[k2, :] -= l[i, :] * factor
                    r[k2, :] -= r[i, :] * factor
                break
    for i in range(n):                                                                 # left_solved, gauss.rs:66-83
        for j in range(n):
            x = l[i, j]
            if i == j:
                if x != 1.0 and x != 0.0:
                    return None
            elif x > 1e-8:
                return None
    return r.ravel()


def gauss_solve(left, right):
    """gauss.rs:42-51: the eps ladder 1e-8, 1e-7, ... while eps <= 1.0. Returns (solution, eps) or None."""
    eps = 1e-8
    while eps <= 1.0:
        x = gauss_solve_inner(left, right, eps)
        if x is not None:
            return x, eps
        eps *= 10.0
    return None


# ---------------------------------------------------------------------------------------------------- linear_discriminant.rs, qvalue.rs
def lda_train(X, decoy):
    """LinearDiscriminantAnalysis::train (linear_discriminant.rs:63-124) over the rows of X: (coef, eps) or None."""
    with np.errstate(all="ignore"):
        return _lda_train(np.asarray(X, f64), np.asarray(decoy, bool))


def _lda_train(X, decoy):
    D = X.shape[1]
    cls = [np.nonzero(decoy)[0], np.nonzero(~decoy)[0]]                                # 0 = decoy, 1 = target
    if len(cls[0]) == 0 or len(cls[1]) == 0:                                           # :82-84
        return None
    means = []
    for c in (0, 1):                                                                   # :74-81, each class sum in row order from 0.0
        s = np.zeros(D)
        for row in X[cls[c]]:
            s = s + row
        means.append(s / f64(len(cls[c])))                                             # :85-91
    scatter = []
    for c in (0, 1):                                                                   # :95-105
        S = np.zeros((D, D))
        cen = X[cls[c]] - means[c]
        for blk in range(0, len(cen), 4096):
            prod = cen[blk:blk + 4096, :, None] * cen[blk:blk + 4096, None, :]
            for p in prod:
                S = S + p
        scatter.append(S)
    sw = np.zeros((D, D))
    for c in (0, 1):                                                                   # :107-110
        sw = sw + scatter[c] / f64(len(cls[c]))
    mu_diff = means[1] - means[0]                                                      # :116-118
    return gauss_solve(sw, mu_diff.reshape(D, 1))                                      # :119


def lda_score(coef, X):
    """LinearDiscriminantAnalysis::score (:127-130) of every row: Σ w * x from -0.0, in feature order."""
    X = np.asarray(X, f64)
    s = np.full(len(X), -0.0)
    for j in range(X.shape[1]):
        s = s + coef[j] * X[:, j]
    return s


def q_reference(disc, label):
    """qvalue.rs:8-36 after runner.rs:289's descending total_cmp sort (stable): (spectrum_q by row, passing, order). The counts are i32 and are
    cast to f32 before the division."""
    disc = np.asarray(disc, f32)
    order = np.argsort(-total_key32(disc), kind="stable")
    dec = np.cumsum(label[order] == -1).astype(np.int64)
    tar = np.arange(1, len(disc) + 1) - dec
    with np.errstate(divide="ignore"):
        q = ((1 + dec).astype(np.int32).astype(f32) / tar.astype(np.int32).astype(f32)).astype(f32)
    qmin = np.minimum(np.minimum.accumulate(q[::-1])[::-1], f32(1.0))
    out = np.empty_like(qmin)
    out[order] = qmin
    return out, int((qmin <= f32(0.01)).sum()), order.astype(np.uint32)


def clamp(x, lo, hi):
    """f64::clamp: NaN passes."""
    x = np.array(x, f64)
    x[x < lo] = lo
    x[x > hi] = hi
    return x


def feature_rows(rows, kind, mass_model, aligned_rt=None, delta_rt_model=None, delta_ims_model=None):
    """compute_features (linear_discriminant.rs:162-193) for every row: [n, 20]."""
    n = len(rows)
    X = np.zeros((n, FEATURES))
    poisson = log1p(-rows["poisson"])                                                  # :163-166
    poisson[~np.isfinite(poisson)] = 3.5
    X[:, 0] = rows["rank"]
    X[:, 1] = rows["charge"]
    X[:, 2] = log1p(rows["hyperscore"])
    X[:, 3] = log1p(rows["delta_next"])
    X[:, 4] = log1p(rows["delta_best"])
    X[:, 5] = mass_model.posterior_error(mass_error(rows, kind))
    X[:, 6] = rows["isotope_error"].astype(f64)
    X[:, 7] = rows["average_ppm"].astype(f64)
    X[:, 8] = poisson
    X[:, 9] = log1p(rows["matched_intensity_pct"].astype(f64))
    X[:, 10] = rows["matched_peaks"].astype(f64)                                      # :182: not ln_1p, whatever FEATURE_NAMES says
    X[:, 11] = log1p(rows["longest_b"].astype(f64))
    X[:, 12] = log1p(rows["longest_y"].astype(f64))
    with np.errstate(all="ignore"):
        X[:, 13] = rows["longest_y"].astype(f64) / rows["peptide_len"].astype(f64)    # :185: not the f32 longest_y_pct
    X[:, 14] = log1p(rows["peptide_len"].astype(f64))
    X[:, 15] = rows["missed_cleavages"].astype(f64)
    X[:, 16] = (rows["rt"] if aligned_rt is None else np.asarray(aligned_rt, f32)).astype(f64)   # Feature::aligned_rt defaults to the rt
    X[:, 17] = rows["ims"].astype(f64)
    for j, col in ((18, delta_rt_model), (19, delta_ims_model)):                       # :190-191, Feature default 0.999
        v = np.full(n, f32(0.999)) if col is None else np.asarray(col, f32)
        X[:, j] = np.sqrt(clamp(v.astype(f64), 0.001, 0.999))
    return X


def mass_error(rows, kind):
    """linear_discriminant.rs:140-144: delta_mass (Ppm), or the f32 difference expmass - calcmass (Da), widened to f64."""
    if kind == PPM:
        return rows["delta_mass"].astype(f64)
    return (rows["expmass"] - rows["calcmass"]).astype(f32).astype(f64)


def mass_bins(kind, lo, hi) -> int:
    """linear_discriminant.rs:146-150, 157: (hi - lo).max(100 | 1000) in f32, then .ceil().abs() as usize."""
    lo, hi = f32(lo), f32(hi)
    span = f32(hi - lo)
    floor_ = f32(100.0) if kind == PPM else f32(1000.0)
    span = floor_ if (math.isnan(span) or span < floor_) else span                    # f32::max: NaN yields the other operand
    return int(abs(math.ceil(float(span))))


def spectrum_fdr(rows, tol, aligned_rt=None, delta_rt_model=None, delta_ims_model=None, with_features=False) -> dict:
    """runner.rs:280-291: score_psms (linear_discriminant.rs:133-231), the heuristic fallback, the descending sort and spectrum_q_value. The
    same keys as sage_b200.spectrum_fdr's outputs."""
    rows = np.asarray(rows)
    n = len(rows)
    kind = tol.kind
    assert kind in (PPM, DA), "Pct is unreachable in score_psms"
    decoy = rows["label"] == -1                                                        # :135-138
    bw = 2.0 if kind == PPM else 0.1                                                   # :146-150
    dm = mass_error(rows, kind)
    mass_model = Estimator(*kde_build(dm, decoy, mass_bins(kind, tol.lo, tol.hi), False, lambda x: x * bw))   # :154-158
    X = feature_rows(rows, kind, mass_model, aligned_rt, delta_rt_model, delta_ims_model)
    fit = lda_train(X, decoy)                                                          # :195
    coef, eps = np.zeros(FEATURES), 0.0
    fitted = fit is not None and bool(np.isfinite(fit[0]).all())                       # :196-208
    pep = np.ones(n, f32)                                                              # Feature::posterior_error default
    if fitted:
        coef, eps = fit
        scores = lda_score(coef, X)                                                    # :209-212
        kde = Estimator(*kde_build(scores, decoy))                                     # :215, Builder::default()
        disc = scores.astype(f32)                                                      # :221
        with np.errstate(all="ignore"):
            pep = log10(kde.posterior_error(scores)).astype(f32)                       # :222
        pep[np.isinf(pep)] = f32(-324.0)                                               # :223-227
    else:                                                                              # runner.rs:284-287
        with np.errstate(all="ignore"):
            disc = log1pf((-rows["poisson"]).astype(f32)) + rows["longest_y_pct"] / f32(3.0)
    q, passing, order = q_reference(disc, rows["label"])                               # runner.rs:289-290
    out = dict(discriminant_score=disc.astype(f32), posterior_error=pep.astype(f32), spectrum_q=q, order=order, passing=passing,
               lda_fitted=fitted, coef=np.asarray(coef, f64) if fitted else np.zeros(FEATURES), eps=eps if fitted else 0.0)
    if with_features:
        out["features"] = X
    return out


# ---------------------------------------------------------------------------------------------------- retention_alignment.rs
def poisson_order_and_q(rows):
    """runner.rs:519-522: the ascending total_cmp sort of poisson (stable) and spectrum_q_value over it, as a loop: (order, q by row)."""
    order = np.argsort(total_key64(rows["poisson"]), kind="stable")
    dec, tar, qs = 1, 0, []
    for r in order:
        if rows["label"][r] == -1:
            dec += 1
        else:
            tar += 1
        qs.append(f32(dec) / f32(tar))
    q = np.zeros(len(rows), f32)
    qm = f32(1.0)
    for p in range(len(order) - 1, -1, -1):
        qm = min(qm, qs[p])
        q[order[p]] = qm
    return order, q


def ceil_as_u32(x: float) -> int:
    """`rt.ceil() as u32` (retention_alignment.rs:33): saturating, NaN to 0."""
    if math.isnan(x):
        return 0
    if math.isinf(x):
        return 0 if x < 0 else 2**32 - 1
    return min(max(math.ceil(x), 0), 2**32 - 1)


def global_alignment(rows, fid, n_files, order, q):
    """retention_alignment.rs:95-173 over rows in poisson order: (alignments [(max_rt, slope, intercept) as f32], matrix rows kept)."""
    max_rt = [0] * n_files                                                             # :26-40
    for i in range(len(rows)):
        max_rt[fid[i]] = max(max_rt[fid[i]], ceil_as_u32(float(rows["rt"][i])))
    max_rt = [float(v) for v in max_rt]
    mins = {}                                                                          # :44-57, in poisson order
    for r in order:
        if rows["label"][r] == 1 and q[r] <= f32(0.01):
            k = (int(rows["peptide_idx"][r]), int(fid[r]))
            x = float(rows["rt"][r])
            mins[k] = x if k not in mins else rust_min(mins[k], x)
    by_pep = {}
    for (p, f), v in mins.items():
        by_pep.setdefault(p, []).append((f, v))
    mat = []
    for pep in sorted(by_pep):                                                         # :59-85, ascending PeptideIx
        v = [math.nan] * n_files
        s, n = 0.0, 0.0
        for f, rt in sorted(by_pep[pep]):                                              # ascending file
            v[f] = div(rt, max_rt[f])
            s += v[f]
            n += 1.0
        m = div(s, n)
        if math.isfinite(m) and abs(m) >= 2.2250738585072014e-308:                    # f64::is_normal
            mat.append(v)
    means = []                                                                         # :99-109
    for v in mat:
        ln, s = 0, 0.0
        for x in v:
            if math.isfinite(x):
                ln, s = ln + 1, s + x
        means.append(div(s, ln))
    out = []
    for f in range(n_files):                                                           # :112-159
        n, dot, sx, sy = 0, 0.0, 0.0, 0.0
        for v, y in zip(mat, means):
            if math.isfinite(v[f]):
                n, dot, sx, sy = n + 1, dot + v[f] * y, sx + v[f], sy + y
        xm, ym = div(sx, n), div(sy, n)
        ssxy = dot - n * xm * ym
        sx2 = 1e-8
        for v in mat:
            if math.isfinite(v[f]):
                d = v[f] - xm
                sx2 = sx2 + d * d
        slope = div(ssxy, sx2)
        icpt = ym - slope * xm
        slope = slope if math.isfinite(slope) else 1.0
        icpt = icpt if math.isfinite(icpt) else 0.0
        with np.errstate(all="ignore"):
            out.append((f32(max_rt[f]), f32(slope), f32(icpt)))
    return out, len(mat)


def py_alignment(rows, fid, n_files):
    """The alignments of global_alignment after the runner's poisson sort and q-values (runner.rs:517-527)."""
    order, q = poisson_order_and_q(rows)
    return global_alignment(rows, fid, n_files, order, q)[0]


# ---------------------------------------------------------------------------------------------------- retention_model.rs, mobility_model.rs
RT_D = len(VALID_AA) * 3 + 3                                                           # retention_model.rs:32
IMS_D = len(VALID_AA) * 4 + 12                                                         # mobility_model.rs:75
_MAP = [0] * 26                                                                        # retention_model.rs:64-67: other letters stay 0
for _i, _a in enumerate(VALID_AA):
    _MAP[_a - ord("A")] = _i


def rt_embed(seq: bytes, mono) -> np.ndarray:
    """RetentionModel::embed (retention_model.rs:42-59)."""
    NT, CT = len(VALID_AA), len(VALID_AA) * 2
    e = np.zeros(RT_D)
    cterm = max(len(seq) - 3, 0)                                                       # saturating_sub(3)
    for i, res in enumerate(seq):
        assert ord("A") <= res <= ord("Z")
        idx = _MAP[res - ord("A")]
        e[idx] += 1.0
        if i in (0, 1):
            e[NT + idx] += 1.0
        elif i == cterm or i == cterm + 1:
            e[CT + idx] += 1.0
    e[RT_D - 3] = float(len(seq))
    e[RT_D - 2] = _libm.log1p(float(f32(mono)))                                        # ln_1p of the f32 mass widened
    e[RT_D - 1] = 1.0
    return e


_GROUPS = dict(bulky=b"LVIFWY", polar=b"STNQ", positive=b"RKH", negative=b"DE", tiny=b"GAS", branched=b"LIV")   # mobility_model.rs:39-73


def ims_embed(seq: bytes, mono, charge: int) -> np.ndarray:
    """MobilityModel::embed (mobility_model.rs:97-149). The group constants are letter offsets (b'L' - b'A'), compared as written with the
    residue's VALID_AA position."""
    F, PCT, NT, CT = IMS_D, len(VALID_AA), len(VALID_AA) * 2, len(VALID_AA) * 3
    slot = dict(branched=F - 12, tiny=F - 11, polar=F - 10, bulky=F - 9, positive=F - 8, negative=F - 7)
    groups = {g: {c - ord("A") for c in letters} for g, letters in _GROUPS.items()}
    e = np.zeros(IMS_D)
    cterm = max(len(seq) - 3, 0)
    for i, res in enumerate(seq):
        assert ord("A") <= res <= ord("Z")
        idx = _MAP[res - ord("A")]
        e[idx] += 1.0
        if i in (0, 1):
            e[NT + idx] += 1.0
        elif i > cterm:
            e[CT + idx] += 1.0
        for g, members in groups.items():
            if idx in members:
                e[slot[g]] += 1.0
    with np.errstate(all="ignore"):
        plen = f64(len(seq))
        for idx in range(len(VALID_AA)):                                               # :136-139
            e[PCT + idx] = f64(e[idx]) / plen
        z = f64(charge & 0xFF)                                                         # Feature::charge is a u8
        m = f64(f32(mono))
        e[F - 5] = z
        e[F - 6] = f64(1.0) / z
        e[F - 3] = plen
        e[F - 2] = m / 1000.0
        e[F - 4] = (m / z) / 1000.0
    e[F - 1] = 1.0
    return e


def linreg_fit(X, y):
    """LinearRegression::fit (regression.rs:72-117) over rows that all pass the filter, in order: (beta, r2, eps) or None."""
    X, y = np.asarray(X, f64), np.asarray(y, f64)
    n, d = X.shape
    if n == 0:                                                                         # :91-93
        return None
    tot_cov, tot_b, tot_y, tot_y2 = np.zeros((d, d)), np.zeros(d), 0.0, 0.0           # reduce identity Acc::zero
    with np.errstate(all="ignore"):
        for c0 in range(0, n, RT_CHUNK):                                               # fold per chunk (DESIGN.md §11), Acc::add_row :38-51
            cov, b, sy, sy2 = np.zeros((d, d)), np.zeros(d), 0.0, 0.0
            for row, t in zip(X[c0:c0 + RT_CHUNK], y[c0:c0 + RT_CHUNK].tolist()):
                b = b + row * t
                cov = cov + row[:, None] * row[None, :]
                sy += t
                sy2 += t * t
            tot_cov, tot_b, tot_y, tot_y2 = tot_cov + cov, tot_b + b, tot_y + sy, tot_y2 + sy2   # Acc::merge :53-64
    nf = float(n)
    y_mean = div(tot_y, nf)
    y_var = tot_y2 - nf * y_mean * y_mean                                              # :97
    sol = gauss_solve(tot_cov, tot_b.reshape(d, 1))
    if sol is None:
        return None
    beta, eps = sol
    with np.errstate(all="ignore"):
        pred = np.full(n, -0.0)                                                        # :109, a Sum from -0.0
        for j in range(d):
            pred = pred + X[:, j] * beta[j]
        diff = pred - y
        sq = (diff * diff).tolist()
    sse = -0.0
    for c0 in range(0, n, RT_CHUNK):                                                   # :104-113, chunk sums from -0.0 in order
        s = -0.0
        for v in sq[c0:c0 + RT_CHUNK]:
            s += v
        sse += s
    return beta, 1.0 - div(sse, y_var), eps


def predict_peptide(E, beta, hi):
    """predict_peptide (retention_model.rs:85-90, mobility_model.rs:175-180), a fold from 0.0, then clamp(0, hi) as f32 (:20, :26)."""
    v = np.zeros(len(E))
    with np.errstate(all="ignore"):
        for j in range(E.shape[1]):
            v = v + E[:, j] * beta[j]
    return clamp(v, 0.0, hi).astype(f32)


def predict_rt(peptides, rows, file_id, n_files) -> dict:
    """runner.rs:513-531: the poisson sort, spectrum_q_value, global_alignment, retention_model::predict and mobility_model::predict. The same
    keys as sage_b200.predict_rt's outputs."""
    from sage_b200.api import ALIGNMENT_DTYPE
    rows = np.asarray(rows)
    fid = np.asarray(file_id, np.int64)
    n = len(rows)
    order, q = poisson_order_and_q(rows)
    align, kept = global_alignment(rows, fid, n_files, order, q)
    a = np.array(align, f32).reshape(-1, 3)
    with np.errstate(all="ignore"):
        aligned_rt = ((rows["rt"] / a[fid, 0]) * a[fid, 1] + a[fid, 2]).astype(f32)   # retention_alignment.rs:163-170
    train = np.array([r for r in order if rows["label"][r] == 1 and q[r] <= f32(0.01)], np.int64)   # regression filter, poisson order
    off = np.asarray(peptides.seq_off, np.int64)
    seq = np.asarray(peptides.seq, np.uint8)
    mono = np.asarray(peptides.mono, f32)
    out = dict(aligned_rt=aligned_rt, spectrum_q=q, alignments=a.view(ALIGNMENT_DTYPE).reshape(-1), training_rows=len(train), aligned_peptides=kept)
    charge = rows["charge"].astype(np.int64) & 0xFF
    for name, d, hi in (("rt", RT_D, 1.0), ("ims", IMS_D, 2.0)):
        key = rows["peptide_idx"].astype(np.int64) if name == "rt" else rows["peptide_idx"].astype(np.int64) * 256 + charge
        uk, inv = np.unique(key, return_inverse=True)
        E = np.zeros((len(uk), d))
        for i, k in enumerate(uk.tolist()):
            p = k if name == "rt" else k >> 8
            s = seq[off[p]:off[p + 1]].tobytes()
            E[i] = rt_embed(s, mono[p]) if name == "rt" else ims_embed(s, mono[p], k & 0xFF)
        target = aligned_rt if name == "rt" else rows["ims"]                          # retention_model.rs:73, mobility_model.rs:163
        fit = linreg_fit(E[inv[train]], target[train].astype(f64)) if len(train) else None
        pred, delta = np.zeros(n, f32), np.full(n, f32(0.999))                         # Feature defaults when predict returns None
        beta, r2, eps = np.zeros(d), 0.0, 0.0
        if fit is not None:
            beta, r2, eps = fit
            pred = predict_peptide(E, beta, hi)[inv]
            with np.errstate(all="ignore"):
                delta = np.abs(target - pred).astype(f32)                              # retention_model.rs:22, mobility_model.rs:29
        out.update({f"predicted_{name}": pred, f"delta_{name}_model": delta, f"{name}_fitted": fit is not None, f"{name}_r2": r2,
                    f"{name}_eps": eps, f"{name}_beta": np.asarray(beta, f64)})
    return out
