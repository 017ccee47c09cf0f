"""The CPU oracle of rescoring and RT / mobility prediction (oracle_ml/) against the independent numpy restatement of Sage's ml/ modules
(tests/ml_reference.py), bit for bit (NaN payloads aside): every output of spectrum_fdr including the 20-feature rows, and every output of
predict_rt, on each workload of tests/fdr_cases.py and tests/rt_cases.py of at most 10^5 rows; kde_build, LDA training, the embeddings and the
regression alone; and the reference's own known answers (linear_discriminant.rs, regression.rs, mobility_model.rs) through the restatement."""
import math

import numpy as np
import pytest

import fdr_cases
import ml_reference as R
import rt_cases
from oracle_ml import ml_oracle
from sage_b200 import Tolerance

MAX_ROWS = 100_000   # the 10^6-row workloads are checked against the oracle only (tests/test_gpu_*.py)
FDR_ROW_KEYS = ("discriminant_score", "posterior_error", "spectrum_q", "order")
RT_COLUMNS = ("aligned_rt", "predicted_rt", "delta_rt_model", "predicted_ims", "delta_ims_model", "spectrum_q")


def same_bits(a, b):
    """Bit for bit, except that any two NaNs match."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    w = {8: np.uint64, 4: np.uint32}[a.dtype.itemsize]
    eq = a.view(w) == b.view(w)
    if a.dtype.kind == "f":
        eq |= np.isnan(a) & np.isnan(b)
    return eq


def assert_fdr_same(got, want, what):
    for k in FDR_ROW_KEYS + ("coef",) + (("features",) if "features" in want else ()):
        eq = same_bits(got[k], want[k])
        assert eq.all(), f"{what}: {k} differs at {np.argwhere(~eq)[:5].tolist()}"
    for k in ("passing", "lda_fitted", "eps"):
        assert got[k] == want[k], f"{what}: {k} {got[k]} != {want[k]}"


def assert_rt_same(got, want, what):
    for k in RT_COLUMNS + ("rt_beta", "ims_beta"):
        eq = same_bits(got[k], want[k])
        assert eq.all(), f"{what}: {k} differs at {np.nonzero(~eq)[0][:5].tolist()}"
    assert same_bits(got["alignments"].view(np.float32), want["alignments"].view(np.float32)).all(), f"{what}: alignments"
    for k in ("training_rows", "aligned_peptides", "rt_fitted", "rt_eps", "ims_fitted", "ims_eps"):
        assert got[k] == want[k], f"{what}: {k} {got[k]} != {want[k]}"
    for k in ("rt_r2", "ims_r2"):
        assert same_bits(np.float64([got[k]]), np.float64([want[k]])).all(), f"{what}: {k} {got[k]} != {want[k]}"


_FDR = {k: v for k, v in fdr_cases.cases().items() if len(v["rows"]) <= MAX_ROWS}
_RT = {k: v for k, v in rt_cases.cases().items() if len(v["rows"]) <= MAX_ROWS}
FALLBACK = {"no_decoys", "no_targets", "nan_delta_next", "q_at_threshold", "one_decoy", "one_target", "mass_nan_ppm", "mass_inf_ppm",
            "mass_nonfinite_da", "mass_inf_da", "hyperscore_minus_one"}


@pytest.mark.parametrize("name", sorted(_FDR))
def test_spectrum_fdr_matches_oracle(name):
    c = dict(_FDR[name])
    rows, tol = c.pop("rows"), c.pop("tol")
    got = R.spectrum_fdr(rows, tol, with_features=True, **c)
    assert_fdr_same(got, ml_oracle.spectrum_fdr(rows, tol, with_features=True, **c), name)
    if name in FALLBACK or name.startswith(("lda_", "kde_", "tol_", "mass_on")):       # each edge workload reaches the branch it was built for
        assert got["lda_fitted"] == (name not in FALLBACK), name
    if name.startswith(("mass_", "one_")) and name != "mass_on_bin_points":
        assert np.isnan(got["features"][:, 5]).all()                                  # a NaN mass-error estimator
    if name == "mass_on_bin_points":
        dm = rows["delta_mass"].astype(np.float64)
        assert (got["features"][:, 5] == R.Estimator(*R.kde_build(dm, rows["label"] == -1, 100, False, lambda x: x * 2.0)).bins[dm.astype(int)]).all()


@pytest.mark.parametrize("name", sorted(_RT))
def test_predict_rt_matches_oracle(name):
    c = _RT[name]
    got = R.predict_rt(c["pep"], c["rows"], c["file_id"], c["n_files"])
    assert_rt_same(got, ml_oracle.predict_rt(c["pep"], c["rows"], c["file_id"], c["n_files"]), name)
    if name.startswith("predict_rows_"):
        assert got["training_rows"] == int(name.split("_")[-1]) and got["rt_fitted"] and got["ims_fitted"]
    if name == "clamps":
        p, q = got["predicted_rt"], got["predicted_ims"]
        assert (p == 0).any() and (p == 1).any() and (q == 0).any() and (q == 2).any()
    if name == "charges_u8":
        assert got["ims_fitted"] and np.isnan(got["predicted_ims"][c["rows"]["label"] == -1][::2]).all()   # z = 0: 1/z = inf
    if name == "charges_zero_trained":
        assert got["rt_fitted"] and not got["ims_fitted"]
    if name == "ims_nan_target":
        assert got["ims_fitted"] and np.isnan(got["ims_beta"]).all() and np.isnan(got["predicted_ims"]).all()
    if name == "one_segment":
        assert got["aligned_peptides"] == 1 and got["alignments"]["slope"][1] == 0


def test_mass_bins():
    """linear_discriminant.rs:146-157: (hi - lo).max(100 | 1000) in f32, ceil, abs."""
    for tol, bins in ((Tolerance.ppm(-20, 20), 100), (Tolerance.ppm(-50.25, 50.5), 101), (Tolerance.ppm(30, -30), 100), (Tolerance.ppm(-150, 150), 300),
                      (Tolerance.da(-0.5, 0.5), 1000), (Tolerance.da(-1000.4, 1000.4), 2001), (Tolerance.ppm(0, 1 << 24), 1 << 24)):
        assert R.mass_bins(tol.kind, tol.lo, tol.hi) == bins, tol


@pytest.mark.parametrize("monotonic,bw", [(True, 1.0), (False, 2.0), (False, 0.1)])
def test_kde_build_matches_oracle(monotonic, bw):
    """Builder::build on scores that lie exactly on the bin points (min_score and max_score repeated), with one decoy (bandwidth 0) and on a
    sample of 2 x 4096 + 1 scores."""
    rng = np.random.default_rng(42)
    s2 = np.concatenate([rng.normal(0, 1, 4097), rng.normal(3, 2, 4096)])
    for s, d in list(fdr_cases.kde_samples().values()) + [(s2, rng.random(len(s2)) < 0.5)]:
        got = R.kde_build(s, d, 1000, monotonic, lambda x: x * bw)
        want = ml_oracle.kde_build(s, d, 1000, monotonic, bw)
        assert same_bits(got[0], want[0]).all() and got[1:] == want[1:]


def test_lda_known_answer():
    """linear_discriminant.rs:248-287 through the restatement, and its coefficients equal the oracle's."""
    X = np.array([[5., 4., 3., 2.], [4., 5., 4., 3.], [6., 3., 4., 5.], [1., 0., 2., 9.], [5., 4., 4., 3.], [2., 1., 1., 9.5], [1., 0., 2., 8.], [3., 2., -2., 10.]])
    decoy = np.array([0, 0, 0, 1, 0, 1, 1, 1], bool)
    coef, eps = R.lda_train(X, decoy)
    s = R.lda_score(coef, X)
    norm = 0.0
    for v in s:                                                                        # ml/mod.rs:20-22
        norm = norm + v * v
    s = s / math.sqrt(norm)
    expected = [0.49706043, 0.48920177, 0.48920177, -0.07209359, 0.51204672, -0.02849527, -0.04924864, -0.06055943]
    assert all(abs(a - b) <= 1e-8 for a, b in zip(s, expected)), s
    oc, oe = ml_oracle.lda_train(X, decoy)
    assert same_bits(coef, oc).all() and eps == oe == 1e-8


def test_fit_perfect_line():   # regression.rs:124-133
    x = np.arange(50.0)
    X, y = np.stack([x, np.ones(50)], 1), 2 * x + 1
    beta, r2, eps = R.linreg_fit(X, y)
    assert abs(beta[0] - 2) < 1e-9 and abs(beta[1] - 1) < 1e-9 and abs(r2 - 1) < 1e-9
    ob, or2, oe = ml_oracle.linreg_fit(X, y)
    assert same_bits(beta, ob).all() and same_bits(np.float64([r2]), np.float64([or2])).all() and eps == oe


def test_fit_with_noise():     # regression.rs:135-150
    i = np.arange(200.0)
    x = i / 10.0
    y = 3 * x + 2 + np.array([math.sin(v * 0.7) for v in i]) * 0.1
    X = np.stack([x, np.ones(200)], 1)
    beta, r2, eps = R.linreg_fit(X, y)
    assert abs(beta[0] - 3) < 0.05 and abs(beta[1] - 2) < 0.1 and r2 > 0.99
    ob, or2, oe = ml_oracle.linreg_fit(X, y)
    assert same_bits(beta, ob).all() and same_bits(np.float64([r2]), np.float64([or2])).all() and eps == oe


def test_empty_filter_returns_none():   # regression.rs:152-157
    assert R.linreg_fit(np.zeros((0, 1)), np.zeros(0)) is None


def test_linreg_chunks_match_oracle():
    """RT_CHUNK - 1 .. 2 RT_CHUNK + 1 rows of a 7-column design: the chunked fold, the merge and the SSE."""
    rng = np.random.default_rng(7)
    for n in (1023, 1024, 1025, 2049):
        X = np.concatenate([rng.normal(0, 1, (n, 6)), np.ones((n, 1))], 1)
        y = X @ rng.normal(0, 1, 7) + rng.normal(0, 0.1, n)
        beta, r2, eps = R.linreg_fit(X, y)
        ob, or2, oe = ml_oracle.linreg_fit(X, y)
        assert same_bits(beta, ob).all() and same_bits(np.float64([r2]), np.float64([or2])).all() and eps == oe, n


def test_feature_embed():      # mobility_model.rs:188-266
    e = [R.ims_embed(s.encode(), 1000.0, 2) for s in ("LEKSLIEK", "LERSLIEWK", "LWESLIEK", "CHADWICK")]
    nt, ct = 44, 66
    ix = {a: R.VALID_AA.index(a.encode()) for a in "KWLI"}
    assert [x[nt + ix["L"]] for x in e] == [1, 1, 1, 0]
    assert [x[nt + ix["K"]] for x in e] == [0, 0, 0, 0]
    assert [x[nt + ix["W"]] for x in e] == [0, 0, 1, 0]
    assert [x[ct + ix["K"]] for x in e] == [1, 1, 1, 1]
    assert [x[ct + ix["W"]] for x in e] == [0, 1, 0, 0]
    assert [x[ct + ix["I"]] for x in e] == [0, 0, 0, 0]


def test_embeddings_match_oracle():
    """Both embeddings of odd sequences, lengths 1 .. 255 and charges whose low byte is 0, 1 or 255."""
    rng = np.random.default_rng(8)
    letters = list("ACDEFGHIKLMNPQRSTVWYUOBJXZ")
    seqs = ["".join(rng.choice(letters, n)) for n in (1, 2, 3, 4, 31, 32, 33, 64, 65, 255)] + ["LEKSLIEK", "NOKGLVIFWY", "BJXZ"]
    for s in seqs:
        mono = float(np.float32(rng.uniform(100.0, 30000.0)))
        assert same_bits(R.rt_embed(s.encode(), mono), ml_oracle.rt_embed(0, s, mono)).all(), s
        for z in (0, 1, 2, 255, 256, 257):
            assert same_bits(R.ims_embed(s.encode(), mono, z), ml_oracle.rt_embed(1, s, mono, z)).all(), (s, z)
