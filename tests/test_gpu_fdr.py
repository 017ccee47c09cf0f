"""GPU: rescoring on the device (sage_b200.spectrum_fdr) is bit-identical to the CPU oracle (oracle_ml) on every output."""
import ctypes

import numpy as np
import pytest

import ml_reference
from fdr_cases import cases, kde_samples
from ml_reference import q_reference
from oracle_ml import ml_oracle
from sage_b200 import Tolerance, api, synth

pytestmark = pytest.mark.gpu
KEYS = ("discriminant_score", "posterior_error", "spectrum_q", "order")
RESTATED_ROWS = 100_000   # the numpy restatement (tests/ml_reference.py) is checked up to this size


def same_bits(a, b):
    """Bit for bit, except that any two NaNs match (the device and the host CPU write different NaN payloads)."""
    w = np.uint64 if a.dtype.itemsize == 8 else np.uint32
    eq = a.view(w) == b.view(w)
    if a.dtype.kind == "f":
        eq |= np.isnan(a) & np.isnan(b)
    return eq


def assert_same(got, want, what):
    for k in KEYS:
        eq = same_bits(got[k], want[k])
        assert eq.all(), f"{what}: {k} differs at {np.nonzero(~eq)[0][:5]}"
    assert got["passing"] == want["passing"] and got["lda_fitted"] == want["lda_fitted"], what
    assert same_bits(got["coef"], want["coef"]).all() and got["eps"] == want["eps"], what


_CASES = cases()


@pytest.mark.parametrize("name", sorted(_CASES))
def test_edge_workloads(name):
    c = dict(_CASES[name])
    rows, tol = c.pop("rows"), c.pop("tol")
    got = api.spectrum_fdr(rows, tol, **c)
    assert_same(got, ml_oracle.spectrum_fdr(rows, tol, **c), name)
    if len(rows) <= RESTATED_ROWS:
        assert_same(got, ml_reference.spectrum_fdr(rows, tol, **c), name + " (restatement)")
    if name in ("no_decoys", "no_targets", "nan_delta_next"):
        assert not got["lda_fitted"] and (got["posterior_error"] == 1.0).all()
    if name == "psms_100000":
        assert (got["posterior_error"] == -324.0).any()   # PEP exactly 0
    if name == "da_500":
        assert got["eps"] == 1.0                           # Gauss::solve needed the last rung of the eps ladder
    if name == "all_equal":
        assert got["lda_fitted"] and (got["coef"] == 0).all() and (got["discriminant_score"] == 0).all() and np.isnan(got["posterior_error"]).all()
    if name == "q_at_threshold":
        assert got["passing"] == 100 and (got["spectrum_q"][:100] == np.float32(0.01)).all()   # passes under <= only


def test_end_to_end_search_then_fdr():
    from sage_b200 import IndexedDatabase, Scorer
    pep = synth.make_peptides(6000, seed=301, static_c=True)
    spectra = synth.make_spectra(pep, 2000, seed=302)
    sc = Scorer(IndexedDatabase.build_from_peptides(pep), precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), report_psms=3)
    f, counts = sc.score_batch(spectra)
    rows = f[(np.arange(len(f)) % 3) < np.repeat(counts, 3)]
    assert (rows["label"] == -1).sum() > 50 and (rows["label"] == 1).sum() > 50
    got = api.spectrum_fdr(rows, Tolerance.ppm(-20, 20))
    assert_same(got, ml_oracle.spectrum_fdr(rows, Tolerance.ppm(-20, 20)), "search")
    assert got["lda_fitted"]


def test_twice_identical_bytes():
    rows = synth.make_psms(50_000, seed=31)
    a, b = api.spectrum_fdr(rows, Tolerance.ppm(-20, 20)), api.spectrum_fdr(rows, Tolerance.ppm(-20, 20))
    for k in KEYS:
        assert a[k].tobytes() == b[k].tobytes()


@pytest.mark.parametrize("monotonic,bw", [(True, 1.0), (False, 2.0), (False, 0.1)])
def test_kde_build_hook(monotonic, bw):
    rng = np.random.default_rng(41)
    s = np.concatenate([rng.normal(0, 1, 30_000), rng.normal(4, 2, 50_000)])
    d = rng.random(len(s)) < 0.4
    got = api.kde_build(s, d, 1000, monotonic, bw)
    want = ml_oracle.kde_build(s, d, 1000, monotonic, bw)
    assert same_bits(got[0], want[0]).all() and got[1:] == want[1:]


@pytest.mark.parametrize("monotonic,bw", [(True, 1.0), (False, 2.0)])
@pytest.mark.parametrize("sample", sorted(kde_samples()))
def test_kde_build_samples(sample, monotonic, bw):
    """Scores exactly on the 1000 bin points (min_score and max_score repeated), and one decoy (bandwidth 0): against the oracle and the
    restatement."""
    s, d = kde_samples()[sample]
    got = api.kde_build(s, d, 1000, monotonic, bw)
    for want in (ml_oracle.kde_build(s, d, 1000, monotonic, bw), ml_reference.kde_build(s, d, 1000, monotonic, lambda x: x * bw)):
        assert same_bits(got[0], want[0]).all() and got[1:] == want[1:]


def test_mass_bins_limit():
    """A tolerance span of 2^24 - 1 mass-error bins runs and equals the oracle; 2^24 bins is refused with ELIMIT, Ppm and Da alike."""
    rows = synth.make_psms(4, seed=42)
    rows["label"] = [-1, 1, -1, 1]
    tol = Tolerance.ppm(-8388608, 8388607)
    assert_same(api.spectrum_fdr(rows, tol), ml_oracle.spectrum_fdr(rows, tol), "2^24 - 1 bins")
    for tol in (Tolerance.ppm(-8388608, 8388608), Tolerance.da(0, 1 << 24), Tolerance.ppm(0, 1 << 30)):
        with pytest.raises(api.SageB200Error) as e:
            api.spectrum_fdr(rows, tol)
        assert e.value.code == -5, tol


def test_kde_build_all_scores_equal():
    """score_step == 0: every bin evaluates at the one score, and the estimator's NaN bin index saturates to 0."""
    s = np.full(5000, 1.5)
    d = np.arange(5000) % 3 == 0
    got = api.kde_build(s, d, 1000, True, 1.0)
    want = ml_oracle.kde_build(s, d, 1000, True, 1.0)
    assert got[2] == 0.0 and got[1] == 1.5 and same_bits(got[0], want[0]).all() and got[1:] == want[1:]


@pytest.mark.parametrize("function", ["exp", "log1p", "log10"])
def test_device_math_equals_libm(function):
    """Every one of 10^6 inputs against the host libm called through ctypes: all bit patterns, exp's special-case range, KDE arguments and
    log1p's (-1, 1)."""
    rng = np.random.default_rng(51)
    n = 1_000_000
    x = np.concatenate([rng.integers(0, 1 << 64, n // 4, dtype=np.uint64).view(np.float64), (rng.random(n // 4) - 0.5) * 1500.0,
                        -0.5 * (rng.random(n // 4) * 40) ** 2, rng.random(n // 4) * 2.0 - 1.0])
    got = api.device_math(function, x)
    fn = getattr(ctypes.CDLL("libm.so.6"), function)
    fn.restype, fn.argtypes = ctypes.c_double, [ctypes.c_double]
    want = np.frompyfunc(fn, 1, 1)(x).astype(np.float64)
    same = (got.view(np.uint64) == want.view(np.uint64)) | (np.isnan(got) & np.isnan(want))
    assert same.all(), f"{int((~same).sum())} differ, e.g. x={x[~same][:3]}"


def test_q_values_past_2_24_rows():
    """2^24 + 2^20 rows: the i32 -> f32 casts of the q-value counts round. Checked against the numpy restatement of qvalue.rs on the device's own
    discriminants."""
    n = (1 << 24) + (1 << 20)
    rows = np.tile(synth.make_psms(1 << 20, seed=61), 17)[:n]
    rows["hyperscore"] += np.arange(n) % 1000 * 1e-3
    got = api.spectrum_fdr(rows, Tolerance.ppm(-20, 20))
    q, passing, order = q_reference(got["discriminant_score"], rows["label"])
    assert np.array_equal(order, got["order"]) and passing == got["passing"]
    assert np.array_equal(q.view(np.uint32), got["spectrum_q"].view(np.uint32))


def test_errors():
    rows = synth.make_psms(10, seed=1)
    with pytest.raises(api.SageB200Error) as e:
        api.spectrum_fdr(rows, Tolerance.pct(-1, 1))
    assert e.value.code == -1
    r = api.spectrum_fdr(rows[:0], Tolerance.ppm(-20, 20))
    assert r["passing"] == 0 and not r["lda_fitted"]
