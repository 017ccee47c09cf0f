"""CPU checks of the rescoring oracle (oracle_ml/ml_oracle.cpp) against the reference's known answer and independent numpy restatements, of the
host evaluation of the reproduced glibc exp / log1p / log10, and of the C header against the ctypes structs."""
import os
import subprocess

import numpy as np

from ml_reference import q_reference
from oracle_ml import ml_oracle
from sage_b200 import Tolerance, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_lda_known_answer():
    """linear_discriminant.rs:248-287: the normalised projections of the 8 x 4 example."""
    X = np.array([[5., 4., 3., 2.], [4., 5., 4., 3.], [6., 3., 4., 5.], [1., 0., 2., 9.], [5., 4., 4., 3.], [2., 1., 1., 9.5], [1., 0., 2., 8.], [3., 2., -2., 10.]])
    decoy = np.array([0, 0, 0, 1, 0, 1, 1, 1])
    coef, eps = ml_oracle.lda_train(X, decoy)
    s = X @ coef
    s = s / np.sqrt((s ** 2).sum())
    expected = [0.49706043, 0.48920177, 0.48920177, -0.07209359, 0.51204672, -0.02849527, -0.04924864, -0.06055943]
    assert np.allclose(s, expected, atol=1e-8, rtol=0), s
    assert eps == 1e-8


def test_lda_coefficients_against_numpy():
    p = synth.make_psms(20_000, seed=3)
    r = ml_oracle.spectrum_fdr(p, Tolerance.ppm(-20, 20), with_features=True)
    X, d = r["features"], p["label"] == -1
    mu_d, mu_t = X[d].mean(axis=0), X[~d].mean(axis=0)
    sw = np.cov(X[d].T, bias=True) + np.cov(X[~d].T, bias=True)
    want = np.linalg.solve(sw + r["eps"] * np.eye(20), mu_t - mu_d)
    assert r["lda_fitted"]
    assert np.allclose(r["coef"], want, rtol=1e-9, atol=1e-9 * np.abs(want).max()), (r["coef"], want)


def test_kde_bins_against_numpy():
    rng = np.random.default_rng(4)
    s = np.concatenate([rng.normal(0, 1, 9000), rng.normal(3, 1.5, 11000)])
    d = np.arange(len(s)) < 9000
    for monotonic, bw in ((True, 1.0), (False, 2.0)):
        bins, lo, step = ml_oracle.kde_build(s, d, 300, monotonic, bw)

        def pdf(x, xs):
            h = xs.std() * (4 / 3 / len(xs)) ** 0.2 * bw
            return np.exp(-0.5 * ((x[:, None] - xs[None, :]) / h) ** 2).sum(axis=1) / (np.sqrt(2 * np.pi) * h * len(xs))

        x = np.arange(300) * step + lo
        pi = d.mean()
        want = pdf(x, s[d]) * pi / (pdf(x, s[~d]) * (1 - pi) + pdf(x, s[d]) * pi)
        if monotonic:
            want = np.maximum.accumulate(want[::-1])[::-1]
        assert np.allclose(bins, want, rtol=1e-12, atol=1e-12), np.abs(bins - want).max()


def test_q_values_against_numpy():
    for seed, n in ((5, 1), (6, 50_000)):
        p = synth.make_psms(n, seed=seed)
        p = np.concatenate([p, p[: n // 3]])   # ties
        r = ml_oracle.spectrum_fdr(p, Tolerance.ppm(-20, 20))
        q, passing, order = q_reference(r["discriminant_score"], p["label"])
        assert np.array_equal(q.view(np.uint32), r["spectrum_q"].view(np.uint32)) and passing == r["passing"] and np.array_equal(order, r["order"])


def test_host_math_matches_libm(tmp_path):
    """The exp / log1p / log10 the kernels evaluate (glibc_math.cuh, compiled here for the host) equal this host's libm bit for bit on 3e6
    inputs per function: every exponent, subnormals, near 0 and 1, the special cases and the values rescoring feeds them."""
    exe = str(tmp_path / "glibc_math_check")
    subprocess.check_call(["g++", "-O2", "-I", os.path.join(ROOT, "sage_b200", "csrc"), os.path.join(ROOT, "tests", "glibc_math_check.cpp"), "-o", exe])
    out = subprocess.check_output([exe, "3000000"]).decode()
    bad = {k: int(v) for k, v in (t.split("=") for t in out.split() if "=" in t)}
    assert bad["n"] >= 3_000_000
    ok = [v for v in (0, 1) if all(bad[f"{f}_variant{v}"] == 0 for f in ("exp", "log1p", "log10"))]
    assert ok, out
    assert any(bad[f"{f}_variant{1 - ok[0]}"] for f in ("exp", "log1p", "log10")), out   # the variants differ: the probe means something


def test_header_matches_ctypes(tmp_path):
    from sage_b200 import api
    src = tmp_path / "h.c"
    fields = [f[0] for f in api.CFdrOut._fields_]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "sage_b200.h"\nint main(void){printf("%zu %zu", sizeof(sage_b200_fdr_out), sizeof(sage_b200_fdr_params));'
                   + "".join(f'printf(" %zu", offsetof(sage_b200_fdr_out, {f}));' for f in fields) + "return 0;}\n")
    exe = str(tmp_path / "h")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    got = [int(x) for x in subprocess.check_output([exe]).split()]
    import ctypes as C
    want = [C.sizeof(api.CFdrOut), C.sizeof(api.CFdrParams)] + [getattr(api.CFdrOut, f).offset for f in fields]
    assert got == want
