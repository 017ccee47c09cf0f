"""CPU checks of the predict_rt oracle (oracle_ml/ml_oracle.cpp): the reference's own known answers (regression.rs, mobility_model.rs), the
embedding quirks it keeps, global_alignment against a pure-Python restatement, the fit against numpy, and the C header against ctypes."""
import ctypes as C
import os
import subprocess

import numpy as np

from ml_reference import py_alignment
from oracle_ml import ml_oracle
from rt_cases import base_peptides, peptides_from
from sage_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VALID_AA = "ACDEFGHIKLMNPQRSTVWYUO"


def test_fit_perfect_line():   # regression.rs:124-133
    x = np.arange(50.0)
    beta, r2, _ = ml_oracle.linreg_fit(np.stack([x, np.ones(50)], 1), 2 * x + 1)
    assert abs(beta[0] - 2) < 1e-9 and abs(beta[1] - 1) < 1e-9 and abs(r2 - 1) < 1e-9


def test_fit_with_noise():     # regression.rs:135-150
    i = np.arange(200.0)
    x = i / 10.0
    y = 3 * x + 2 + np.sin(i * 0.7) * 0.1
    beta, r2, _ = ml_oracle.linreg_fit(np.stack([x, np.ones(200)], 1), y)
    assert abs(beta[0] - 3) < 0.05 and abs(beta[1] - 2) < 0.1 and r2 > 0.99


def test_empty_filter_returns_none():   # regression.rs:152-157
    assert ml_oracle.linreg_fit(np.zeros((0, 1)), np.zeros(0)) is None


def test_feature_embed():      # mobility_model.rs:188-266
    e = [ml_oracle.rt_embed(1, s, 1000.0, 2) for s in ("LEKSLIEK", "LERSLIEWK", "LWESLIEK", "CHADWICK")]
    nt, ct = 44, 66
    ix = {a: VALID_AA.index(a) for a in "KWLI"}
    assert [x[nt + ix["L"]] for x in e] == [1, 1, 1, 0]
    assert [x[nt + ix["K"]] for x in e] == [0, 0, 0, 0]
    assert [x[nt + ix["W"]] for x in e] == [0, 0, 1, 0]
    assert [x[ct + ix["K"]] for x in e] == [1, 1, 1, 1]
    assert [x[ct + ix["W"]] for x in e] == [0, 1, 0, 0]
    assert [x[ct + ix["I"]] for x in e] == [0, 0, 0, 0]


def test_short_peptides_terminal_rules_and_groups():
    """Lengths 1-4: the N-terminal arm wins at positions 0 and 1; the RT model counts positions len-3 and len-2 as C-terminal, the mobility
    model every position past len-3. The mobility groups compare letter offsets with VALID_AA positions: 'bulky' counts N, O, K and G."""
    for seq in ("W", "WY", "WYF", "WYFH"):
        rt, ims = ml_oracle.rt_embed(0, seq, 900.0), ml_oracle.rt_embed(1, seq, 900.0, 2)
        L = len(seq)
        for p, a in enumerate(seq):
            k = VALID_AA.index(a)
            in_n = p <= 1
            assert rt[22 + k] == in_n and ims[44 + k] == in_n, (seq, p)
            assert rt[44 + k] == (not in_n and p in (L - 3, L - 2)), (seq, p)
            assert ims[66 + k] == (not in_n and p > max(L - 3, 0)), (seq, p)
    bulky = ml_oracle.rt_embed(1, "NOKGLVIFWY", 900.0, 2)
    assert bulky[91] == 4                                                    # N, O, K, G; none of L V I F W Y
    assert ml_oracle.rt_embed(1, "BJXZ", 900.0, 2)[0] == 4                    # letters outside VALID_AA land in A's column


def test_alignment_against_python():
    pep = base_peptides()
    for seed, n, nf in ((1, 3000, 3), (2, 1500, 5), (3, 40, 2)):
        rows, fid = synth.make_rt_psms(pep, n, nf, seed=seed)
        rows["rt"][::11] = np.round(rows["rt"][::11])
        got = ml_oracle.predict_rt(pep, rows, fid, nf)
        want = py_alignment(rows, fid, nf)
        assert [tuple(a) for a in got["alignments"].tolist()] == [tuple(float(x) for x in w) for w in want], seed
        a = got["alignments"][fid]
        aligned = (rows["rt"] / a["max_rt"]) * a["slope"] + a["intercept"]
        assert np.array_equal(aligned.astype(np.float32).view(np.uint32), got["aligned_rt"].view(np.uint32))


def test_rt_fit_against_lstsq():
    """On the training rows of make_rt_psms, the oracle's RT predictions equal numpy lstsq's (the RT design is collinear, so the coefficients
    themselves are not unique); on a well-conditioned matrix the bare fit equals lstsq's coefficients."""
    pep = base_peptides()
    rows, fid = synth.make_rt_psms(pep, 30_000, 3, seed=9)
    r = ml_oracle.predict_rt(pep, rows, fid, 3)
    train = (rows["label"] == 1) & (r["spectrum_q"] <= np.float32(0.01))
    X = np.array([ml_oracle.rt_embed(0, pep.sequence(p), pep.mono[p]) for p in rows["peptide_idx"][train]])
    y = r["aligned_rt"][train].astype(np.float64)
    ls = np.linalg.lstsq(X, y, rcond=None)[0]
    assert np.abs(X @ r["rt_beta"] - X @ ls).max() < 1e-6
    rng = np.random.default_rng(10)
    Xw = np.concatenate([rng.normal(0, 1, (5000, 6)), np.ones((5000, 1))], 1)
    yw = Xw @ rng.normal(0, 1, 7) + rng.normal(0, 0.01, 5000)
    beta, r2, eps = ml_oracle.linreg_fit(Xw, yw)
    assert np.allclose(beta, np.linalg.lstsq(Xw, yw, rcond=None)[0], rtol=1e-7, atol=1e-9) and eps == 1e-8 and r2 > 0.99


def test_chunked_fold_is_deterministic_across_threads():
    pep = peptides_from(["PEPTIDEK", "LESLIEK", "UOBJXZ"])
    rows, fid = synth.make_rt_psms(pep, 5000, 2, seed=11, mobility=True)
    a, b = ml_oracle.predict_rt(pep, rows, fid, 2, threads=1), ml_oracle.predict_rt(pep, rows, fid, 2, threads=7)
    for k in ("aligned_rt", "predicted_rt", "predicted_ims", "rt_beta", "ims_beta"):
        assert a[k].tobytes() == b[k].tobytes()


def test_header_matches_ctypes(tmp_path):
    from sage_b200 import api
    fields = [f[0] for f in api.CRtOut._fields_]
    src = tmp_path / "h.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "sage_b200.h"\nint main(void){printf("%zu", sizeof(sage_b200_rt_out));'
                   + "".join(f'printf(" %zu", offsetof(sage_b200_rt_out, {f}));' for f in fields) + "return 0;}\n")
    exe = str(tmp_path / "h")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [C.sizeof(api.CRtOut)] + [getattr(api.CRtOut, f).offset for f in fields]
