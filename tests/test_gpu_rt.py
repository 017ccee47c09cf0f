"""GPU: the predict_rt stage on the device (sage_b200.predict_rt) is bit-identical to the CPU oracle (oracle_ml) on every output."""
import numpy as np
import pytest

import ml_reference
from oracle_ml import ml_oracle
from rt_cases import base_peptides, cases
from sage_b200 import FeatureMap, IndexedDatabase, LfqSettings, Tolerance, api, synth

pytestmark = pytest.mark.gpu
COLUMNS = ("aligned_rt", "predicted_rt", "delta_rt_model", "predicted_ims", "delta_ims_model", "spectrum_q")
SCALARS = ("training_rows", "aligned_peptides", "rt_fitted", "rt_eps", "ims_fitted", "ims_eps")
RESTATED_ROWS = 100_000   # the numpy restatement (tests/ml_reference.py) is checked up to this size


def same_bits(a, b):
    """Bit for bit, except that any two NaNs match (the device and the host CPU write different NaN payloads)."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    w = {8: np.uint64, 4: np.uint32}[a.dtype.itemsize]
    return (a.view(w) == b.view(w)) | (np.isnan(a) & np.isnan(b))


def assert_same(got, want, what):
    for k in COLUMNS:
        eq = same_bits(got[k], want[k])
        assert eq.all(), f"{what}: {k} differs at {np.nonzero(~eq)[0][:5]}"
    ga, wa = got["alignments"].view(np.float32), want["alignments"].view(np.float32)
    assert same_bits(ga, wa).all(), f"{what}: alignments {got['alignments']} != {want['alignments']}"
    for k in SCALARS:
        assert got[k] == want[k], f"{what}: {k} {got[k]} != {want[k]}"
    for k in ("rt_r2", "ims_r2", "rt_beta", "ims_beta"):
        assert same_bits(np.atleast_1d(np.float64(got[k])), np.atleast_1d(np.float64(want[k]))).all(), f"{what}: {k}"


_CASES = cases()
_DB = {}


def db_for(pep):
    key = id(pep)
    if key not in _DB:
        _DB[key] = (IndexedDatabase.build_from_peptides(pep), pep)
    return _DB[key][0]


def run_both(c):
    got = api.predict_rt(db_for(c["pep"]), c["pep"], c["rows"], c["file_id"], c["n_files"])
    want = ml_oracle.predict_rt(c["pep"], c["rows"], c["file_id"], c["n_files"])
    return got, want


@pytest.mark.parametrize("name", sorted(_CASES))
def test_edge_workloads(name):
    c = _CASES[name]
    got, want = run_both(c)
    assert_same(got, want, name)
    if len(c["rows"]) <= RESTATED_ROWS:
        assert_same(got, ml_reference.predict_rt(c["pep"], c["rows"], c["file_id"], c["n_files"]), name + " (restatement)")
    if name.startswith("train_"):
        assert got["training_rows"] == int(name.split("_")[1]) and got["rt_fitted"] and got["ims_fitted"]
    if name in ("no_training", "rows_1_files_1"):
        assert got["training_rows"] == 0 and not got["rt_fitted"] and not got["ims_fitted"]
        assert (got["alignments"]["slope"] == 1).all() and (got["alignments"]["intercept"] == 0).all()
        assert (got["predicted_rt"] == 0).all() and (got["delta_rt_model"] == np.float32(0.999)).all()
    if name == "empty_and_zero_files":
        a = got["alignments"]
        assert a["max_rt"][2] == 0 and a["max_rt"][4] == 0 and a["slope"][2] == 1 and a["intercept"][4] == 0
    if name == "odd_rts":
        assert got["alignments"]["max_rt"][1] == np.float32(4294967295.0)
    if name == "no_mobility":
        assert got["ims_fitted"] and np.isnan(got["ims_r2"]) and (got["ims_beta"] == 0).all()
    if name == "collinear":
        assert got["rt_fitted"] and not got["ims_fitted"] and (got["delta_ims_model"] == np.float32(0.999)).all()
    if name == "rt0_every_file":
        assert got["aligned_peptides"] < len(np.unique(c["rows"]["peptide_idx"][got["spectrum_q"] <= 0.01]))


def test_recovers_synthetic_alignment():
    """The device alignments undo each file's synthetic distortion: on true matches, aligned RT against the hidden RT has the same line in
    every file; and the RT model explains the aligned RTs."""
    pep = base_peptides()
    rows, fid, truth = synth.make_rt_psms(pep, 200_000, 6, seed=77, mobility=True, with_truth=True)
    got = api.predict_rt(db_for(pep), pep, rows, fid, 6)
    t = truth["is_true"]
    a = got["alignments"][fid]
    unaligned = rows["rt"] / a["max_rt"]
    lines = np.array([np.polyfit(truth["rt_true"][t & (fid == f)], got["aligned_rt"][t & (fid == f)], 1) for f in range(6)])
    before = np.array([np.polyfit(truth["rt_true"][t & (fid == f)], unaligned[t & (fid == f)], 1) for f in range(6)])
    assert np.ptp(lines[:, 0]) < 0.05 and np.ptp(lines[:, 1]) < 0.02, lines
    assert np.ptp(lines[:, 0]) * 3 < np.ptp(before[:, 0]) and np.ptp(lines[:, 1]) * 3 < np.ptp(before[:, 1]), (lines, before)
    assert got["rt_r2"] > 0.9 and got["ims_r2"] > 0.9
    assert np.median(got["delta_rt_model"][t]) < 0.02


def test_search_then_predict_rt_then_fdr():
    """search -> predict_rt -> spectrum_fdr with its three columns, against the oracle chain; the alignments build a FeatureMap."""
    from sage_b200 import Scorer
    pep = synth.make_peptides(6000, seed=301, static_c=True)
    spectra = synth.make_spectra(pep, 4000, seed=302)
    db = IndexedDatabase.build_from_peptides(pep)
    sc = Scorer(db, precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20))
    f, counts = sc.score_batch(spectra)
    rows = f[counts > 0]
    fid = (rows["spectrum"] % 3).astype(np.uint32)
    got = api.predict_rt(db, pep, rows, fid, 3)
    want = ml_oracle.predict_rt(pep, rows, fid, 3)
    assert_same(got, want, "search")
    assert got["training_rows"] > 100 and got["rt_fitted"]
    kw = dict(aligned_rt=got["aligned_rt"], delta_rt_model=got["delta_rt_model"], delta_ims_model=got["delta_ims_model"])
    fd = api.spectrum_fdr(rows, Tolerance.ppm(-20, 20), **kw)
    fo = ml_oracle.spectrum_fdr(rows, Tolerance.ppm(-20, 20), **{k: want[k] for k in kw})
    for k in ("discriminant_score", "posterior_error", "spectrum_q", "order"):
        assert same_bits(fd[k], fo[k]).all(), k
    feats = dict(peptide_idx=rows["peptide_idx"], peptide_q=fd["spectrum_q"], label=rows["label"], aligned_rt=got["aligned_rt"],
                 calcmass=rows["calcmass"], file_id=fid, ims=rows["ims"])
    fm = FeatureMap.build(db, pep, LfqSettings(), (2, 4), feats, got["alignments"])
    assert fm.info()["n_peptides"] > 0


def test_twice_identical_bytes():
    c = _CASES["rows_100000_files_3"]
    a = api.predict_rt(db_for(c["pep"]), c["pep"], c["rows"], c["file_id"], c["n_files"])
    b = api.predict_rt(db_for(c["pep"]), c["pep"], c["rows"], c["file_id"], c["n_files"])
    for k in COLUMNS + ("alignments", "rt_beta", "ims_beta"):
        assert a[k].tobytes() == b[k].tobytes(), k


def test_errors():
    pep = base_peptides()
    db = db_for(pep)
    rows, fid = synth.make_rt_psms(pep, 100, 2, seed=3)

    def code(**kw):
        args = dict(rows=rows, fid=fid, n_files=2, pep=pep)
        args.update(kw)
        with pytest.raises(api.SageB200Error) as e:
            api.predict_rt(db, args["pep"], args["rows"], args["fid"], args["n_files"])
        return e.value.code

    bad = fid.copy()
    bad[7] = 2
    assert code(fid=bad) == -1                                          # file_id >= n_files
    r = rows.copy()
    r["peptide_idx"][3] = len(pep)
    assert code(rows=r) == -1                                           # peptide_idx outside the db
    assert code(n_files=0) == -1                                        # rows but no files
    seq = pep.seq.copy()
    p0 = int(rows["peptide_idx"][0])
    seq[pep.seq_off[p0]] = ord("a")
    bad_pep = api.Peptides(pep.seq_off, seq, pep.mods, pep.nterm, pep.mono, pep.decoy, pep.missed)
    assert code(pep=bad_pep) == -1                                      # a residue outside 'A'..'Z'
    assert code(n_files=1 << 40) == -5                                  # the per-file arrays and matrix cannot fit
    e = api.predict_rt(db, pep, rows[:0], fid[:0], 3)
    assert e["alignments"].tolist() == [(0.0, 1.0, 0.0)] * 3 and not e["rt_fitted"] and not e["ims_fitted"]
