"""Picked FDR on the device (sage_b200.picked_fdr / picked_precursor / competition_keys) against the C++ oracle (oracle_ml) and, where the
workload is small, the restatement of fdr.rs in tests/picked_reference.py, bit for bit. Workloads: tests/picked_cases.py."""
import numpy as np
import pytest

import picked_cases as PC
import picked_reference as R
import sage_b200
from oracle_ml import ml_oracle
from sage_b200 import SageB200Error

pytestmark = pytest.mark.gpu

EINVAL, ELIMIT = -1, -5
KEYS = ("peptide_q", "protein_q", "peptide_passing", "protein_passing", "peptide_entries", "protein_entries")


def _same(got, want, what):
    for k in KEYS:
        g, w = got[k], want[k]
        if isinstance(w, np.ndarray):
            gn, wn = np.isnan(g), np.isnan(w)
            assert np.array_equal(gn, wn), f"{what}: {k} NaN pattern"
            bad = np.flatnonzero(g[~gn].view(np.uint32) != w[~wn].view(np.uint32))
            assert bad.size == 0, f"{what}: {k} differs at {bad[:5]}: {g[~gn][bad[:5]]} vs {w[~wn][bad[:5]]}"
        else:
            assert g == w, f"{what}: {k} {g} != {w}"


def _oracle_kde(scores, decoy):
    return ml_oracle.kde_build(scores, decoy, 1000, True, 1.0)


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("generate_decoys", [True, False])
def test_edge_workloads(seed, generate_decoys):
    case = PC.edge_case(seed, generate_decoys)
    got = PC.device(case)
    _same(got, PC.oracle(case), f"edge seed {seed} gen {generate_decoys} (oracle)")
    _same(got, PC.reference(case), f"edge seed {seed} gen {generate_decoys}")


@pytest.mark.parametrize("name", sorted(PC.degenerate_cases()))
def test_degenerate(name):
    case = PC.degenerate_cases()[name]
    got = PC.device(case)
    _same(got, PC.oracle(case), f"{name} (oracle)")
    _same(got, PC.reference(case), name)


@pytest.mark.parametrize("n_rows,gen", [(10_000, True), (10_000, False), (100_000, True)])
def test_synth(n_rows, gen):
    case = PC.synth_case(n_rows, seed=n_rows + gen, generate_decoys=gen, n_target=max(20_000, n_rows // 2))
    kde = None if n_rows <= 10_000 else _oracle_kde
    got = PC.device(case)
    _same(got, PC.oracle(case), f"synth {n_rows} (oracle)")
    _same(got, PC.reference(case, kde=kde), f"synth {n_rows}")
    assert got["peptide_entries"] > 1000 and got["protein_entries"] > 0
    again = PC.device(case)
    for k in ("peptide_q", "protein_q"):
        assert got[k].tobytes() == again[k].tobytes()


@pytest.mark.parametrize("generate_decoys", [True, False])
def test_tied_scores(generate_decoys):
    case = PC.tied_case(5, generate_decoys)
    got = PC.device(case)
    _same(got, PC.oracle(case), f"tied gen {generate_decoys} (oracle)")
    _same(got, PC.reference(case), f"tied gen {generate_decoys}")


@pytest.mark.parametrize("generate_decoys", [True, False])
def test_fasta_databases(generate_decoys):
    case = PC.fasta_case(2, generate_decoys)
    got = PC.device(case)
    _same(got, PC.oracle(case), f"fasta gen {generate_decoys} (oracle)")
    _same(got, PC.reference(case), f"fasta gen {generate_decoys}")


def test_synth_1e6_against_oracle():
    case = PC.synth_case(1_000_000, seed=2024, n_target=500_000)
    got = PC.device(case)
    _same(got, PC.oracle(case), "synth 1e6 (oracle)")
    assert got["peptide_entries"] > 100_000


def test_search_to_picked_precursor_chain():
    """search -> predict_rt -> spectrum_fdr -> rows in spectrum_fdr's order -> picked_fdr -> FeatureMap on the device peptide_q -> add_ms1 ->
    quantify -> picked_precursor, each stage against the CPU chain (oracle_ml, oracle_lfq)."""
    import lfq_cases
    from oracle_lfq import lfq_oracle as LO
    from sage_b200 import FeatureMap, IndexedDatabase, LfqSettings, Scorer, Tolerance, api, synth
    pep = synth.make_peptides(6000, seed=301, static_c=True)
    spectra = synth.make_spectra(pep, 4000, seed=302)
    db = IndexedDatabase.build_from_peptides(pep)
    f, counts = Scorer(db, precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20)).score_batch(spectra)
    rows = f[counts > 0]
    fid = (rows["spectrum"] % 3).astype(np.uint32)
    rt = api.predict_rt(db, pep, rows, fid, 3)
    rto = ml_oracle.predict_rt(pep, rows, fid, 3)
    kw = dict(aligned_rt=rt["aligned_rt"], delta_rt_model=rt["delta_rt_model"], delta_ims_model=rt["delta_ims_model"])
    fd = api.spectrum_fdr(rows, Tolerance.ppm(-20, 20), **kw)
    fo = ml_oracle.spectrum_fdr(rows, Tolerance.ppm(-20, 20), **{k: rto[k] for k in kw})
    for k in ("discriminant_score", "order"):
        assert fd[k].tobytes() == fo[k].tobytes(), k
    order = fd["order"]
    srows, score = rows[order], fd["discriminant_score"][order]
    rng = np.random.default_rng(303)
    n_prot = np.where(rng.random(len(pep)) < 0.8, 1, 2).astype(np.uint32)
    protein = rng.integers(0, 300, len(pep)).astype(np.uint32)
    case = dict(peptides=pep, pep_idx=srows["peptide_idx"], score=score, n_proteins=n_prot, protein=protein, cterm=None, generate_decoys=True)
    got = sage_b200.picked_fdr(pep, srows, score, n_prot, protein)
    _same(got, PC.oracle(case), "chain picked_fdr")
    # this search has few decoys and no row passes at 1 %: the feature map filters at the smallest target peptide_q the device gave
    settings = LfqSettings(peptide_q_value=float(got["peptide_q"][srows["label"] == 1].min()))
    assert ((got["peptide_q"] <= settings.peptide_q_value) & (srows["label"] == 1)).sum() > 0
    feats = dict(peptide_idx=srows["peptide_idx"], peptide_q=got["peptide_q"], label=srows["label"], aligned_rt=rt["aligned_rt"][order],
                 calcmass=srows["calcmass"], file_id=fid[order], ims=srows["ims"])
    fm = FeatureMap.build(db, pep, settings, (2, 4), feats, rt["alignments"])
    orc = LO.LfqOracle(pep, settings, (2, 4), feats, rt["alignments"])
    ranges = fm.export()["ranges"]
    assert len(ranges) > 0
    srts = np.repeat(np.linspace(float(ranges["rt"].min()), float(ranges["rt"].max()), 200), 3).astype(np.float32)
    sp = lfq_cases._spectra_from_ranges(ranges, srts, np.tile(np.arange(3), 200), rng)
    sp = [(fi, t, m[np.argsort(m, kind="stable")], i[np.argsort(m, kind="stable")], mob) for fi, t, m, i, mob in sp]
    batch = lfq_cases._batch(sp)
    fm.add_ms1(batch)
    orc.add_ms1(batch)
    qd, qo = fm.quantify(), orc.quantify()
    keep = qo["present"]
    assert qd["id"].tolist() == qo["id"][keep].tolist() and qd["decoy"].tolist() == qo["decoy"][keep].tolist()
    # quantify's scores go through acos, which the device and the host libm may round apart (DESIGN.md §9): close, not bit-equal
    assert np.allclose(qd["score"], qo["score"][keep], rtol=1e-9, atol=0.0)
    q, passing = sage_b200.picked_precursor(qd["score"], qd["decoy"])
    wq, wp = ml_oracle.picked_precursor(qd["score"], qd["decoy"])
    assert len(q) > 20 and passing == wp and q.tobytes() == wq.tobytes()


@pytest.mark.parametrize("hash_bits", [64, 3])
def test_competition_keys_collisions(hash_bits):
    case = PC.synth_case(30_000, seed=11, n_target=5_000)
    pep = case["peptides"]
    ranks = sage_b200.competition_keys(pep, case["pep_idx"], generate_decoys=True, hash_bits=hash_bits)
    first = {}
    want = np.array([first.setdefault(R.peptide_key(pep, p, True), len(first)) for p in case["pep_idx"].tolist()], np.uint32)
    assert len(first) > 2000
    assert np.array_equal(ranks, want)
    edge = PC.edge_case(5, True)
    first = {}
    want = [first.setdefault(R.peptide_key(edge["peptides"], p, True, edge["cterm"]), len(first)) for p in edge["pep_idx"].tolist()]
    got = sage_b200.competition_keys(edge["peptides"], edge["pep_idx"], cterm=edge["cterm"], hash_bits=hash_bits)
    assert got.tolist() == want


def test_precursor_known_answer():
    score = np.array([5, 4, 3, 2, 1, 0.5, 0.4, 0.3], np.float64)
    decoy = np.array([0, 0, 1, 0, 0, 1, 0, 1], bool)
    perm = np.array([3, 7, 0, 5, 1, 6, 2, 4])
    q, passing = sage_b200.picked_precursor(score[perm], decoy[perm])
    assert passing == 0 and q.tobytes() == np.float32([0.5, 0.5, 0.5, 0.5, 0.5, 0.6, 0.6, 0.8])[perm].tobytes()


@pytest.mark.parametrize("seed", [1, 2])
def test_precursor_random(seed):
    rng = np.random.default_rng(seed)
    n = 5000
    score = rng.normal(0, 1, n) + np.where(rng.random(n) < 0.3, 0.0, 2.0)
    score[rng.random(n) < 0.02] = np.nan
    score[:50] = 1.0
    decoy = rng.random(n) < 0.3
    q, passing = sage_b200.picked_precursor(score, decoy)
    wq, wp = R.picked_precursor(score, decoy)
    assert passing == wp and q.tobytes() == wq.tobytes()
    oq, op = ml_oracle.picked_precursor(score, decoy)
    assert passing == op and q.tobytes() == oq.tobytes()


def test_precursor_past_counter_saturation():
    n = (1 << 24) + (1 << 20)
    rng = np.random.default_rng(3)
    score = rng.permutation(n).astype(np.float64)           # above 2^24 the f32 cast makes ties, which keep the row order
    decoy = rng.random(n) < 0.01
    q, passing = sage_b200.picked_precursor(score, decoy)
    order = np.argsort(-score.astype(np.float32), kind="stable")
    d = decoy[order]
    # f32 `+= 1.0` is exact up to 2^24 and then stays there (DESIGN.md §12)
    dec = np.minimum(1 + np.cumsum(d), 1 << 24).astype(np.float32)
    tar = np.minimum(np.cumsum(~d), 1 << 24).astype(np.float32)
    with np.errstate(all="ignore"):
        raw = dec / tar
    qmin = np.minimum(np.minimum.accumulate(raw[::-1])[::-1], np.float32(1.0))
    want = np.empty(n, np.float32)
    want[order] = qmin
    assert q.tobytes() == want.tobytes()
    assert passing == int(np.sum((qmin <= np.float32(0.05)) & ~d))
    assert np.cumsum(~d)[-1] > (1 << 24)


def test_errors():
    with pytest.raises(SageB200Error) as e:
        PC.device(PC.clash_case())
    assert e.value.code == EINVAL and "0 and 1" in e.value.message
    case = PC.degenerate_cases()["decoy_first"]
    with pytest.raises(SageB200Error) as e:
        PC.device(dict(case, pep_idx=np.array([0, 4], np.uint32), score=np.float32([1, 2])))
    assert e.value.code == EINVAL
    with pytest.raises(SageB200Error) as e:
        sage_b200.competition_keys(case["peptides"], np.array([0], np.uint32), hash_bits=65)
    assert e.value.code == EINVAL
    with pytest.raises(SageB200Error) as e:   # a truncated hash over more than 2^16 rows
        sage_b200.competition_keys(case["peptides"], np.zeros(70_000, np.uint32), hash_bits=3)
    assert e.value.code == ELIMIT
    empty = PC.device(dict(case, pep_idx=np.zeros(0, np.uint32), score=np.zeros(0, np.float32)))
    assert empty["peptide_entries"] == 0 and len(empty["peptide_q"]) == 0
    q, passing = sage_b200.picked_precursor(np.zeros(0), np.zeros(0, bool))
    assert len(q) == 0 and passing == 0
