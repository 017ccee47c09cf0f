"""Protein grouping and picked protein-group FDR on the device (sage_b200.protein_groups / bipartite_cover) against the C++ oracle (oracle_ml)
and, up to 10^5 rows, the restatement in tests/protein_group_reference.py: every string built from the device's ids, num_protein_groups, the
pass, the group tables with cover flags, protein_group_q bit for bit, passing and entries. Workloads: tests/protein_group_cases.py."""
import numpy as np
import pytest

import picked_cases as PC
import protein_group_cases as G
import protein_group_reference as R
import sage_b200
from oracle_ml import ml_oracle
from sage_b200 import SageB200Error

pytestmark = pytest.mark.gpu

EINVAL = -1


def _oracle_kde(s, d):
    return ml_oracle.kde_build(s, d, 1000, True, 1.0)


def _check(case, what, restatement=True, kde=None):
    got = G.device(case)
    G.same(got, G.oracle(case), f"{what} (oracle)")
    if restatement:
        G.same(got, G.reference(case, kde=kde), what)
    return got


@pytest.mark.parametrize("name", sorted(G.all_small_cases()))
def test_small_workloads(name):
    case = G.all_small_cases()[name]
    got = _check(case, name)
    if "expect" in case:
        for i, v in case["expect"].items():
            assert got["protein_groups"][i] == (v[0] if isinstance(v, tuple) else v)


@pytest.mark.parametrize("generate_decoys", [True, False])
def test_fasta_databases(generate_decoys):
    _check(G.fasta_case(2, generate_decoys), f"fasta gen {generate_decoys}")


@pytest.mark.parametrize("n_rows,gen", [(10_000, True), (10_000, False), (100_000, True)])
def test_family(n_rows, gen):
    case = G.family_case(n_rows, n_rows + gen, gen)
    got = _check(case, f"family {n_rows}", kde=None if n_rows <= 10_000 else _oracle_kde)
    assert sum(got["greedy_picks"]) > 0 and got["entries"] > 100
    again = G.device(case)
    for k in ("num_protein_groups", "protein_group_q", "pass", "row_group_offsets", "row_groups", "group_offsets", "group_members", "group_covered",
              "group_decoy"):
        assert got[k].tobytes() == again[k].tobytes(), k


def test_family_1e6_against_oracle():
    case = G.family_case(1_000_000, 2024)
    got = _check(case, "family 1e6", restatement=False)
    assert sum(got["greedy_picks"]) > 1000 and got["passing"] > 0


def _covers(left, right, nl, nr):
    got = sage_b200.bipartite_cover(left, right, nl, nr)
    lit, _ = ml_oracle.bipartite_cover(left, right, nl, nr)
    comp, _ = R.cover(list(zip(np.asarray(left).tolist(), np.asarray(right).tolist())), nl, nr)
    assert got.tolist() == lit.tolist() == comp
    return got


@pytest.mark.parametrize("name", sorted(G.KNOWN_COVERS))
def test_cover_hook_known(name):
    edges, nl, nr, want = G.KNOWN_COVERS[name]
    got = _covers(np.array([e[0] for e in edges], np.uint32), np.array([e[1] for e in edges], np.uint32), nl, nr)
    assert got.tolist() == want


@pytest.mark.parametrize("seed", range(8))
def test_cover_hook_random(seed):
    _covers(*G.random_multigraph(seed, n_left=100 + 300 * seed, n_right=120 + 400 * seed, n_edges=300 + 900 * seed))


@pytest.mark.parametrize("k", [511, 513, 4000])
def test_cover_hook_giant_component(k):
    # 511 groups run on one warp, 513 and 4000 on one CTA
    assert _covers(*G.ring_graph(k)).sum() == (k + 1) // 2


def test_search_to_protein_groups_chain():
    """search -> predict_rt -> spectrum_fdr -> rows in spectrum_fdr's order -> picked_fdr -> protein_groups on the device peptide_q, over a
    FASTA-built database, each stage against the CPU chain (oracle_ml)."""
    from sage_b200 import IndexedDatabase, Scorer, Tolerance, api, synth
    fc = PC.fasta_case(3, True, n_proteins=200, n_rows=10)
    pep, proteins = fc["peptides"], fc["proteins"]
    spectra = synth.make_spectra(pep, 3000, seed=304)
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
    got = sage_b200.picked_fdr(pep, srows, score, fc["n_proteins"], fc["protein"], cterm=fc["cterm"])
    want = ml_oracle.picked_fdr(pep, srows["peptide_idx"], score, proteins, cterm=fc["cterm"])
    assert got["peptide_q"].tobytes() == want["peptide_q"].tobytes()
    case = G.make(proteins, pep.decoy, q=got["peptide_q"], label=srows["label"], pep_idx=srows["peptide_idx"], score=score, generate_decoys=True,
                  peptides=pep, seed=5)
    res = _check(case, "chain")
    assert len(srows) > 1000 and res["groups"][0] > 0 and res["annotated"][0] > 0


def test_errors():
    case = G.known_cases()["expected_groups"]
    off, ids, names = G.name_ids(case)
    with pytest.raises(SageB200Error) as e:
        sage_b200.protein_groups(case["peptides"], G.rows_of(case), case["peptide_q"], case["score"], off, ids, len(names) - 1)
    assert e.value.code == EINVAL
    with pytest.raises(SageB200Error) as e:
        sage_b200.bipartite_cover(np.array([0], np.uint32), np.array([3], np.uint32), 1, 3)
    assert e.value.code == EINVAL
    empty = G.make([["A"]], [0], pep_idx=np.zeros(0, np.uint32))
    res = G.device(empty)
    assert res["entries"] == 0 and len(res["protein_groups"]) == 0
    assert sage_b200.bipartite_cover(np.zeros(0, np.uint32), np.zeros(0, np.uint32), 3, 0).tolist() == [False] * 3
