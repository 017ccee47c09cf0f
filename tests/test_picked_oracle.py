"""The two CPU authorities of picked FDR agree bit for bit: the C++ oracle (oracle_ml, fdr.rs with real key strings) and the numpy
restatement (tests/picked_reference.py), on every workload of tests/picked_cases.py of at most 10^5 rows, on the LFQ edge workloads'
quantify rows (picked_precursor) and on a hand-computed picked_precursor."""
import numpy as np
import pytest

import lfq_cases
import picked_cases as PC
import picked_reference as R
from oracle_lfq import lfq_oracle as LO
from oracle_ml import ml_oracle

KEYS = ("peptide_q", "protein_q", "peptide_passing", "protein_passing", "peptide_entries", "protein_entries")


def _same(a, b, what):
    for k in KEYS:
        if isinstance(b[k], np.ndarray):
            assert a[k].tobytes() == b[k].tobytes(), f"{what}: {k}"
        else:
            assert a[k] == b[k], f"{what}: {k} {a[k]} != {b[k]}"


def _oracle_kde(s, d):
    return ml_oracle.kde_build(s, d, 1000, True, 1.0)


CASES = {f"edge_{s}_{g}": (lambda s=s, g=g: PC.edge_case(s, g)) for s in (1, 2, 3) for g in (True, False)}
CASES.update({f"degenerate_{k}": (lambda k=k: PC.degenerate_cases()[k]) for k in PC.degenerate_cases()})
CASES.update({f"fasta_{g}": (lambda g=g: PC.fasta_case(1, g)) for g in (True, False)})
CASES.update({f"tied_{g}": (lambda g=g: PC.tied_case(5, g)) for g in (True, False)})
CASES.update({f"synth_10000_{g}": (lambda g=g: PC.synth_case(10_000, seed=10_000 + g, generate_decoys=g)) for g in (True, False)})


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_restatement(name):
    case = CASES[name]()
    _same(PC.oracle(case), PC.reference(case), name)


def test_oracle_equals_restatement_1e5():
    # the restatement's own KDE would take minutes at 10^5 entries; kde_build itself is cross-checked in tests/test_ml_reference.py
    case = PC.synth_case(100_000, seed=100_001, n_target=50_000)
    _same(PC.oracle(case), PC.reference(case, kde=_oracle_kde), "synth 1e5")


def test_fasta_keys_are_the_oracle_db_strings():
    case = PC.fasta_case(1, True)
    db, pep = case["db"], case["peptides"]
    checked = 0
    for i in range(len(pep)):
        # the oracle db prints modifications with %g (6 digits), not Rust's shortest round-trip: compare the unmodified peptides
        if not pep.decoy[i] and "[" not in db.peptide_string(i)[0]:
            assert R.peptide_key(pep, i, True, case["cterm"]) == db.peptide_string(i)[0]
            checked += 1
    assert checked > 500


def test_clash_both():
    case = PC.clash_case()
    with pytest.raises(ml_oracle.PickedClash):
        PC.oracle(case)
    with pytest.raises(R.PickedClash):
        PC.reference(case)


def test_precursor_known_answer():
    score = np.array([5, 4, 3, 2, 1, 0.5, 0.4, 0.3], np.float64)
    decoy = np.array([0, 0, 1, 0, 0, 1, 0, 1], bool)
    perm = np.array([3, 7, 0, 5, 1, 6, 2, 4])
    q, passing = ml_oracle.picked_precursor(score[perm], decoy[perm])
    assert passing == 0 and q.tobytes() == np.float32([0.5, 0.5, 0.5, 0.5, 0.5, 0.6, 0.6, 0.8])[perm].tobytes()


def quantify_rows(name):
    c = lfq_cases.case(name)
    o = LO.LfqOracle(c["peptides"], c["settings"], c["charges"], c["features"], c["alignments"])
    for b in c["batches"]:
        o.add_ms1(b)
    q = o.quantify()
    keep = q["present"]
    return q["score"][keep], q["decoy"][keep]


@pytest.mark.parametrize("name", ["files9", "charges_1_8", "charges_1_8_combined", "pages", "mobility_mixed", "degenerate_input"])
def test_precursor_on_quantify_rows(name):
    score, decoy = quantify_rows(name)
    q, passing = ml_oracle.picked_precursor(score, decoy)
    wq, wp = R.picked_precursor(score, decoy)
    assert passing == wp and q.tobytes() == wq.tobytes()
