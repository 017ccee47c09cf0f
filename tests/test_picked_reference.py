"""CPU checks of the picked-FDR restatement (tests/picked_reference.py): Rust's Display of peptides and f32, Peptide::reverse, a hand-computed
picked_precursor, and the peptide / protein competitions on the edge workloads of tests/picked_cases.py."""
import numpy as np
import pytest

import picked_cases as PC
import picked_reference as R

f32 = np.float32


@pytest.mark.parametrize("x,s", [(15.9949, "+15.9949"), (-17.02655, "-17.02655"), (0.0, "+0"), (-0.0, "-0"), (1e-7, "+0.0000001"),
                                 (1e20, "+100000000000000000000"), (float("nan"), "NaN"), (float("inf"), "+inf"), (42.0, "+42")])
def test_fmt_plus(x, s):
    assert R.fmt_plus(f32(x)) == s


def test_display_and_reverse():
    assert R.reverse(b"K", [0.0]) == (b"K", [0.0])
    assert R.reverse(b"ACK", [0.0, 1.0, 0.0])[0] == b"ACK"
    assert R.reverse(b"ACDK", [0.0, 1.0, 2.0, 0.0]) == (b"ADCK", [0.0, 2.0, 1.0, 0.0])
    nan = float("nan")
    assert R.display(b"MSTK", [0.0, f32(15.9949), -0.0, 0.0], f32(-0.0), nan) == "[-0]-MS[+15.9949]TK"
    assert R.display(b"WK", [nan, 0.0], nan, f32(0.0)) == "W[NaN]K-[+0]"


def test_picked_precursor_known_answer():
    score = np.array([5, 4, 3, 2, 1, 0.5, 0.4, 0.3], np.float64)
    decoy = np.array([0, 0, 1, 0, 0, 1, 0, 1], bool)
    perm = np.array([3, 7, 0, 5, 1, 6, 2, 4])
    q, passing = R.picked_precursor(score[perm], decoy[perm])
    want = f32([0.5, 0.5, 0.5, 0.5, 0.5, 0.6, 0.6, 0.8])[perm]
    assert passing == 0 and q.tobytes() == want.tobytes()
    q, passing = R.picked_precursor(np.arange(40, 0, -1.0), np.zeros(40, bool))
    assert passing == 40 and np.all(q == f32(1.0) / np.arange(1, 41, dtype=f32)[-1])


@pytest.mark.parametrize("generate_decoys", [True, False])
def test_edge_workload_runs(generate_decoys):
    case = PC.edge_case(7, generate_decoys)
    res = PC.reference(case)
    assert len(res["peptide_q"]) == len(case["pep_idx"]) and res["peptide_entries"] > 10
    # a target and its generated decoy share one entry only with generate_decoys
    keys = {R.peptide_key(case["peptides"], p, generate_decoys, case["cterm"]) for p in case["pep_idx"].tolist()}
    assert res["peptide_entries"] == len(keys)


def test_clash_raises():
    case = PC.clash_case()
    with pytest.raises(R.PickedClash):
        PC.reference(case)
