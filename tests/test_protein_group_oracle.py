"""The two CPU authorities of protein grouping agree exactly: the C++ oracle (oracle_ml, protein_grouping.rs with name strings and the
literal BipartiteGraph loop) and the Python restatement (tests/protein_group_reference.py, whose cover is the forced picks plus a greedy per
component). Both match protein_grouping.rs's own known answers. The C structs of the new entry points match their ctypes mirrors."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import protein_group_cases as G
import protein_group_reference as R
from oracle_ml import ml_oracle
from sage_b200 import api

CASES = dict(G.all_small_cases())
CASES.update({f"fasta_{g}": (lambda g=g: G.fasta_case(1, g)) for g in (True, False)})
CASES.update({f"family_10000_{g}": (lambda g=g: G.family_case(10_000, 10 + g, g)) for g in (True, False)})


def _case(name):
    c = CASES[name]
    return c() if callable(c) else c


def _check_expect(res, case, what):
    for i, v in case["expect"].items():
        s, k = v if isinstance(v, tuple) else (v, None)
        assert res["protein_groups"][i] == s, f"{what}: row {i} {res['protein_groups'][i]!r} != {s!r}"
        if k is not None:
            assert res["num_protein_groups"][i] == k, f"{what}: row {i} count"
    assert all(s is not None for s in res["protein_groups"])


@pytest.mark.parametrize("name", sorted(G.known_cases()))
def test_known_answers(name):
    case = G.known_cases()[name]
    _check_expect(G.oracle(case), case, f"{name} (oracle)")
    _check_expect(G.reference(case), case, f"{name} (restatement)")


@pytest.mark.parametrize("name", sorted(G.KNOWN_COVERS))
def test_known_covers(name):
    edges, nl, nr, want = G.KNOWN_COVERS[name]
    left, right = np.array([e[0] for e in edges], np.uint32), np.array([e[1] for e in edges], np.uint32)
    assert ml_oracle.bipartite_cover(left, right, nl, nr)[0].tolist() == want
    assert R.cover(edges, nl, nr)[0] == want


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_restatement(name):
    case = _case(name)
    G.same(G.oracle(case), G.reference(case), name)


def test_oracle_equals_restatement_1e5():
    case = G.family_case(100_000, 100_001)
    o = G.oracle(case)
    G.same(o, G.reference(case, kde=lambda s, d: ml_oracle.kde_build(s, d, 1000, True, 1.0)), "family 1e5")
    assert sum(o["greedy_picks"]) > 100 and o["entries"] > 1000 and o["passing"] > 0


@pytest.mark.parametrize("seed", range(12))
def test_literal_cover_equals_components(seed):
    """Both facts of DESIGN.md §13 at once: the literal trim / add_largest loop equals the forced picks plus a greedy per component."""
    left, right, nl, nr = G.random_multigraph(seed, n_left=50 + 40 * seed, n_right=60 + 50 * seed, n_edges=150 + 120 * seed)
    cover, picks = ml_oracle.bipartite_cover(left, right, nl, nr)
    want, want_picks = R.cover(list(zip(left.tolist(), right.tolist())), nl, nr)
    assert cover.tolist() == want and picks == want_picks
    assert picks > 0


def test_literal_cover_equals_components_ring():
    left, right, nl, nr = G.ring_graph(3001)
    cover, picks = ml_oracle.bipartite_cover(left, right, nl, nr)
    want, want_picks = R.cover(list(zip(left.tolist(), right.tolist())), nl, nr)
    assert cover.tolist() == want and picks == want_picks == 1501


def test_struct_layout(tmp_path):
    """sizeof / offsetof of the new structs, compiled from include/sage_b200.h, equal their ctypes mirrors."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    fields = [("sage_b200_protein_group_params", api.CProteinGroupParams, ["protein_ids", "n_names", "protein_grouping", "threshold"]),
              ("sage_b200_protein_group_out", api.CProteinGroupOut, ["group_decoy", "peptides", "annotated", "passing", "entries", "ms_build", "ms_lookup",
                                                                    "ms_total"])]
    src = ["#include <stdio.h>", "#include <stddef.h>", '#include "sage_b200.h"', "int main(void) {"]
    for st, _, fs in fields:
        src.append(f'printf("%zu\\n", sizeof({st}));')
        src += [f'printf("%zu\\n", offsetof({st}, {f}));' for f in fs]
    src.append("return 0; }")
    (tmp_path / "layout.c").write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(root, "include"), "-o", str(exe), str(tmp_path / "layout.c")])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = []
    for _, cls, fs in fields:
        want.append(C.sizeof(cls))
        want += [getattr(cls, f).offset for f in fs]
    assert got == want
