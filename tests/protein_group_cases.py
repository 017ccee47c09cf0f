"""Workloads of protein grouping and picked protein-group FDR (protein_grouping.rs, fdr.rs:192-226). A case is dict(peptides, proteins,
decoy, pep_idx, label, peptide_q, score, protein_grouping, threshold, decoy_tag, generate_decoys), with proteins[p] the name list of peptide
p; `expect` (row -> string or (string, count)) holds the reference's own known answers where it states them. Name ids for the device are a
seeded shuffle of the names, so that numbering by id and numbering by first encounter differ."""
from __future__ import annotations

import numpy as np

from sage_b200 import Peptides, synth

f32 = np.float32
NAN = float("nan")


def dummy_peptides(decoy) -> Peptides:
    """A peptide table whose only meaningful field is the decoy flag (protein grouping reads nothing else)."""
    n = len(decoy)
    return Peptides(np.zeros(n + 1, np.uint32), np.zeros(0, np.uint8), np.zeros(0, f32), np.full(n, NAN, f32), np.zeros(n, f32),
                    np.asarray(decoy, np.uint8), np.zeros(n, np.uint8))


def make(proteins, decoy, q=None, label=None, pep_idx=None, score=None, protein_grouping=True, threshold=0.01, generate_decoys=False, peptides=None,
         seed=0, **extra):
    n_pep = len(proteins)
    decoy = np.zeros(n_pep, np.uint8) if decoy is None else np.asarray(decoy, np.uint8)
    pep_idx = np.arange(n_pep, dtype=np.uint32) if pep_idx is None else np.asarray(pep_idx, np.uint32)
    n = len(pep_idx)
    label = np.where(decoy[pep_idx] != 0, -1, 1).astype(np.int32) if label is None else np.asarray(label, np.int32)
    q = np.zeros(n, f32) if q is None else np.asarray(q, f32)
    score = np.random.default_rng(seed).normal(0.0, 1.0, n).astype(f32) if score is None else np.asarray(score, f32)
    return dict(peptides=peptides if peptides is not None else dummy_peptides(decoy), proteins=[list(x) for x in proteins], decoy=decoy, pep_idx=pep_idx,
                label=label, peptide_q=q, score=score, protein_grouping=protein_grouping, threshold=threshold, decoy_tag="rev_",
                generate_decoys=generate_decoys, seed=seed, **extra)


def name_ids(case):
    """(protein_offsets, protein_ids, names): ids are a seeded permutation of the distinct names in order of appearance."""
    names = list(dict.fromkeys(nm for lst in case["proteins"] for nm in lst))
    perm = np.random.default_rng(case.get("seed", 0) + 7).permutation(len(names))
    order = [names[i] for i in np.argsort(perm)]        # order[id] = name
    id_of = {nm: i for i, nm in enumerate(order)}
    off = np.zeros(len(case["proteins"]) + 1, np.uint32)
    off[1:] = np.cumsum([len(lst) for lst in case["proteins"]])
    ids = np.array([id_of[nm] for lst in case["proteins"] for nm in lst], np.uint32)
    return off, ids, order


# ---------------------------------------------------------------------------------------------------- protein_grouping.rs's test module
TEN = [["protein_7"], ["protein_4", "protein_6", "protein_9"], ["protein_1"], ["protein_1", "protein_5"], ["protein_7"], ["protein_3", "protein_6"],
       ["protein_1"], ["protein_1", "protein_2", "protein_5", "protein_8"], ["protein_1"], ["protein_4", "protein_9"]]


def known_cases():
    A, B, C = "protA", "protB", "protC"
    return {
        "expected_groups": make(TEN, [0] * 10, expect=dict(enumerate(["protein_7", "protein_4/protein_9;protein_6", "protein_1", "protein_1", "protein_7",
                                                                       "protein_6", "protein_1", "protein_1", "protein_1", "protein_4/protein_9"]))),
        "decoy_excluded": make([[A], [A], [B]], [0, 1, 0], expect={1: A}),
        "generate_decoys_tag": make([[A], [A]], [0, 1], protein_grouping=False, threshold=None, generate_decoys=True, expect={0: A, 1: "rev_protA"}),
        "grouping_disabled": make([[A, B], [C]], [0, 0], protein_grouping=False, threshold=None, expect={0: ("protA;protB", 2), 1: (C, 1)}),
        "single": make([[A]], [0], expect={0: (A, 1)}),
        "all_shared": make([[A, B]] * 3, [0, 0, 0], expect={i: ("protA/protB", 1) for i in range(3)}),
        "threshold_filtering": make([[A], [B]], [0, 0], q=[0.001, 0.5], expect={0: A, 1: B}),
        "all_decoys": make([[A], [B]], [1, 1], expect={0: A, 1: B}),
        "identical_evidence": make([[A, B], [A, B], [C]], [0, 0, 0], expect={0: "protA/protB", 1: "protA/protB", 2: C}),
        "distinct_group_count": make([[A], [B], [A, B]], [0, 0, 0], expect={0: (A, 1), 1: (B, 1), 2: ("protA;protB", 2)}),
    }


# BipartiteGraph's known answers: (edges, n_left, n_right, cover)
KNOWN_COVERS = {
    "unique_peptides": ([(0, 0), (1, 1), (2, 2)], 3, 3, [True, True, True]),
    "subset_protein": ([(0, 0), (0, 1), (0, 2), (1, 0), (1, 1)], 2, 3, [True, False]),
    "shared_peptide": ([(0, 0), (0, 1), (1, 1), (1, 2)], 2, 3, [True, True]),
    "empty": ([], 0, 0, []),
    "single": ([(0, 0)], 1, 1, [True]),
}


# ---------------------------------------------------------------------------------------------------- edges
def ring(k: int, prefix="R", unique_every=0):
    """k proteins in a ring: peptide i is shared by proteins i and i+1 (mod k); every unique_every-th protein also has a unique peptide."""
    lists = [[f"{prefix}{i}", f"{prefix}{(i + 1) % k}"] for i in range(k)]
    if unique_every:
        lists += [[f"{prefix}{i}"] for i in range(0, k, unique_every)]
    return lists


def edge_cases():
    A, B, C, D = "A", "B", "C", "D"
    return {
        "repeated_name": make([[A, A], [A, B], [B, C], [C], [D, D, D]], [0] * 5),
        "repeated_name_only": make([[A, A], [A]], [0, 0]),
        "no_proteins": make([[], [A], [], [A, B]], [0, 0, 1, 0]),
        "nan_q": make([[A], [B], [A, C]], [0, 0, 0], q=[NAN, 0.001, NAN]),
        "threshold_nan": make([[A], [B], [A, B]], [0, 0, 0], threshold=NAN),
        "threshold_below_0": make([[A], [B], [A, B]], [0, 0, 0], q=[-0.0, -1.0, 0.0], threshold=-0.5),
        "threshold_above_1": make([[A], [B], [A, B]], [0, 0, 0], q=[0.5, 1.0, 2.0], threshold=1.5),
        "q_equals_threshold": make([[A], [B], [C]], [0, 0, 0], q=[0.01, f32(0.01), 0.0100001]),
        "no_threshold": make([[A], [B], [A, B, C]], [0, 0, 0], q=[0.5, 1.0, 0.99], threshold=None),
        "tie_last_index": make([[A, B], [B, C], [C, A]], [0, 0, 0]),
        "tie_original_degree": make([[A], [A, B], [A, C], [B, C], [C, D], [B, D]], [0] * 6),
        "ring_7": make(ring(7), None),
        "ring_9_uniques": make(ring(9, unique_every=4), None),
        "giant_ring": make(ring(4000), None, seed=3),
        "giant_ring_uniques": make(ring(3001, unique_every=50), None, seed=4),
        "fallback_shares_entry": make([[A], [A], [B], [A]], [0, 0, 0, 1], q=[0.001, 0.5, 0.5, 0.0], pep_idx=[0, 1, 2, 3, 0, 3], q_rows=True),
        "same_name_both_sides": make([[A], [A], [B], [B]], [0, 1, 0, 1], pep_idx=[0, 1, 2, 3, 1, 0], generate_decoys=False),
        "same_name_both_sides_tagged": make([[A], [A], [B], [B]], [0, 1, 0, 1], pep_idx=[0, 1, 2, 3, 1, 0], generate_decoys=True),
        "label_inconsistent": make([[A], [A], [B], [B, C]], [0, 1, 0, 1], label=[1, 1, -1, 1], generate_decoys=True),
        "label_inconsistent_untagged": make([[A], [A], [B], [B, C]], [0, 1, 0, 1], label=[1, 1, -1, 1], generate_decoys=False),
        "grouping_off_tagged": make([[A, B], [A], [C]], [0, 1, 1], protein_grouping=False, generate_decoys=True),
    }


def _fix_rows(case):
    # make(..., q_rows=True) keeps one q per row when pep_idx repeats peptides
    if case.pop("q_rows", False):
        q = case["peptide_q"]
        case["peptide_q"] = np.asarray([q[p] for p in case["pep_idx"]], f32)
    return case


def random_case(seed: int, n_pep: int = 60, n_rows: int = 200):
    """Small random workloads: a pool of 12 names, lists of 0..4 names with repeats, labels that disagree with the decoy flag now and then,
    q-values with NaN and values on the threshold, and a threshold drawn from the edge values."""
    rng = np.random.default_rng(seed)
    pool = [f"N{k}" for k in range(12)]
    proteins = [[pool[j] for j in rng.integers(0, len(pool), int(rng.integers(0, 5)))] for _ in range(n_pep)]
    decoy = (rng.random(n_pep) < 0.3).astype(np.uint8)
    idx = rng.integers(0, n_pep, n_rows).astype(np.uint32)
    label = np.where(decoy[idx] != 0, -1, 1).astype(np.int32)
    flip = rng.random(n_rows) < 0.08
    label[flip] = -label[flip]
    thresholds = [0.01, 0.05, NAN, -0.5, 1.5, None, 0.25]
    threshold = thresholds[seed % len(thresholds)]
    q = rng.choice(np.array([0.0, 0.001, 0.01, 0.05, 0.25, 0.5, 1.0, NAN], f32), n_rows)
    cont = rng.random(n_rows) < 0.3
    q[cont] = rng.random(int(cont.sum())).astype(f32)
    return make(proteins, decoy, q=q, label=label, pep_idx=idx, threshold=threshold, generate_decoys=bool(seed % 2), protein_grouping=seed % 11 != 5,
                seed=seed)


def family_case(n_rows: int, seed: int, generate_decoys: bool = True):
    """Proteins in isoform-like families over a make_peptides table: each family has 1..6 proteins in 1..2 subfamilies; a peptide is unique to
    a protein, shared by two neighbouring proteins, shared within a subfamily or shared by the whole family (some proteins have no unique
    peptide, so the greedy has work), and
    a decoy peptide carries its target's names. Rows are drawn with repeats; targets score higher and have lower peptide q-values."""
    rng = np.random.default_rng(seed)
    pep = synth.make_peptides(max(1000, n_rows // 2), seed=seed)
    n = len(pep)
    proteins, fam = [], 0
    while len(proteins) < n:
        k = int(rng.integers(1, 7))
        members = [f"F{fam}_{j}" for j in range(k)]
        split = int(rng.integers(1, k)) if k > 1 and rng.random() < 0.6 else k
        subs = [members[:split], members[split:]] if split < k else [members]
        for m in members:
            proteins += [[m]] * int(rng.choice([0, 1, 2, 3], p=[0.3, 0.3, 0.25, 0.15]))
        for s in subs:
            if len(s) > 1:
                proteins += [list(rng.permutation(s))] * int(rng.integers(0, 3))
        for j in range(k - 1):   # exons shared by neighbouring isoforms: chains the greedy has to cut
            if rng.random() < 0.5:
                proteins.append([members[j], members[j + 1]])
        if k > 1:
            proteins += [list(rng.permutation(members))] * int(rng.integers(0, 2))
        fam += 1
    proteins = proteins[:n]
    order = rng.permutation(n)
    proteins = [proteins[i] for i in order]
    decoy = np.asarray(pep.decoy, np.uint8)
    idx = rng.integers(0, n, n_rows).astype(np.uint32)
    dec_rows = decoy[idx] != 0
    label = np.where(dec_rows, -1, 1).astype(np.int32)
    q = np.where(dec_rows, rng.random(n_rows), rng.exponential(0.02, n_rows)).astype(f32)
    q[rng.random(n_rows) < 0.01] = NAN
    score = (rng.normal(0.0, 1.0, n_rows) + np.where(dec_rows, 0.0, 4.0)).astype(f32)
    return make(proteins, decoy, q=q, label=label, pep_idx=idx, score=score, generate_decoys=generate_decoys, peptides=pep, seed=seed)


def fasta_case(seed: int, generate_decoys: bool, n_proteins: int = 60, n_rows: int = 3000):
    """A database digested from a seeded FASTA by the CPU oracle (tests/picked_cases.py fasta_case): real protein lists and shared peptides."""
    import picked_cases as PC
    c = PC.fasta_case(seed, generate_decoys, n_proteins, n_rows)
    rng = np.random.default_rng(seed + 99)
    pep, idx = c["peptides"], c["pep_idx"]
    dec_rows = np.asarray(pep.decoy)[idx] != 0
    q = np.where(dec_rows, rng.random(len(idx)), rng.exponential(0.02, len(idx))).astype(f32)
    return make(c["proteins"], pep.decoy, q=q, pep_idx=idx, score=c["score"], generate_decoys=generate_decoys, peptides=pep, seed=seed)


def random_multigraph(seed: int, n_left: int = 300, n_right: int = 400, n_edges: int = 900):
    """Edges (left, right) with parallel edges, isolated nodes and small degrees, so that forced picks, ties and multi-pick components occur."""
    rng = np.random.default_rng(seed)
    left = rng.integers(0, n_left, n_edges)
    right = np.clip(left * n_right // max(n_left, 1) + rng.integers(-3, 4, n_edges), 0, n_right - 1)   # local structure: many components
    dup = rng.random(n_edges) < 0.1
    left = np.concatenate([left, left[dup]]).astype(np.uint32)
    right = np.concatenate([right, right[dup]]).astype(np.uint32)
    return left, right, n_left, n_right


def ring_graph(k: int):
    """The giant component of the cover hook: k groups in a ring, right node i shared by groups i and i+1 (mod k)."""
    left = np.concatenate([np.arange(k), (np.arange(k) + 1) % k]).astype(np.uint32)
    right = np.concatenate([np.arange(k), np.arange(k)]).astype(np.uint32)
    return left, right, k, k


def all_small_cases():
    cases = {f"known_{k}": v for k, v in known_cases().items()}
    cases.update({f"edge_{k}": _fix_rows(v) for k, v in edge_cases().items()})
    cases.update({f"random_{s}": random_case(s) for s in range(14)})
    return cases


# ---------------------------------------------------------------------------------------------------- runners
def oracle(case):
    from oracle_ml import ml_oracle
    return ml_oracle.protein_groups(case["decoy"], case["proteins"], case["pep_idx"], case["label"], case["peptide_q"], case["score"],
                                    case["protein_grouping"], case["threshold"], case["generate_decoys"], case["decoy_tag"])


def reference(case, kde=None):
    import protein_group_reference as R
    return R.run(case, kde=kde)


def rows_of(case):
    from sage_b200.api import FEATURE_DTYPE
    rows = np.zeros(len(case["pep_idx"]), FEATURE_DTYPE)
    rows["peptide_idx"] = case["pep_idx"]
    rows["label"] = case["label"]
    return rows


def device(case, device_id=0):
    """sage_b200.protein_groups on the case, with the strings and the group tables built from ids as the oracle reports them."""
    import sage_b200
    from sage_b200 import api
    off, ids, names = name_ids(case)
    rows = rows_of(case)
    res = sage_b200.protein_groups(case["peptides"], rows, case["peptide_q"], case["score"], off, ids, len(names), case["protein_grouping"], case["threshold"],
                                   case["generate_decoys"], device=device_id)
    res["protein_groups"] = sage_b200.protein_group_strings(res, rows, case["peptides"], off, ids, names, case["decoy_tag"], case["generate_decoys"])
    tables, g0 = [], 0
    for k in range(2):
        g1 = g0 + res["groups"][k]
        tables.append([(int(res["group_covered"][g]), int(res["group_decoy"][g]), api.group_string(res, g, names, generate_decoys=False)) for g in range(g0, g1)])
        g0 = g1
    res["tables"] = tables
    return res


ROW_KEYS = ("protein_groups", "num_protein_groups", "pass", "protein_group_q")
SCALAR_KEYS = ("passing", "entries", "tables", "peptides", "meta_peptides", "groups", "covered", "greedy_picks", "annotated")


def same(got, want, what):
    """Exact equality of every output both sides report; q-values bit for bit."""
    for k in ROW_KEYS:
        g, w = got[k], want[k]
        if isinstance(w, np.ndarray):
            g = np.asarray(g)
            if w.dtype == np.float32:
                bad = np.flatnonzero(g.view(np.uint32) != w.view(np.uint32))
            else:
                bad = np.flatnonzero(g != w)
            assert bad.size == 0, f"{what}: {k} differs at rows {bad[:5]}: {g[bad[:5]]} vs {w[bad[:5]]}"
        else:
            bad = [i for i, (a, b) in enumerate(zip(g, w)) if a != b]
            assert len(g) == len(w) and not bad, f"{what}: {k} differs at rows {bad[:5]}: {[g[i] for i in bad[:5]]} vs {[w[i] for i in bad[:5]]}"
    for k in SCALAR_KEYS:
        assert got[k] == want[k], f"{what}: {k} {str(got[k])[:300]} != {str(want[k])[:300]}"
