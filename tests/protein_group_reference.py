"""A Python restatement of sage's protein grouping and picked protein-group FDR, written from crates/sage/src/protein_grouping.rs and
fdr.rs:192-226, with Python sets, dicts and name strings. TEST INFRASTRUCTURE ONLY: it shares no code with the device kernels
(sage_b200/csrc/protein_groups.cuh) or the C++ oracle (oracle_ml); the q-values reuse tests/picked_reference.py's assign_q_value.

The cover is not the reference's loop: it is the form DESIGN.md §13 proves equal to it. The forced picks of the first trim come from the
original right degrees; then each connected component of what remains runs the greedy alone, picking the last index among the maxima of
(remaining, original). The C++ oracle runs the literal loop, so their agreement checks both facts.
"""
from __future__ import annotations

import math

import numpy as np

import picked_reference as PR

f32 = np.float32


def cover(edges, n_left: int, n_right: int):
    """BipartiteGraph::new(edges, n_left, n_right).into_cover() by the forced picks and a greedy per component: (cover, greedy picks)."""
    left_adj = [[] for _ in range(n_left)]
    right_adj = [[] for _ in range(n_right)]
    for l, r in edges:
        left_adj[l].append(r)
        right_adj[r].append(l)
    original = [len(a) for a in left_adj]
    covered = [False] * n_left
    right_covered = [False] * n_right
    for r in range(n_right):                       # a peptide seen by one edge forces its group
        if len(right_adj[r]) == 1:
            covered[right_adj[r][0]] = True
    for l in range(n_left):
        if covered[l]:
            for r in left_adj[l]:
                right_covered[r] = True
    remaining = [0 if covered[l] else sum(1 for r in left_adj[l] if not right_covered[r]) for l in range(n_left)]
    # components of the remaining graph, by a search from each group with remaining edges
    seen, picks = [False] * n_left, 0
    for start in range(n_left):
        if seen[start] or remaining[start] == 0:
            continue
        comp, stack, seen[start] = [], [start], True
        while stack:
            l = stack.pop()
            comp.append(l)
            for r in left_adj[l]:
                if right_covered[r]:
                    continue
                for l2 in right_adj[r]:
                    if not seen[l2]:
                        seen[l2] = True
                        stack.append(l2)
        comp.sort()
        while True:
            best = max(comp, key=lambda l: (remaining[l], original[l], l))
            if remaining[best] == 0:
                break
            covered[best] = True
            picks += 1
            for r in set(left_adj[best]):
                if right_covered[r]:
                    continue
                right_covered[r] = True
                for l2 in right_adj[r]:
                    remaining[l2] -= 1
    return covered, picks


def format_name(key, decoy_tag, generate_decoys):
    """ProteinIx::format: decoy_tag + name for a decoy key when generate_decoys."""
    name, decoy = key
    return decoy_tag + name if decoy and generate_decoys else name


def annotate(proteins, decoy, pep_idx, label, peptide_q, threshold, decoy_tag, generate_decoys, strings, pass_of, pass_no):
    """annotate_features at one threshold; fills strings / pass_of for rows still unannotated. Returns the pass's table and counts."""
    peptides = sorted({p for p, lab, q in zip(pep_idx, label, peptide_q) if lab != -1 and q < threshold})
    index = {}                                                   # (name, decoy) -> ProteinIx, by first encounter
    metas = set()
    for p in peptides:
        metas.add(tuple(sorted(index.setdefault((nm, bool(decoy[p])), len(index)) for nm in proteins[p])))
    evidence = {}                                                # ProteinIx -> meta-peptide indices, with multiplicity
    for i, meta in enumerate(sorted(metas)):
        for ix in meta:
            evidence.setdefault(ix, []).append(i)
    by_evidence = {}
    for ix, ev in evidence.items():
        by_evidence.setdefault(tuple(ev), []).append(ix)
    groups, edges = [], []
    for g, ev in enumerate(sorted(by_evidence)):
        groups.append(by_evidence[ev])
        edges += [(g, m) for m in ev]
    chosen, picks = cover(edges, len(groups), len(metas))
    key_of = {ix: key for key, ix in index.items()}
    group_string = ["/".join(sorted(format_name(key_of[ix], decoy_tag, generate_decoys) for ix in grp)) for grp in groups]
    table = [(int(c), int(key_of[grp[0]][1]), "/".join(sorted(key_of[ix][0] for ix in grp))) for grp, c in zip(groups, chosen)]
    to_groups = {}
    for g, grp in enumerate(groups):
        if chosen[g]:
            for ix in grp:
                to_groups.setdefault(key_of[ix], set()).add(g)
    annotated = 0
    for i, p in enumerate(pep_idx):
        if pass_of[i]:
            continue
        found = set()
        for nm in proteins[p]:
            found |= to_groups.get((nm, bool(decoy[p])), set())
        if found:
            strings[i] = ";".join(sorted(group_string[g] for g in found))
            pass_of[i] = pass_no
            annotated += 1
    counts = dict(peptides=len(peptides), meta_peptides=len(metas), groups=len(groups), covered=sum(chosen), greedy_picks=picks, annotated=annotated)
    return table, counts


def generate_protein_groups(proteins, decoy, pep_idx, label, peptide_q, protein_grouping=True, threshold=0.01, decoy_tag="rev_", generate_decoys=True):
    """generate_protein_groups (protein_grouping.rs): (strings, num_protein_groups, pass, tables, counts per pass)."""
    pep_idx = [int(p) for p in pep_idx]
    label = [int(x) for x in label]
    peptide_q = [f32(x) for x in peptide_q]
    n = len(pep_idx)
    strings, pass_of = [None] * n, [0] * n
    tables, counts = [[], []], [None, None]
    if protein_grouping:
        if threshold is not None:
            t = f32(threshold)                                   # f32::clamp(0.0, 1.0) keeps NaN
            t = t if math.isnan(t) else min(max(t, f32(0.0)), f32(1.0))
            tables[0], counts[0] = annotate(proteins, decoy, pep_idx, label, peptide_q, t, decoy_tag, generate_decoys, strings, pass_of, 1)
        tables[1], counts[1] = annotate(proteins, decoy, pep_idx, label, peptide_q, f32(1.0), decoy_tag, generate_decoys, strings, pass_of, 2)
    num = []
    for i, p in enumerate(pep_idx):
        if strings[i] is None:                                   # Peptide::proteins(decoy_tag, generate_decoys)
            strings[i] = ";".join(format_name((nm, bool(decoy[p])), decoy_tag, generate_decoys) for nm in proteins[p])
            num.append(len(proteins[p]))
        else:
            num.append(strings[i].count(";") + 1)
    zero = dict(peptides=0, meta_peptides=0, groups=0, covered=0, greedy_picks=0, annotated=0)
    return strings, num, pass_of, tables, [c or zero for c in counts]


def picked_protein_group(strings, num, decoy, pep_idx, score, kde=None):
    """picked_protein_group (fdr.rs:192-226): the key and the Ix are the string. (protein_group_q per row, passing, entries)."""
    entries = {}
    for s, k, p, sc in zip(strings, num, pep_idx, np.asarray(score, f32)):
        if k != 1:
            continue
        e = entries.setdefault(s, [PR.F32_MIN, None, PR.F32_MIN, None])
        side = 2 if decoy[int(p)] else 0
        e[side] = PR.f32_max(e[side], sc)
        e[side + 1] = s
    qmap, passing = PR.assign_q_value(entries, kde)
    q = np.array([qmap[s] if k == 1 else f32(1.0) for s, k in zip(strings, num)], f32)
    return q, passing, len(entries)


def run(case, kde=None) -> dict:
    """Both stages on a case of tests/protein_group_cases.py, in the oracle's result shape."""
    strings, num, passes, tables, counts = generate_protein_groups(case["proteins"], case["decoy"], case["pep_idx"], case["label"], case["peptide_q"],
                                                                   case["protein_grouping"], case["threshold"], case["decoy_tag"], case["generate_decoys"])
    q, passing, entries = picked_protein_group(strings, num, case["decoy"], case["pep_idx"], case["score"], kde=kde)
    res = dict(protein_groups=strings, num_protein_groups=np.array(num, np.uint32), protein_group_q=q, passing=passing, entries=entries, tables=tables,
               **{"pass": np.array(passes, np.uint8)})
    res.update({k: [c[k] for c in counts] for k in counts[0]})
    return res
