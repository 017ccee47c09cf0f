"""A numpy / Python restatement of sage's picked FDR, written from crates/sage/src/fdr.rs and peptide.rs (cited as file:line), with real key
strings: Peptide::reverse and Display written out, Rust's shortest round-trip f32 formatting, Python dicts (insertion-ordered) for the maps.
TEST INFRASTRUCTURE ONLY: it shares no code with the device kernels (sage_b200/csrc/picked.cuh).

Where the Rust leaves an order to a HashMap or to rayon, this module uses the definitions of DESIGN.md §12:
- entries are ordered by the first row that reaches them (dict insertion order), which fixes the KDE's sample order and the rows' order
  before the stable sort (forward row before reverse row);
- f32::max is `v > acc ? v : acc`; f32::min on the q-values ignores NaN and keeps -0.0 over +0.0 (ml_reference.rust_min);
- when two rows carry one Ix, the later row in sorted order wins (rayon's ordered collect);
- two distinct peptides on one side with one key (the reference's panic) raise PickedClash.
The KDE and posterior_error are tests/ml_reference.py's (kde.rs), or any function with its signature (the C++ oracle's for large inputs).
"""
from __future__ import annotations

import math

import numpy as np

import ml_reference as ML

f32, f64 = np.float32, np.float64
F32_MIN = f32(-3.40282347e38)   # f32::MIN, Competition::default (fdr.rs:31-39)


class PickedClash(ValueError):
    def __init__(self, a: int, b: int):
        super().__init__(f"peptides {a} and {b} share a key on one side")
        self.peptides = (a, b)


# ---------------------------------------------------------------------------------------------------- peptide.rs
def fmt_plus(x) -> str:
    """`{:+}` of an f32: the shortest decimal that round-trips, never in exponent form, with its sign; NaN prints "NaN"."""
    x = f32(x)
    if math.isnan(x):
        return "NaN"
    if math.isinf(x):
        return "+inf" if x > 0 else "-inf"
    return np.format_float_positional(x, unique=True, trim="-", sign=True)


def reverse(seq: bytes, mods):
    """Peptide::reverse (peptide.rs:307-318): sequence[1..n] and modifications[1..n] reversed, n = len - 1, when n > 1."""
    s, m = bytearray(seq), list(mods)
    n = max(len(s) - 1, 0)
    if n > 1:
        s[1:n] = s[1:n][::-1]
        m[1:n] = m[1:n][::-1]
    return bytes(s), m


def display(seq: bytes, mods, nterm, cterm) -> str:
    """impl Display for Peptide (peptide.rs:390-406). nterm / cterm: NaN (or None) = None."""
    out = []
    if nterm is not None and not math.isnan(nterm):
        out.append(f"[{fmt_plus(nterm)}]-")
    for c, m in zip(seq, mods):
        out.append(f"{chr(c)}[{fmt_plus(m)}]" if f32(m) != 0.0 or math.isnan(m) else chr(c))
    if cterm is not None and not math.isnan(cterm):
        out.append(f"-[{fmt_plus(cterm)}]")
    return "".join(out)


def peptide_key(peptides, i: int, generate_decoys: bool, cterm=None) -> str:
    """fdr.rs:128-131: `peptide.reverse().to_string()` when generate_decoys && decoy, else `peptide.to_string()`."""
    a, b = int(peptides.seq_off[i]), int(peptides.seq_off[i + 1])
    seq, mods = bytes(peptides.seq[a:b]), [f32(m) for m in peptides.mods[a:b]]
    if generate_decoys and peptides.decoy[i]:
        seq, mods = reverse(seq, mods)
    return display(seq, mods, f32(peptides.nterm[i]), None if cterm is None else f32(cterm[i]))


# ---------------------------------------------------------------------------------------------------- fdr.rs
def f32_max(acc, v):
    """f32::max as DESIGN.md §12 defines it."""
    return v if v > acc else acc


def q_tail(rows, pep_of, threshold):
    """fdr.rs:87-111 over rows [(ix, decoy, score f32)] in pre-sort order: stable descending sort by total_cmp, the running f32 sum of
    pep_of(sorted scores, decoy flags) from 1.0, target += 1.0, q = decoy / target, the suffix minimum from 1.0. Returns ([(ix, decoy, q)]
    in sorted order, passing)."""
    scores = np.array([r[2] for r in rows], f32)
    order = sorted(range(len(rows)), key=lambda j: -int(ML.total_key32(scores[j])))   # `b.score.total_cmp(&a.score)`, stable
    rows = [rows[j] for j in order]
    peps = pep_of(np.array([r[2] for r in rows], f32), np.array([r[1] for r in rows], bool))
    decoy, target = f32(1.0), f32(0.0)
    qs = []
    with np.errstate(all="ignore"):
        for (ix, dec, _), pep in zip(rows, peps):
            decoy = f32(decoy + f32(pep))
            if not dec:
                target = f32(target + f32(1.0))
            qs.append(f32(decoy / target))
    q_min, passing = f32(1.0), 0
    for k in range(len(rows) - 1, -1, -1):
        q_min = f32(ML.rust_min(float(q_min), float(qs[k])))
        qs[k] = q_min
        if q_min <= threshold and not rows[k][1]:
            passing += 1
    return [(r[0], r[1], q) for r, q in zip(rows, qs)], passing


def assign_q_value(entries: dict, kde=None):
    """Competition::assign_q_value (fdr.rs:59-120). entries: key -> [forward, forward_ix, reverse, reverse_ix] in insertion order.
    Returns ({ix: q}, passing)."""
    kde = kde or ML.kde_build
    comps = list(entries.values())
    score = [float(f64(r if r > f else f)) for f, _, r, _ in comps]              # score(): forward.max(reverse), fdr.rs:43-45
    is_decoy = [bool(r >= f) for f, _, r, _ in comps]                            # fdr.rs:47-49
    bins, mn, step = kde(np.array(score, f64), np.array(is_decoy, bool))         # Builder::default().build, fdr.rs:51-57
    est = ML.Estimator(bins, mn, step)
    rows = []
    for f, fix, r, rix in comps:                                                 # fdr.rs:71-85
        if fix is not None:
            rows.append((fix, False, f))
        if rix is not None:
            rows.append((rix, True, r))
    if not rows:
        return {}, 0
    pep_of = lambda s, d: est.posterior_error(s.astype(f64)).astype(f32)         # noqa: E731  fdr.rs:92
    out, passing = q_tail(rows, pep_of, f32(0.01))
    qmap = {}
    for ix, _, q in out:                                                         # fdr.rs:113-117: later rows overwrite
        qmap[ix] = q
    return qmap, passing


def picked_peptide(peptides, pep_idx, score, generate_decoys=True, cterm=None, kde=None, keys=None):
    """picked_peptide (fdr.rs:123-153): (peptide_q per row, passing, entries). keys: optional precomputed key string per peptide."""
    cache = {} if keys is None else keys
    entries: dict = {}
    for p, s in zip(np.asarray(pep_idx).tolist(), np.asarray(score, f32)):
        if p not in cache:
            cache[p] = peptide_key(peptides, p, generate_decoys, cterm)
        e = entries.setdefault(cache[p], [F32_MIN, None, F32_MIN, None])
        side = 2 if peptides.decoy[p] else 0
        if e[side + 1] is not None and e[side + 1] != p:
            raise PickedClash(e[side + 1], p)
        e[side] = f32_max(e[side], s)
        e[side + 1] = p
    qmap, passing = assign_q_value(entries, kde)
    return np.array([qmap[p] for p in np.asarray(pep_idx).tolist()], f32), passing, len(entries)


def picked_protein(decoy_of, pep_idx, score, protein_names, generate_decoys=True, decoy_tag="rev_", kde=None):
    """picked_protein (fdr.rs:155-190). protein_names[p]: Peptide::proteins of peptide p (a list of names); decoy_of[p]: Peptide::decoy.
    (protein_q per row, passing, entries)."""
    def ix_of(p):                                                                # Peptide::proteins(decoy_tag, generate_decoys), peptide.rs:81-96
        names = protein_names[p]
        return ";".join(decoy_tag + s if (decoy_of[p] and generate_decoys) else s for s in names)
    entries: dict = {}
    for p, s in zip(np.asarray(pep_idx).tolist(), np.asarray(score, f32)):
        if len(protein_names[p]) != 1:
            continue
        e = entries.setdefault(tuple(protein_names[p]), [F32_MIN, None, F32_MIN, None])
        side = 2 if decoy_of[p] else 0
        e[side] = f32_max(e[side], s)
        e[side + 1] = ix_of(p)
    qmap, passing = assign_q_value(entries, kde)
    q = np.array([qmap[ix_of(p)] if len(protein_names[p]) == 1 else f32(1.0) for p in np.asarray(pep_idx).tolist()], f32)
    return q, passing, len(entries)


def picked_precursor(score, decoy):
    """picked_precursor (fdr.rs:228-287) over the rows in the given order: (q per row, passing)."""
    rows = [(i, bool(d), f32(s)) for i, (s, d) in enumerate(zip(np.asarray(score, f64), np.asarray(decoy, bool)))]
    if not rows:
        return np.zeros(0, f32), 0
    out, passing = q_tail(rows, lambda s, d: np.where(d, f32(1.0), f32(0.0)).astype(f32), f32(0.05))
    q = np.zeros(len(rows), f32)
    for ix, _, v in out:
        q[ix] = v
    return q, passing
