"""Seeded workloads of picked FDR (fdr.rs): hand-made peptide tables that reach the key and score edges, and make_peptides tables at size.
Each case is dict(peptides, pep_idx, score, n_proteins, protein, cterm, generate_decoys)."""
from __future__ import annotations

import numpy as np

from sage_b200 import Peptides, synth

f32 = np.float32
F32_MIN = f32(-3.40282347e38)
NAN = f32("nan")


def table(specs) -> Peptides:
    """specs: [(sequence, mods or None, nterm (NaN = None), decoy)]."""
    off, seq, mods, nterm, decoy = [0], [], [], [], []
    for s, m, nt, d in specs:
        seq += list(s.encode())
        mods += list(m) if m is not None else [0.0] * len(s)
        off.append(len(seq))
        nterm.append(nt)
        decoy.append(d)
    n = len(specs)
    return Peptides(np.array(off, np.uint32), np.array(seq, np.uint8), np.array(mods, f32), np.array(nterm, f32), np.zeros(n, f32),
                    np.array(decoy, np.uint8), np.zeros(n, np.uint8))


def rev(s: str) -> str:
    n = len(s) - 1
    return s[0] + s[1:n][::-1] + s[n:] if n > 1 else s


def edge_specs():
    """Lengths 1..4 (reverse is a no-op up to 3), nterm None / +0 / -0, modifications +-0 and NaN, variable modifications that the reversal
    moves; each target with its decoy (interior reversed, as generate_decoys makes them) and some without."""
    sp = []
    for s in ("K", "AK", "ACK", "ACDK", "PEPTIDEK", "MSTYLK", "GGGGK"):
        sp += [(s, None, NAN, 0), (rev(s), None, NAN, 1)]
    sp += [("ACDK", None, f32(0.0), 0), ("ACDK", None, f32(-0.0), 0), ("ACDK", None, f32(42.010565), 0)]
    sp += [("MSTK", [0.0, 15.9949, 0.0, 0.0], NAN, 0), ("MTSK", [0.0, 0.0, 15.9949, 0.0], NAN, 1)]   # the decoy's key is the target's
    sp += [("MSTK", [0.0, -0.0, 0.0, 0.0], NAN, 0)]                                                   # -0.0 prints nothing: key "MSTK"
    sp += [("WYLK", [0.0, float("nan"), 0.0, 0.0], NAN, 0), ("WLYK", [0.0, 0.0, float("nan"), 0.0], NAN, 1)]
    sp += [("QRSTVK", [0.0, 79.96633, 0.0, 1e-7, 0.0, 0.0], NAN, 0), ("DECOYK", None, NAN, 1), ("TARGETK", None, NAN, 0)]
    sp += [("NNK", [0.0, 0.0, -17.026549], f32(0.0), 1), ("NNK", [0.0, 0.0, -17.026549], NAN, 0)]
    return sp


def edge_scores(rng, n):
    s = rng.normal(0.0, 2.0, n).astype(f32)
    special = np.array([np.nan, np.inf, -np.inf, F32_MIN, 0.0, -0.0, 1.5, 1.5], f32)
    pick = rng.random(n) < 0.15
    s[pick] = special[rng.integers(0, len(special), pick.sum())]
    return s


def edge_case(seed: int, generate_decoys: bool, n_rows: int = 400, clash_free: bool = True):
    rng = np.random.default_rng(seed)
    specs = edge_specs()
    if not generate_decoys:
        specs = [s for s in specs if s[0] != "MSTK" or s[1] is None or s[1][1] != -0.0]
    pep = table(specs)
    n = len(pep)
    n_prot = rng.integers(0, 3, n).astype(np.uint32)
    protein = rng.integers(0, 6, n).astype(np.uint32)
    cterm = np.full(n, np.nan, f32)
    cterm[rng.random(n) < 0.2] = f32(-0.0)
    cterm[rng.random(n) < 0.1] = f32(0.0)
    idx = rng.integers(0, n, n_rows).astype(np.uint32)
    case = dict(peptides=pep, pep_idx=idx, score=edge_scores(rng, n_rows), n_proteins=n_prot, protein=protein, cterm=cterm, generate_decoys=generate_decoys)
    if clash_free:
        import picked_reference as R
        # with generate_decoys, "MSTK" with -0.0 and the plain-key peptides of one side would clash: keep one PeptideIx per (key, side)
        seen, keep = {}, []
        for p in idx.tolist():
            k = (R.peptide_key(pep, p, generate_decoys, cterm), int(pep.decoy[p]))
            keep.append(seen.setdefault(k, p) == p)
        keep = np.array(keep)
        case["pep_idx"], case["score"] = idx[keep], case["score"][keep]
    return case


def synth_case(n_rows: int, seed: int, generate_decoys: bool = True, n_target: int = 20000):
    """make_peptides table with synthetic protein ids: 0, 1 and 2+ proteins per peptide; rows drawn with repeats, decoys scoring lower."""
    rng = np.random.default_rng(seed)
    pep = synth.make_peptides(n_target, seed=seed)
    n = len(pep)
    idx = rng.integers(0, n, n_rows).astype(np.uint32)
    score = (rng.normal(0.0, 1.0, n_rows) + np.where(pep.decoy[idx] != 0, 0.0, 1.5)).astype(f32)
    n_prot = np.where(rng.random(n) < 0.8, 1, rng.integers(0, 4, n)).astype(np.uint32)
    protein = rng.integers(0, max(1, n // 20), n).astype(np.uint32)
    return dict(peptides=pep, pep_idx=idx, score=score, n_proteins=n_prot, protein=protein, cterm=None, generate_decoys=generate_decoys)


def degenerate_cases():
    pep = table([("PEPTIDEK", None, NAN, 0), ("PEDITPEK", None, NAN, 1), ("SAMPLEK", None, NAN, 0), ("SELPMAK", None, NAN, 1)])
    one = np.ones(4, np.uint32)
    prot = np.array([0, 0, 1, 1], np.uint32)
    base = dict(peptides=pep, n_proteins=one, protein=prot, cterm=None, generate_decoys=True)
    return {
        "one_row": dict(base, pep_idx=np.array([2], np.uint32), score=f32([3.0])),
        "no_decoys": dict(base, pep_idx=np.array([0, 2, 0, 2], np.uint32), score=f32([1.0, 2.0, 3.0, 0.5])),
        "no_targets": dict(base, pep_idx=np.array([1, 3, 3], np.uint32), score=f32([1.0, 2.0, 3.0])),
        "all_equal": dict(base, pep_idx=np.array([0, 1, 2, 3, 0, 3], np.uint32), score=f32([2.0] * 6)),
        "decoy_first": dict(base, pep_idx=np.array([1, 0, 3, 2, 1], np.uint32), score=f32([4.0, 1.0, -1.0, 5.0, 0.25])),
        # without generate_decoys one protein id on both sides: its target and decoy rows share one Ix, the later sorted row wins
        "protein_both_sides": dict(base, generate_decoys=False, pep_idx=np.array([0, 1, 2, 3, 0], np.uint32), score=f32([1.0, 2.0, 3.0, 4.0, 0.5])),
    }


def clash_case():
    """Two distinct target peptides with one key ("MSTK": a -0.0 modification prints nothing): the reference panics."""
    pep = table([("MSTK", None, NAN, 0), ("MSTK", [0.0, -0.0, 0.0, 0.0], NAN, 0)])
    return dict(peptides=pep, pep_idx=np.array([0, 1], np.uint32), score=f32([1.0, 2.0]), n_proteins=np.ones(2, np.uint32),
                protein=np.zeros(2, np.uint32), cterm=None, generate_decoys=True)


def protein_names(case):
    """Peptide::proteins for the reference: one name per id where n_proteins == 1, distinct filler names otherwise."""
    return [[f"P{int(case['protein'][p])}"] if k == 1 else [f"Q{p}_{j}" for j in range(int(k))] for p, k in enumerate(case["n_proteins"])]


def reference(case, kde=None):
    import picked_reference as R
    pep = case["peptides"]
    q, pp, pe = R.picked_peptide(pep, case["pep_idx"], case["score"], case["generate_decoys"], case["cterm"], kde=kde)
    proteins = case.get("proteins") or protein_names(case)
    pq, prp, pre = R.picked_protein(pep.decoy, case["pep_idx"], case["score"], proteins, case["generate_decoys"], kde=kde)
    return dict(peptide_q=q, protein_q=pq, peptide_passing=pp, protein_passing=prp, peptide_entries=pe, protein_entries=pre)


def rows_of(case):
    from sage_b200.api import FEATURE_DTYPE
    rows = np.zeros(len(case["pep_idx"]), FEATURE_DTYPE)
    rows["peptide_idx"] = case["pep_idx"]
    rows["label"] = 1
    return rows


def device(case, device_id=0):
    import sage_b200
    return sage_b200.picked_fdr(case["peptides"], rows_of(case), case["score"], case["n_proteins"], case["protein"], cterm=case["cterm"],
                                generate_decoys=case["generate_decoys"], device=device_id)


def fasta_case(seed: int, generate_decoys: bool, n_proteins: int = 60, n_rows: int = 3000):
    """A database digested from a seeded FASTA by the CPU oracle (OracleDB.from_fasta): real protein lists, peptides shared between proteins
    (each protein repeats a segment of an earlier one), an N-terminal variable modification. Without generate_decoys the FASTA carries
    tagged decoy proteins (the reversed sequences)."""
    from oracle.oracle import OracleDB
    rng = np.random.default_rng(seed)
    aa = np.array(list("ACDEFGHIKLMNPQRSTVWY"))
    seqs = []
    for i in range(n_proteins):
        s = "".join(rng.choice(aa, int(rng.integers(120, 400))))
        if seqs and rng.random() < 0.5:
            src = seqs[int(rng.integers(0, len(seqs)))]
            a = int(rng.integers(0, len(src) - 60))
            s = s[:50] + src[a:a + 60] + s[50:]
        seqs.append(s)
    text = "".join(f">sp|P{i:05d}\n{s}\n" for i, s in enumerate(seqs))
    if not generate_decoys:
        text += "".join(f">rev_sp|P{i:05d}\n{s[::-1]}\n" for i, s in enumerate(seqs))
    db = OracleDB.from_fasta(text, missed_cleavages=1, variable_mods={"[": [42.010565]}, generate_decoys=generate_decoys)
    e = db.export()
    pep = Peptides(e["seq_off"], e["seq"], e["mods"], e["nterm"], e["pep_mono"], e["decoy"], e["missed"])
    proteins = [db.peptide_proteins(i) for i in range(len(pep))]
    ids: dict = {}
    protein = np.array([ids.setdefault(lst[0], len(ids)) if len(lst) == 1 else 0 for lst in proteins], np.uint32)
    idx = rng.integers(0, len(pep), n_rows).astype(np.uint32)
    score = (rng.normal(0.0, 1.0, n_rows) + np.where(pep.decoy[idx] != 0, 0.0, 2.0)).astype(f32)
    return dict(peptides=pep, pep_idx=idx, score=score, n_proteins=np.array([len(x) for x in proteins], np.uint32), protein=protein,
                cterm=e["cterm"], generate_decoys=generate_decoys, proteins=proteins, db=db)


def oracle(case):
    from oracle_ml import ml_oracle
    proteins = case.get("proteins") or protein_names(case)
    return ml_oracle.picked_fdr(case["peptides"], case["pep_idx"], case["score"], proteins, cterm=case["cterm"], generate_decoys=case["generate_decoys"])


def tied_case(seed: int, generate_decoys: bool = True, n_rows: int = 5000):
    """Scores on a coarse grid: many entries whose forward and reverse scores are equal, where `is_decoy` (reverse >= forward) and the
    forward-before-reverse row order decide."""
    case = synth_case(n_rows, seed, generate_decoys, n_target=3000)
    case["score"] = (np.round(case["score"] * 2.0) / 2.0).astype(f32)
    return case
