"""Workloads of the predict_rt stage (retention-time alignment, RT and mobility models), shared by the CPU and GPU tests. Each entry: name ->
dict(pep, rows, file_id, n_files)."""
import numpy as np

from sage_b200 import Peptides, synth

RT_CHUNK = 1024   # rt.cuh / ml_oracle.cpp


def peptides_from(seqs, mono=None) -> Peptides:
    """A peptide table from sequences (no modifications), every one a target."""
    lens = np.array([len(s) for s in seqs])
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
    seq = np.frombuffer("".join(seqs).encode(), np.uint8).copy()
    mono = np.asarray(mono if mono is not None else 500.0 + 110.0 * lens, np.float32)
    n = len(seqs)
    return Peptides(seq_off=off, seq=seq, mods=np.zeros(len(seq), np.float32), nterm=np.full(n, np.nan, np.float32), mono=mono,
                    decoy=np.zeros(n, np.uint8), missed=np.zeros(n, np.uint8))


_PEP = None


def base_peptides() -> Peptides:
    global _PEP
    if _PEP is None:
        _PEP = synth.make_peptides(6000, seed=101, static_c=True)
    return _PEP


def _case(pep, rows, fid, n_files):
    return dict(pep=pep, rows=rows, file_id=np.asarray(fid, np.uint32), n_files=int(n_files))


def training_set_of(pep, k, seed):
    """Exactly k training rows: k targets first in poisson order (q = 1/k), then k/2 decoys, then targets whose q-values stay above 0.01."""
    rows, fid = synth.make_rt_psms(pep, 2 * k, 3, seed=seed, mobility=True)
    rows["label"][:k], rows["label"][k:k + k // 2], rows["label"][k + k // 2:] = 1, -1, 1
    rows["poisson"][:k] = -10.0 - np.arange(k) * 1e-3
    rows["poisson"][k:] = np.linspace(-1.0, 0.0, 2 * k - k)
    return _case(pep, rows, fid, 3)


def cases():
    pep = base_peptides()
    out = {}
    for n, nf in ((1, 1), (2, 3), (100_000, 3), (100_000, 128), (1_000_000, 8)):
        rows, fid = synth.make_rt_psms(pep, n, nf, seed=n + nf, mobility=n >= 100_000)
        out[f"rows_{n}_files_{nf}"] = _case(pep, rows, fid, nf)
    for k in (RT_CHUNK - 1, RT_CHUNK, RT_CHUNK + 1):
        out[f"train_{k}"] = training_set_of(pep, k, seed=k)
    rows, fid = synth.make_rt_psms(pep, 4000, 3, seed=21, mobility=True)
    rows["label"] = np.where(np.arange(4000) % 2 == 0, 1, -1)                       # q about 1 everywhere: no training row
    rows["poisson"] = -5.0
    out["no_training"] = _case(pep, rows, fid, 3)
    rows, fid = synth.make_rt_psms(pep, 20_000, 4, seed=22, mobility=True)
    fid = np.where(fid == 2, 4, fid)                                                  # file 2 has no rows
    four = fid == 4
    rows["rt"][four] = -np.abs(rows["rt"][four])                                      # file 4: every RT <= 0, max_rt 0
    rows["rt"][np.nonzero(four)[0][::3]] = 0.0
    out["empty_and_zero_files"] = _case(pep, rows, fid, 5)
    rows, fid = synth.make_rt_psms(pep, 20_000, 3, seed=23, mobility=True)
    rows["rt"][::97] = np.nan                                                         # NaN RTs: f64::min skips them unless first
    rows["rt"][1::5] = np.round(rows["rt"][1::5])                                     # integral RTs: ceil is the value itself
    rows["rt"][np.nonzero(fid == 1)[0][:3]] = np.float32(6.0e9)                       # > 2^32: `as u32` saturates, file 1's max_rt
    out["odd_rts"] = _case(pep, rows, fid, 3)
    rows, fid = synth.make_rt_psms(pep, 20_000, 3, seed=24, mobility=True)
    true = np.nonzero(rows["poisson"] < -5)[0]
    zero_peps = rows["peptide_idx"][true[:30]]
    extra = rows[true[:90]].copy()                                                    # 30 peptides at RT 0 in every file: mean 0 is
    extra["peptide_idx"] = np.repeat(zero_peps, 3)                                    # not normal, the matrix row is dropped
    extra["rt"] = 0.0
    sel = np.isin(rows["peptide_idx"], zero_peps)
    rows["rt"][sel] = 0.0
    out["rt0_every_file"] = _case(pep, np.concatenate([rows, extra]), np.concatenate([fid, np.tile(np.arange(3, dtype=np.uint32), 30)]), 3)
    rows, fid = synth.make_rt_psms(pep, 6000, 3, seed=25, mobility=True)
    rows["poisson"] = np.round(rows["poisson"] * 2.0) / 2.0                           # many equal poisson values
    flip = rows[::200].copy()
    flip["label"] = -flip["label"]                                                    # the same poisson with the other label
    out["ties_mixed_labels"] = _case(pep, np.concatenate([rows, flip]), np.concatenate([fid, fid[::200]]), 3)
    rng = np.random.default_rng(26)
    letters = np.array(list("ACDEFGHIKLMNPQRSTVWYUOBJXZ"))
    seqs = ["".join(rng.choice(letters, rng.integers(1, 16))) for _ in range(400)] + ["U", "OB", "JXZ", "BUOZ", "XXXXX", "ZJBO"]
    opep = peptides_from(seqs, rng.uniform(200.0, 3000.0, len(seqs)))
    rows, fid = synth.make_rt_psms(opep, 30_000, 3, seed=27, mobility=True)
    out["odd_residues"] = _case(opep, rows, fid, 3)
    rows, fid = synth.make_rt_psms(pep, 20_000, 3, seed=28, mobility=False)
    out["no_mobility"] = _case(pep, rows, fid, 3)
    lens = np.diff(pep.seq_off.astype(np.int64))
    common = np.bincount(lens).argmax()
    same = np.nonzero(lens == common)[0]
    cpep = peptides_from([pep.sequence(i) for i in same], np.random.default_rng(29).uniform(1e6, 2e6, len(same)))
    rows, fid = synth.make_rt_psms(cpep, 20_000, 3, seed=29, mobility=True)
    rows["charge"] = 2                                                                # one charge, one length: a collinear design; the
    out["collinear"] = _case(cpep, rows, fid, 3)                                      # m/z column is half the mass column, bit for bit
    return out
