"""Workloads of the predict_rt stage (retention-time alignment, RT and mobility models), shared by the CPU and GPU tests. Each entry: name ->
dict(pep, rows, file_id, n_files)."""
import numpy as np

from sage_b200 import Peptides, synth

RT_CHUNK = 1024   # rt.cuh / ml_oracle.cpp / ml_reference.py


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
    out.update(edge_cases())
    return out


def _all_targets(pep, n, n_files, seed, mobility=True):
    """n rows, every one a target in training (q = 1/n <= 0.01 needs n >= 100)."""
    rows, fid = synth.make_rt_psms(pep, n, n_files, seed=seed, mobility=mobility)
    rows["label"] = 1
    return rows, fid


def edge_cases():
    """Peptide lengths around the embedding's 32-lane stride, u8 charges, clamped predictions and targets, k_rt_predict's RT_TILE edges and a
    single (peptide, file) training set."""
    out = {}
    rng = np.random.default_rng(31)
    valid = np.array(list("ACDEFGHIKLMNPQRSTVWYUO"))
    seqs = ["".join(rng.choice(valid, n)) for n in (31, 32, 33, 64, 65, 255) for _ in range(20)]
    lpep = peptides_from(seqs, rng.uniform(3000.0, 30000.0, len(seqs)))
    rows, fid = synth.make_rt_psms(lpep, 6000, 3, seed=32, mobility=True)
    out["lengths_31_to_255"] = _case(lpep, rows, fid, 3)
    pep = base_peptides()
    rows, fid = synth.make_rt_psms(pep, 8000, 3, seed=33, mobility=True)
    rows["charge"] = np.array([1, 255, 257])[np.arange(8000) % 3]                     # the low byte: 257 reads as 1
    dec = rows["label"] == -1
    rows["charge"][dec] = np.array([0, 256])[np.arange(int(dec.sum())) % 2]           # decoys (never trained on) at z = 0: 1/z and m/z inf
    out["charges_u8"] = _case(pep, rows, fid, 3)
    rows, fid = synth.make_rt_psms(pep, 4000, 3, seed=34, mobility=True)
    rows["charge"] = np.array([0, 1, 255, 256, 257])[np.arange(4000) % 5]              # z = 0 among the training rows: the mobility fit fails
    out["charges_zero_trained"] = _case(pep, rows, fid, 3)
    rows, fid = synth.make_rt_psms(pep, 8000, 3, seed=35, mobility=True)
    odd = np.nonzero(rows["label"] == -1)[0]
    cpep = peptides_from([pep.sequence(i) for i in range(len(pep.mono))] + [a * 255 for a in "ACDEFGHIKLMNPQRSTVWYUO"] + ["G"],
                         np.concatenate([pep.mono, np.full(22, 28000.0), [57.0]]))
    rows["peptide_idx"][odd[1::2]] = len(pep.mono) + np.arange(len(odd[1::2])) % 23    # untrained outliers: predictions past both clamps
    rows["ims"][np.nonzero(rows["label"] == 1)[0][::4]] *= 4.0                         # mobility targets past 2 and below 0
    rows["ims"][np.nonzero(rows["label"] == 1)[0][1::9]] *= -1.0
    out["clamps"] = _case(cpep, rows, fid, 3)
    rows, fid = synth.make_rt_psms(pep, 4000, 3, seed=36, mobility=True)
    rows["ims"][np.argsort(rows["poisson"])[5]] = np.nan                                # a NaN mobility target: NaN coefficients
    out["ims_nan_target"] = _case(pep, rows, fid, 3)
    for n in (127, 128, 129):                                                          # RT_TILE = 32 rows per k_rt_predict warp
        out[f"predict_rows_{n}"] = _case(pep, *_all_targets(pep, n, 1, seed=n), 1)
    rows, fid = _all_targets(pep, 150, 2, seed=37)
    rows["peptide_idx"] = rows["peptide_idx"][0]
    fid[:] = 1
    out["one_segment"] = _case(pep, rows, fid, 2)                                      # one (peptide, file) pair: one matrix row, one entry
    return out
