"""Edge workloads of label-free quantification, shared by the CPU tests (tests/test_lfq_reference.py: restatement against the oracle) and the
GPU tests (tests/test_gpu_lfq.py: device against the oracle), so both run the same inputs.

case(name) returns a dict: peptides (the table the feature map reads), settings, charges, features, alignments, batches (the add_ms1 calls, in
order) and, where the workload was built for them, the time warps its forward grids must produce (warps: file -> warp). The peptide table of
the synthetic workloads is PEPTIDES_SEED's, the table the GPU tests build their database from; a case whose table differs (composition) keeps
its row count, which is all the feature map needs of the database."""
from __future__ import annotations

import functools

import numpy as np

from sage_b200 import synth
from sage_b200.api import ALIGNMENT_DTYPE, LfqSettings, Ms1Batch, Peptides

from lfq_reference import RT_TOL, build_map

f32 = np.float32
PEPTIDES_SEED = 41
BIG = (1 << 24) + (1 << 20)   # peaks of the one-call workload that add_ms1 traces in two passes


@functools.lru_cache(maxsize=1)
def peptides() -> Peptides:
    return synth.make_peptides(20000, seed=PEPTIDES_SEED)


def _identity(n_files, max_rt=1.0):
    al = np.zeros(n_files, ALIGNMENT_DTYPE)
    al["max_rt"], al["slope"], al["intercept"] = max_rt, 1.0, 0.0
    return al


def _features(ids, rt, file_id, mono, ims=None, q=None):
    n = len(ids)
    return dict(peptide_idx=np.asarray(ids, np.uint32), peptide_q=np.zeros(n, f32) if q is None else np.asarray(q, f32), label=np.ones(n, np.int32),
                aligned_rt=np.asarray(rt, f32), calcmass=np.asarray(mono, f32), file_id=np.asarray(file_id, np.uint32),
                ims=np.zeros(n, f32) if ims is None else np.asarray(ims, f32))


def _batch(spectra, mobility=False, lead=0):
    """spectra: [(file, sst, masses, intensities, mobilities)] -> Ms1Batch; `lead` junk peaks before the first spectrum (peak_off[0] = lead)."""
    off = np.concatenate([[lead], lead + np.cumsum([len(s[2]) for s in spectra], dtype=np.int64)]).astype(np.uint64)
    junk = np.full(lead, 777.0, f32)
    cat = lambda i: np.concatenate([junk] + [np.asarray(s[i], f32) for s in spectra]) if spectra else junk   # noqa: E731
    return Ms1Batch(off, cat(2), cat(3), np.array([s[0] for s in spectra], np.uint32), np.array([s[1] for s in spectra], f32),
                    cat(4) if mobility else None)


def _spectra_from_ranges(ranges, srts, files, rng, keep=0.7, noise=4, mob_of=None):
    """One spectrum per (srt, file): a peak inside the mass window of a random `keep` of the ranges within RT_TOL (+10%) of srt, and noise.
    mob_of(range rows, rng) gives the peaks' mobilities (None: no mobilities)."""
    out = []
    for srt, f in zip(srts, files):
        near = ranges[np.abs(ranges["rt"].astype(np.float64) - float(srt)) <= 1.1 * float(RT_TOL)]
        near = near[rng.random(len(near)) < keep]
        u = rng.random(len(near)).astype(f32)
        m = np.concatenate([near["mass_lo"] + (near["mass_hi"] - near["mass_lo"]) * u, rng.uniform(300, 1500, noise).astype(f32)])
        i = rng.lognormal(10.0, 1.0, len(m)).astype(f32)
        mob = np.concatenate([mob_of(near, rng), rng.uniform(0.7, 1.3, noise).astype(f32)]) if mob_of else np.zeros(len(m), f32)
        out.append((f, srt, m, i, mob))
    return out


def _ulps_around(x, n=8):
    out, lo, hi = [x], x, x
    for _ in range(n):
        lo, hi = np.nextafter(lo, f32(-np.inf)), np.nextafter(hi, f32(np.inf))
        out += [lo, hi]
    return out


def _runs_case(settings=None, charges=(2, 3), runs_kw=None, **extra):
    pep = peptides()
    runs = synth.make_ms1_runs(pep, **runs_kw)
    c = dict(peptides=pep, settings=settings or LfqSettings(), charges=charges, features=runs["features"], alignments=runs["alignments"],
             batches=[runs["batch"]])
    c.update(extra)
    return c


# ---------------------------------------------------------------------------------------------------- the cases
def files(n_files):
    """~300 peptides in `n_files` files: k_lfq_integrate's shared memory passes 48 KB at 29 files; apply_time_warps gives one warp two files
    from 9 on."""
    spf, ppk = (80, 30) if n_files > 64 else (200, 60)
    return _runs_case(runs_kw=dict(n_ids=300, n_files=n_files, spectra_per_file=spf, peaks_per_spectrum=ppk, seed=100 + n_files, rt_range=(0.3, 0.5),
                                   scan_range=(0.29, 0.51), absent_fraction=0.3))


# k_ref: the reference file's own offset (its peak sits at bin 50 + k_ref); the other files' warps are offset - k_ref, clamped to +-75
_WARPS = {"early": (3, -35, [-1, 1, 31, 0, 74, 75, 80, 0]), "late": (5, 35, [-80, -75, -74, -31, -1, 0, 0, 1])}


def warps(kind):
    """8 files whose elution peaks are offset by whole grid bins, every file sampling the same aligned RTs one bin apart, so that
    find_time_warps has a single best shift per file; the reference file is not file 0. 'silent': the reference file has no signal, so every
    shift ties at a zero dot product and the last one, +75, wins."""
    ref, k_ref, w = _WARPS["early" if kind == "silent" else kind]
    offsets = [k_ref + x for x in w]
    expect = {f: int(np.clip(x, -75, 75)) for f, x in enumerate(w)} if kind != "silent" else {f: 75 for f in range(8)}
    return _runs_case(runs_kw=dict(n_ids=60, n_files=8, spectra_per_file=1200, peaks_per_spectrum=16, seed=200 + len(kind), rt_range=(0.45, 0.55),
                                   scan_range=(0.44, 0.56), rt_offset_bins=offsets, distort=False, ref_file=ref, absent_fraction=0.0, sigma=0.0004,
                                   silent_files=(ref,) if kind == "silent" else ()), warps=expect)


def charges(lo, hi, combine):
    """Charge ranges the other workloads do not use: (1, 1), and (1, 8) where the uncombined grid index is (slot * 8 + charge - 1) * 2 + decoy."""
    return _runs_case(settings=LfqSettings(combine_charge_states=combine), charges=(lo, hi),
                      runs_kw=dict(n_ids=300, n_files=2, spectra_per_file=200, peaks_per_spectrum=100, seed=300 + hi, charges=tuple(range(lo, hi + 1))))


def composition():
    """Identified peptides whose sequences hold U, O, the zero-composition letters B J X Z and bytes outside A-Z, plus 255-residue runs of O
    (3060 carbons), C and M (255 sulfurs): the ends of the expf tables. The table keeps the synthetic table's row count."""
    base = peptides()
    c = _runs_case(runs_kw=dict(n_ids=300, n_files=2, spectra_per_file=200, peaks_per_spectrum=100, seed=400))
    ids = np.unique(c["features"]["peptide_idx"][:300])
    special = [b"O" * 255, b"C" * 255, b"M" * 255, b"U" * 40, b"BJXZ" * 5, b"\x00\xff@[`{az", b"PEPTUOBK", b"UUOOCCMM", b"W" * 255, b"abcdef"]
    seqs = [bytes(base.seq[base.seq_off[i]:base.seq_off[i + 1]]) for i in range(len(base.mono))]
    for j, i in enumerate(ids[:len(special) * 3]):
        s = special[j % len(special)]
        seqs[i] = s if j < len(special) else (seqs[i][:3] + s[:10] + seqs[i][3:])
    off = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.uint32)
    seq = np.frombuffer(b"".join(seqs), np.uint8).copy()
    c["peptides"] = Peptides(seq_off=off, seq=seq, mods=np.zeros(len(seq), f32), nterm=base.nterm, mono=base.mono, decoy=base.decoy, missed=base.missed)
    return c


def pages():
    """A map of 4 pages: 4000 peptides at one aligned RT (24000 forward ranges at 0.5 and their 24000 decoys at 0.49, so pages share a
    min_rt), aligned RTs below 0.01 (decoys clamped to 0), negative RTs, -0.0 and +0.0; spectra at those RTs, at -0.0, and whose RT window
    ends (or starts) exactly on a page's min_rt."""
    pep = peptides()
    rng = np.random.default_rng(500)
    tg = rng.permutation(np.nonzero(pep.decoy == 0)[0])[:4404]
    rt = np.concatenate([np.full(4000, 0.5), rng.uniform(0.0, 0.01, 100), -rng.uniform(0.0001, 0.004, 50), [-0.0, 0.0, 0.01, 0.015],
                         rng.uniform(0.05, 0.95, 250)]).astype(f32)
    feats = _features(tg, rt, rng.integers(0, 2, len(tg)), pep.mono[tg])
    settings = LfqSettings()
    ranges, min_rts = build_map(settings, (2, 3), feats)
    srts = [f32(0.5), f32(0.4995), f32(0.49), f32(0.4932), f32(-0.0), f32(0.0), f32(0.002), f32(-0.002), f32(0.006), f32(0.011)]
    srts += list(rng.choice(rt[-250:], 40))
    for m in min_rts:   # spectra whose window ends exactly on a min_rt (rt + RT_TOL == m) or starts on it (rt - RT_TOL == m)
        for start, hits in ((f32(m - RT_TOL), lambda y: f32(y + RT_TOL) == m), (f32(m + RT_TOL), lambda y: f32(y - RT_TOL) == m)):
            found = [y for y in _ulps_around(start) if hits(y)]
            assert found, m
            srts.append(found[0])
    srts = np.array(srts, f32)
    sp = _spectra_from_ranges(ranges, srts, rng.integers(0, 2, len(srts)), rng, keep=0.5)
    return dict(peptides=pep, settings=settings, charges=(2, 3), features=feats, alignments=_identity(2), batches=[_batch(sp)], n_pages=len(min_rts))


def mobility(kind):
    """Peaks whose mobility is exactly a range's mobility_lo or mobility_hi (both bounds are inclusive) or the next float outside;
    'zero_tol': mobility_pct_tolerance 0, so only the identified ims itself matches; 'mixed': batches with and without mobilities on one map."""
    pep = peptides()
    rng = np.random.default_rng(600 + len(kind))
    tg = rng.permutation(np.nonzero(pep.decoy == 0)[0])[:300]
    rt = rng.uniform(0.05, 0.95, 300).astype(f32)
    ims = rng.uniform(0.7, 1.3, 300).astype(f32)
    ims[:5] = 0.0
    feats = _features(tg, rt, rng.integers(0, 3, 300), pep.mono[tg], ims=ims)
    settings = LfqSettings(mobility_pct_tolerance=0.0 if kind == "zero_tol" else 1.0, spectral_angle=0.0)
    ranges, _ = build_map(settings, (2, 3), feats)

    def mob_of(near, r):
        choice = r.integers(0, 5, len(near))
        lo, hi = near["mobility_lo"], near["mobility_hi"]
        opts = np.stack([lo, hi, np.nextafter(lo, f32(-np.inf)), np.nextafter(hi, f32(np.inf)), (lo + hi) / f32(2)])
        return opts[choice, np.arange(len(near))]
    srts = np.concatenate([rt + rng.uniform(-0.004, 0.004, 300).astype(f32) for _ in range(3)])
    files = rng.integers(0, 3, len(srts))
    sp = _spectra_from_ranges(ranges, srts, files, rng, mob_of=mob_of)
    if kind == "mixed":
        batches = [_batch(sp[0::3], mobility=True), _batch(sp[1::3], mobility=False), _batch(sp[2::3], mobility=True)]
    else:
        batches = [_batch(sp, mobility=True)]
    return dict(peptides=pep, settings=settings, charges=(2, 3), features=feats, alignments=_identity(3), batches=batches)


def degenerate(kind):
    """'input': an empty batch; a batch of zero-peak spectra only; zero-peak spectra between others; zero, negative and subnormal intensities;
    a NaN scan_start_time; a file whose alignment has max_rt 0; a batch whose peak_off starts past 0. 'no_kept': no feature passes the q-value
    cut, so the map has no ranges, pages or grids."""
    pep = peptides()
    rng = np.random.default_rng(700)
    tg = rng.permutation(np.nonzero(pep.decoy == 0)[0])[:200]
    rt = rng.uniform(0.05, 0.95, 200).astype(f32)
    feats = _features(tg, rt, rng.integers(0, 2, 200), pep.mono[tg], q=np.full(200, 0.5) if kind == "no_kept" else None)
    settings = LfqSettings(spectral_angle=0.0)
    ranges, _ = build_map(LfqSettings(peptide_q_value=1.0), (2, 3), feats)
    al = _identity(3)
    al["max_rt"][2] = 0.0
    srts = np.concatenate([rt + rng.uniform(-0.004, 0.004, 200).astype(f32) for _ in range(2)])
    sp = _spectra_from_ranges(ranges, srts, rng.integers(0, 2, len(srts)), rng)
    special = np.array([0.0, -0.0, -1234.5, 1e-40, -1e-42, 1e-45], f32)   # the signal peaks come first in each spectrum
    for k, s in enumerate(sp):
        m = min(len(s[3]), len(special))
        s[3][:m] = np.roll(special, k)[:m]
    empty = lambda f, t: (f, f32(t), np.zeros(0, f32), np.zeros(0, f32), np.zeros(0, f32))   # noqa: E731
    mid = sp[:40] + [empty(0, 0.5), empty(1, 0.3)] + sp[40:80]
    nan = [(s[0], f32(np.nan), s[2], s[3], s[4]) for s in sp[80:84]]
    file2 = [(2, s[1], s[2], s[3], s[4]) for s in sp[84:88]] + [(2, f32(0.0), sp[88][2], sp[88][3], sp[88][4])]
    batches = [_batch([]), _batch([empty(0, 0.2), empty(1, 0.4), empty(0, 0.6)]), _batch(mid), _batch(nan + file2), _batch(sp[88:], lead=7)]
    return dict(peptides=pep, settings=settings, charges=(2, 3), features=feats, alignments=al, batches=batches)


def big(kind):
    """'batch': one add_ms1 of BIG peaks (ordinary spectra padded with peaks below every mass window), traced in two passes, the second one
    starting at a non-zero peak offset. 'spectrum': one spectrum of 2^24 + 1 peaks between ordinary ones, a pass on its own."""
    c = _runs_case(runs_kw=dict(n_ids=300, n_files=2, spectra_per_file=300, peaks_per_spectrum=200, seed=800))
    b = c["batches"][0]
    n = len(b)
    counts = np.diff(b.peak_off.astype(np.int64))
    if kind == "batch":
        pad = np.full(n, (BIG - int(counts.sum())) // n, np.int64)
        pad[: (BIG - int(counts.sum())) % n] += 1
    else:
        pad = np.zeros(n, np.int64)
        pad[n // 2] = (1 << 24) + 1 - counts[n // 2]
    new = counts + pad
    off = np.concatenate([[0], np.cumsum(new)]).astype(np.uint64)
    masses = np.full(int(off[-1]), 50.0, f32)
    inten = np.full(int(off[-1]), 3.0, f32)
    dst = np.repeat(off[:-1].astype(np.int64), counts) + (np.arange(int(counts.sum())) - np.repeat(np.cumsum(counts) - counts, counts))
    masses[dst] = b.masses
    inten[dst] = b.intensities
    c["batches"] = [Ms1Batch(off, masses, inten, b.file_id, b.scan_start_time)]
    return c


def seed_runs(seed):
    """The synthetic workloads of tests/test_gpu_lfq.py, by seed."""
    kw = dict(n_ids=1500, n_files=3, spectra_per_file=200, peaks_per_spectrum=300)
    kw = {7: dict(kw, seed=7), 8: dict(kw, seed=8, mobility=True), 11: dict(kw, n_files=2, seed=11),
          13: dict(n_ids=1200, n_files=3, spectra_per_file=250, peaks_per_spectrum=300, seed=13, absent_fraction=0.4)}[seed]
    return synth.make_ms1_runs(peptides(), **kw)


_BUILDERS = {
    "files1": lambda: files(1), "files9": lambda: files(9), "files29": lambda: files(29), "files128": lambda: files(128),
    "warps_early_ref": lambda: warps("early"), "warps_late_ref": lambda: warps("late"), "warps_silent_ref": lambda: warps("silent"),
    "charges_1_1": lambda: charges(1, 1, False), "charges_1_8": lambda: charges(1, 8, False), "charges_1_8_combined": lambda: charges(1, 8, True),
    "composition": composition, "pages": pages,
    "mobility_bounds": lambda: mobility("bounds"), "mobility_zero_tol": lambda: mobility("zero_tol"), "mobility_mixed": lambda: mobility("mixed"),
    "degenerate_input": lambda: degenerate("input"), "no_kept_feature": lambda: degenerate("no_kept"),
    "big_batch": lambda: big("batch"), "big_spectrum": lambda: big("spectrum"),
}
NAMES = list(_BUILDERS)
HEAVY = ("big_batch", "big_spectrum")


@functools.lru_cache(maxsize=4)
def case(name: str) -> dict:
    return _BUILDERS[name]()
