"""Edge workloads of the search-and-score path, shared by tests/test_search_reference.py (restatement == oracle) and
tests/test_gpu_search_reference.py (device == restatement == oracle).

Each workload is a seeded function returning (peptides, db kwargs, spectra, scorer kwargs). Small enough that the numpy restatement
(tests/search_reference.py) takes seconds: at most a few hundred spectra and tens of thousands of peptides."""
from __future__ import annotations

import numpy as np

from sage_b200 import Peptides, SpectraBatch, Tolerance, synth

import search_reference as R

F32 = np.float32
H2O = F32(18.010565)
AA = np.frombuffer(b"ACDEFGHIKLMNPQRSTVWY", np.uint8)


# ------------------------------------------------------------------------------------------------ builders
def peptides(seqs, mono=None, mods=None, decoy=None, check=True):
    """A peptide table from sequences; `mono` defaults to H2O + the residues (sequential f32). Rows must be in ascending mass."""
    seqs = [s if isinstance(s, bytes) else s.encode() for s in seqs]
    lens = np.array([len(s) for s in seqs], np.int64)
    seq = np.frombuffer(b"".join(seqs), np.uint8).copy()
    m = np.zeros(len(seq), np.float32) if mods is None else np.asarray(mods, np.float32)
    if mono is None:
        mono = np.empty(len(seqs), np.float32)
        off = 0
        for i, L in enumerate(lens):
            acc = H2O
            for r, x in zip(R.residue_mass(seq[off:off + L]), m[off:off + L]):
                acc = (acc + r) + x
            mono[i] = acc
            off += L
    mono = np.asarray(mono, np.float32)
    assert not check or np.all(R.f32_key(mono)[1:] >= R.f32_key(mono)[:-1]), "peptide rows must be in ascending mass"
    return Peptides(seq_off=np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32), seq=seq, mods=m,
                    nterm=np.full(len(seqs), np.nan, np.float32), mono=mono,
                    decoy=np.zeros(len(seqs), np.uint8) if decoy is None else np.asarray(decoy, np.uint8),
                    missed=(lens % 3).astype(np.uint8))


def spectra(peaks, prec_mz, charge=2, iso=(np.nan, np.nan), tic=None):
    """peaks: list of (masses, intensities); scalar or per-spectrum prec_mz / charge / isolation window / TIC (None: sequential sum)."""
    n = len(peaks)
    off = np.concatenate([[0], np.cumsum([len(m) for m, _ in peaks])]).astype(np.uint64)
    masses = np.concatenate([np.asarray(m, np.float32) for m, _ in peaks]) if off[-1] else np.zeros(0, np.float32)
    intens = np.concatenate([np.asarray(i, np.float32) for _, i in peaks]) if off[-1] else np.zeros(0, np.float32)
    if tic is None:
        tic = []
        for _, it in peaks:
            acc = F32(0.0)
            for x in np.asarray(it, np.float32):
                acc = acc + x
            tic.append(acc)
    full = lambda x, dt: np.broadcast_to(np.asarray(x, dt), (n,)).copy()  # noqa: E731
    iso = np.asarray(iso, np.float32)
    ilo = full(iso[..., 0] if iso.ndim == 2 else iso[0], np.float32)
    ihi = full(iso[..., 1] if iso.ndim == 2 else iso[1], np.float32)
    return SpectraBatch(peak_off=off, masses=masses, intensities=intens, prec_mz=full(prec_mz, np.float32), prec_charge=full(charge, np.uint8),
                        iso_lo=ilo, iso_hi=ihi, tic=full(tic, np.float32), level=np.full(n, 2, np.uint8), rt=np.zeros(n, np.float32),
                        ims=np.full(n, np.nan, np.float32))


def ions_of(pep, i, kinds=("b", "y")):
    """Every ion of peptide i, per kind (ion_series.rs)."""
    sub = Peptides(seq_off=np.array([0, pep.seq_off[i + 1] - pep.seq_off[i]], np.uint32), seq=pep.seq[pep.seq_off[i]:pep.seq_off[i + 1]],
                   mods=pep.mods[pep.seq_off[i]:pep.seq_off[i + 1]], nterm=pep.nterm[i:i + 1], mono=pep.mono[i:i + 1], decoy=pep.decoy[i:i + 1],
                   missed=pep.missed[i:i + 1])
    tabs = R.ion_tables(sub, [R.KINDS[k] for k in kinds])
    return {k: tabs[R.KINDS[k]][0] for k in kinds}


def prec_mz_for(mass, z):
    """An f32 precursor m/z whose (mz - PROTON) * z is within an ulp or two of `mass`."""
    return F32(F32(mass) / F32(z) + R.PROTON)


def random_seqs(rng, n, lo=7, hi=16):
    return [bytes(rng.choice(AA, int(rng.integers(lo, hi + 1)))) for _ in range(n)]


def synth_spectra(pep, n, seed, n_peaks=60, charge_known=True):
    return synth.make_spectra(pep, n, seed=seed, n_peaks=n_peaks, charge_known=charge_known)


NARROW = dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20))
DB = dict(bucket_size=8192, ion_kinds=("b", "y"), min_ion_index=2)


# ------------------------------------------------------------------------------------------------ ties and order
def isobaric_isomers():
    pep = synth.make_peptides(300, seed=11, var_mods=(("M", 15.9949), ("STY", 79.9663)), max_variable_mods=2)
    return pep, DB, synth_spectra(pep, 80, 12), dict(NARROW, report_psms=5, min_matched_peaks=1)


def _isotope(report):
    pep = synth.make_peptides(1500, seed=21)
    sp = synth_spectra(pep, 60, 22)
    # +-3 ppm windows hold 1-2 peptides at some isotopes and none at others; +-0.3 Da windows hold many
    tol = Tolerance.ppm(-3, 3) if report != 64 else Tolerance.da(-0.3, 0.3)
    return pep, DB, sp, dict(precursor_tol=tol, fragment_tol=Tolerance.ppm(-20, 20), min_isotope_err=-1, max_isotope_err=3, report_psms=report,
                             min_matched_peaks=1)


def isotope_defaults_r1():
    return _isotope(1)


def isotope_defaults_r5():
    return _isotope(5)


def isotope_defaults_r64():
    return _isotope(64)


def two_charges_unknown():
    pep = synth.make_peptides(1500, seed=31)
    sp = synth_spectra(pep, 60, 32, charge_known=False)
    return pep, DB, sp, dict(precursor_tol=Tolerance.da(-3, 3), fragment_tol=Tolerance.ppm(-20, 20), min_precursor_charge=2, max_precursor_charge=4,
                             report_psms=5, min_matched_peaks=1)


def two_charges_override():
    pep, db, sp, cfg = two_charges_unknown()
    sp.prec_charge[:] = 3
    return pep, db, sp, dict(cfg, override_precursor_charge=True, min_isotope_err=0, max_isotope_err=1)


def wide_window_isolation():
    pep = synth.make_peptides(1500, seed=41)
    sp = synth_spectra(pep, 60, 42)
    sp.iso_lo[:] = -1.5
    sp.iso_hi[:] = 1.5
    return pep, DB, sp, dict(NARROW, wide_window=True, min_precursor_charge=2, max_precursor_charge=3, report_psms=3, min_matched_peaks=1)


def wide_window_nan_isolation():
    pep, db, sp, cfg = wide_window_isolation()
    sp.iso_lo[::2] = np.nan   # one NaN bound is None: Da(-2.4, 2.4) times the charge
    sp.iso_hi[1::4] = np.nan
    return pep, db, sp, cfg


def equal_intensities():
    """Several peaks of equal intensity inside one fragment window (the last wins), zero-intensity peaks (selectable) and
    negative ones (never selected)."""
    rng = np.random.default_rng(51)
    pep = synth.make_peptides(800, seed=52)
    peaks, pmz = [], []
    for t in rng.choice(len(pep.mono), 40, replace=False):
        ions = ions_of(pep, t)
        m, it = [], []
        for k, arr in ions.items():
            for j, x in enumerate(arr):
                w = float(rng.choice([1000.0, 0.0, 5.0]))
                for d in (-4e-6, 0.0, 4e-6):
                    m.append(x * (1 + d))
                    it.append(w if d != 4e-6 or j % 3 else -w)
        o = np.argsort(np.asarray(m, np.float32), kind="stable")
        peaks.append((np.asarray(m, np.float32)[o], np.asarray(it, np.float32)[o]))
        pmz.append(prec_mz_for(pep.mono[t], 2))
    return pep, DB, spectra(peaks, pmz, 2), dict(NARROW, report_psms=3, min_matched_peaks=0)


def ion_index_zero_two_charges():
    """min_ion_index 0 (b1 / y1 are indexed), charge-3 precursors so every ion is looked up at fragment charges 1 and 2, and spectra
    that hold ion index 0 and both charges of the same ion (Run ignores index 0 and repeated indices)."""
    pep = synth.make_peptides(800, seed=61)
    rng = np.random.default_rng(62)
    peaks, pmz = [], []
    for t in rng.choice(len(pep.mono), 40, replace=False):
        ions = ions_of(pep, t)
        m = []
        for arr in ions.values():
            m += list(arr[: max(3, len(arr) // 2)])
            m += [x / F32(2) for x in arr[:4]]
        m = np.sort(np.asarray(m, np.float32))
        peaks.append((m, rng.lognormal(6, 1, len(m)).astype(np.float32)))
        pmz.append(prec_mz_for(pep.mono[t], 3))
    return pep, dict(DB, min_ion_index=0), spectra(peaks, pmz, 3), dict(NARROW, report_psms=4, min_matched_peaks=0)


def duplicate_peaks():
    """Every peak twice, equal in mass and intensity: the chimera loop removes every peak equal to a removed (mass, intensity) pair."""
    pep = synth.make_peptides(800, seed=75)
    peaks, pmz = _target_spectra(pep, 24, 76)
    rng = np.random.default_rng(77)
    out = []
    for m, it in peaks:
        noise = np.sort(rng.uniform(150, 1500, 30).astype(np.float32))
        mm = np.concatenate([m, m, noise])
        ii = np.concatenate([it, it, rng.lognormal(5, 1, 30).astype(np.float32)])
        o = np.argsort(mm, kind="stable")
        out.append((mm[o], ii[o]))
    return pep, DB, spectra(out, pmz, 3), dict(precursor_tol=Tolerance.da(-2, 2), fragment_tol=Tolerance.ppm(-20, 20), report_psms=3,
                                             min_matched_peaks=1)


def more_candidates_than_reported():
    pep = synth.make_peptides(2000, seed=71)
    return pep, DB, synth_spectra(pep, 60, 72, n_peaks=150), dict(precursor_tol=Tolerance.da(-1, 1), fragment_tol=Tolerance.ppm(-20, 20),
                                                                   report_psms=2, min_matched_peaks=0)


# ------------------------------------------------------------------------------------------------ numeric edges
def _target_spectra(pep, n, seed, scale=None, z=2):
    rng = np.random.default_rng(seed)
    peaks, pmz = [], []
    for t in rng.choice(len(pep.mono), n, replace=False):
        m = np.sort(np.concatenate(list(ions_of(pep, t).values())).astype(np.float32))
        it = rng.lognormal(6, 1, len(m)).astype(np.float32) if scale is None else np.full(len(m), scale, np.float32)
        peaks.append((m, it))
        pmz.append(prec_mz_for(pep.mono[t], z))
    return peaks, pmz


def _fmax(score_type):
    pep = synth.make_peptides(600, seed=81)
    peaks, pmz = _target_spectra(pep, 20, 82, scale=F32(3.0e38))
    return pep, DB, spectra(peaks, pmz, 2), dict(NARROW, report_psms=3, min_matched_peaks=0, score_type=score_type)


def fmax_intensity_sage():
    return _fmax(0)


def fmax_intensity_openms():
    return _fmax(1)


def zero_intensity_matches():
    pep = synth.make_peptides(600, seed=91)
    peaks, pmz = _target_spectra(pep, 20, 92, scale=F32(0.0))
    return pep, DB, spectra(peaks, pmz, 2), dict(NARROW, report_psms=2, min_matched_peaks=0)


def tic_zero():
    pep = synth.make_peptides(600, seed=101)
    peaks, pmz = _target_spectra(pep, 20, 102)
    return pep, DB, spectra(peaks, pmz, 2, tic=0.0), dict(NARROW, report_psms=2, min_matched_peaks=1)


def _asym(ptol, ftol):
    pep = synth.make_peptides(1500, seed=111)
    return pep, DB, synth_spectra(pep, 40, 112), dict(precursor_tol=ptol, fragment_tol=ftol, report_psms=3, min_matched_peaks=0)


def asymmetric_da():
    return _asym(Tolerance.da(-0.05, 2.0), Tolerance.da(0.01, 0.05))


def asymmetric_ppm():
    return _asym(Tolerance.ppm(0.0, 40.0), Tolerance.ppm(-30.0, 0.0))


def asymmetric_pct():
    return _asym(Tolerance.pct(-0.001, 0.01), Tolerance.pct(0.0, 0.002))


def one_sided_positive():
    return _asym(Tolerance.ppm(5.0, 60.0), Tolerance.ppm(2.0, 25.0))


def window_bounds():
    """Peptide masses exactly on a window bound, runs of equal masses across a bound, windows below and above every peptide
    (pre_idx_hi == n_peptides)."""
    rng = np.random.default_rng(121)
    seqs = random_seqs(rng, 400)
    base = np.sort(rng.uniform(800, 1600, 400)).astype(np.float32)
    base[100:110] = base[100]          # a run of equal masses
    base[300:305] = base[300]
    pep = peptides(seqs, mono=base)
    peaks, pmz, chg = [], [], []
    tol = Tolerance.da(-0.5, 0.5)
    for t in list(range(95, 115)) + list(range(295, 310)) + [0, 399]:
        ions = np.sort(np.concatenate(list(ions_of(pep, t).values()))).astype(np.float32)
        peaks.append((ions, np.full(len(ions), 100.0, np.float32)))
        # the window's upper (or lower) bound lands exactly on the peptide mass: center = mono - 0.5 in f32
        pmz.append(F32(F32(base[t] - F32(0.5 if t % 2 else -0.5)) / F32(1.0) + R.PROTON))
        chg.append(1)
    for m in (F32(100.0), F32(1e5)):   # below and above every peptide
        peaks.append((np.array([200.0, 300.0], np.float32), np.array([5.0, 6.0], np.float32)))
        pmz.append(m)
        chg.append(1)
    return pep, DB, spectra(peaks, pmz, chg), dict(precursor_tol=tol, fragment_tol=Tolerance.da(-0.02, 0.02), min_precursor_charge=1,
                                                 max_precursor_charge=3, report_psms=3, min_matched_peaks=0)


def odd_peaks():
    """Peaks at +0.0 and -0.0, negative masses, NaN masses and intensities, and unsorted spectra."""
    pep = synth.make_peptides(800, seed=131)
    peaks, pmz = _target_spectra(pep, 24, 132)
    rng = np.random.default_rng(133)
    out = []
    for i, (m, it) in enumerate(peaks):
        m, it = m.copy(), it.copy()
        extra_m = np.array([0.0, -0.0, -5.0, np.nan, m[len(m) // 2]], np.float32)
        extra_i = np.array([7.0, 8.0, 9.0, 10.0, np.nan], np.float32)
        m, it = np.concatenate([extra_m[:2], m, extra_m[2:]]), np.concatenate([extra_i[:2], it, extra_i[2:]])
        if i % 3 == 0:
            o = rng.permutation(len(m))   # unsorted: the binary search then depends on its probe order
            m, it = m[o], it[o]
        out.append((m, it))
    return pep, DB, spectra(out, pmz, 2), dict(NARROW, report_psms=2, min_matched_peaks=0)


# ------------------------------------------------------------------------------------------------ kernel boundaries
STEP = F32(2.0 ** -7)


def even_masses(n, start=1000.0):
    return (F32(start) + np.arange(n, dtype=np.float32) * STEP).astype(np.float32)


def _even_db(n, seed, lo=6, hi=10, residues=b"GAS"):
    """n peptides of evenly spaced masses. Light residues keep every ion of every kind above 0 m/z (mono is ~1000, residues sum < 900)."""
    rng = np.random.default_rng(seed)
    aa = np.frombuffer(residues, np.uint8)
    return peptides([bytes(rng.choice(aa, int(rng.integers(lo, hi + 1)))) for _ in range(n)], mono=even_masses(n))


def window_spectra(pep, first, count, seed, n_peaks=40):
    """One spectrum per window start: the precursor sits on the middle peptide of [first, first + count), and the Da tolerance
    returned puts both bounds half a step outside that range. Peaks: the ions of a random peptide of the window plus noise."""
    rng = np.random.default_rng(seed)
    mono = pep.mono
    peaks, pmz = [], []
    for f in first:
        t = f + int(rng.integers(count))
        ions = np.concatenate(list(ions_of(pep, t).values())).astype(np.float32)
        m = np.sort(np.concatenate([ions, rng.uniform(100, 1200, n_peaks).astype(np.float32)]))
        peaks.append((m, rng.lognormal(6, 1, len(m)).astype(np.float32)))
        pmz.append(F32(mono[f + count // 2] + R.PROTON))
    lo = -(count // 2) * float(STEP) - float(STEP) / 2
    hi = (count - 1 - count // 2) * float(STEP) + float(STEP) / 2
    return spectra(peaks, pmz, 1), Tolerance.da(lo, hi)


def _window_workload(count, first, n_pep, seed, report_psms=3, residues=b"GAS"):
    pep = _even_db(n_pep, seed, residues=residues, **(dict(lo=7, hi=12) if residues != b"GAS" else {}))
    sp, tol = window_spectra(pep, first, count, seed + 2)
    return pep, dict(DB, bucket_size=2048), sp, dict(precursor_tol=tol, fragment_tol=Tolerance.ppm(-20, 20), report_psms=report_psms,
                                                     min_matched_peaks=1, min_precursor_charge=1, max_precursor_charge=1)


def _cap(count):
    def f():
        # count - 2 peptides inside the bounds: binary_search_slice adds the one below and the one above, pre_idx_hi - pre_idx_lo + 1 == count
        rng = np.random.default_rng(count)
        return _window_workload(count - 2, [int(x) for x in rng.integers(1, 12000 - count, 6)], 12000, 1000 + count)
    f.__name__ = f"window_{count}"
    return f


window_1024, window_1025, window_8192, window_8193 = (_cap(c) for c in (1024, 1025, 8192, 8193))


def block_boundaries():
    """Windows of 300 peptides that start on, or end just before, a multiple of 256 (run with narrow_block 256 on the device)."""
    return _window_workload(300, [256 * 7, 256 * 9 - 300, 256 * 20, 256 * 31 - 300], 14000, 141, report_psms=2)


def block_boundaries_wide():
    """Open-search windows of 9000 peptides that start on, or end just before, a multiple of 4096 (wide_tile 4096 on the device)."""
    return _window_workload(9000, [4096, 4096 * 3 - 9000, 4096 * 2], 20000, 143, report_psms=2)


def negative_fragment_mz():
    """Open-search windows over a table whose masses (~1000) are below the residue sums of its sequences: many y / x / z ions have
    negative m/z, which the index sorts by total_cmp like any other value."""
    return _window_workload(9000, [4096, 4096 * 3 - 9000, 4096 * 2], 20000, 145, report_psms=2, residues=AA.tobytes())


def report_psms_64():
    pep = synth.make_peptides(3000, seed=151)
    return pep, DB, synth_spectra(pep, 24, 152), dict(precursor_tol=Tolerance.da(-5, 5), fragment_tol=Tolerance.ppm(-20, 20), report_psms=64,
                                                      min_matched_peaks=0)


def isotope_range_32():
    pep = synth.make_peptides(800, seed=161)
    return pep, DB, synth_spectra(pep, 12, 162), dict(NARROW, min_isotope_err=-16, max_isotope_err=15, report_psms=2, min_matched_peaks=1)


def charge_range_16():
    pep = synth.make_peptides(800, seed=171)
    sp = synth_spectra(pep, 8, 172, n_peaks=30, charge_known=False)
    return pep, DB, sp, dict(NARROW, min_precursor_charge=1, max_precursor_charge=16, max_fragment_charge=2, report_psms=2, min_matched_peaks=1)


def peptide_lengths():
    """Peptides of length 1, 2, 3 and 255 (a 1-residue peptide has no ions)."""
    rng = np.random.default_rng(181)
    seqs = [b"G", b"AK", b"PEK"] + random_seqs(rng, 40, 5, 20) + [bytes(rng.choice(AA, 255))]
    tmp = peptides(seqs, check=False)
    o = np.argsort(tmp.mono, kind="stable")
    pep = peptides([seqs[i] for i in o])
    peaks, pmz = [], []
    for t in range(len(seqs)):
        ions = np.concatenate([np.zeros(0, np.float32)] + list(ions_of(pep, t).values())).astype(np.float32)
        m = np.sort(np.concatenate([ions, np.array([57.0, 128.0], np.float32)]))
        peaks.append((m, rng.lognormal(6, 1, len(m)).astype(np.float32)))
        pmz.append(prec_mz_for(pep.mono[t], 1))
    return pep, dict(DB, min_ion_index=0), spectra(peaks, pmz, 1), dict(precursor_tol=Tolerance.da(-1, 1), fragment_tol=Tolerance.ppm(-20, 20),
                                                                        report_psms=2, min_matched_peaks=0, min_precursor_charge=1,
                                                                        max_precursor_charge=2)


def single_peptide_db():
    pep = peptides([b"PEPTIDEK"])
    ions = np.sort(np.concatenate(list(ions_of(pep, 0).values()))).astype(np.float32)
    sp = spectra([(ions, np.full(len(ions), 10.0, np.float32)), (ions[:2], np.ones(2, np.float32))], prec_mz_for(pep.mono[0], 2), 2)
    return pep, dict(DB, min_ion_index=0), sp, dict(NARROW, report_psms=3, min_matched_peaks=0)


def fragment_charges_1_to_8():
    pep = synth.make_peptides(800, seed=191)
    rng = np.random.default_rng(192)
    peaks, pmz, chg = [], [], []
    for j, t in enumerate(rng.choice(len(pep.mono), 16, replace=False)):
        z = 2 + j % 8   # precursor charges 2..9: fragment charges up to 8
        ions = np.concatenate(list(ions_of(pep, t).values()))
        m = np.sort(np.concatenate([ions / F32(1 + (i % z)) for i in range(2)] + [ions / F32(max(1, z - 1))]).astype(np.float32))
        peaks.append((m, rng.lognormal(6, 1, len(m)).astype(np.float32)))
        pmz.append(prec_mz_for(pep.mono[t], z))
        chg.append(z)
    return pep, DB, spectra(peaks, pmz, chg), dict(NARROW, report_psms=2, min_matched_peaks=1)


def peak_counts_0_1():
    pep = synth.make_peptides(600, seed=201)
    t = 17
    ions = np.sort(np.concatenate(list(ions_of(pep, t).values()))).astype(np.float32)
    pm = prec_mz_for(pep.mono[t], 2)
    sp = spectra([(np.zeros(0, np.float32), np.zeros(0, np.float32)), (ions[3:4], np.ones(1, np.float32)), (ions, np.ones(len(ions), np.float32))],
                 pm, 2)
    return pep, DB, sp, dict(NARROW, report_psms=2, min_matched_peaks=0)


def many_peaks(n_peaks):
    """One spectrum of `n_peaks` peaks (the shared-memory budget of k_score is found on the device)."""
    pep = synth.make_peptides(600, seed=211)
    rng = np.random.default_rng(212)
    t = 33
    ions = np.concatenate(list(ions_of(pep, t).values())).astype(np.float32)
    m = np.sort(np.concatenate([ions, rng.uniform(100, 3000, max(0, n_peaks - len(ions))).astype(np.float32)])[:n_peaks])
    sp = spectra([(m, rng.lognormal(6, 1, len(m)).astype(np.float32))], prec_mz_for(pep.mono[t], 2), 2)
    return pep, DB, sp, dict(NARROW, report_psms=2, min_matched_peaks=1)


def one_lut_cell():
    """All peaks inside one spectrum-LUT cell (a 0.01 Th cluster), and peaks spread over 1e-3 .. 1e6 Th."""
    pep = synth.make_peptides(600, seed=221)
    rng = np.random.default_rng(222)
    peaks, pmz = [], []
    for j, t in enumerate(rng.choice(len(pep.mono), 12, replace=False)):
        ions = np.concatenate(list(ions_of(pep, t).values())).astype(np.float32)
        if j % 2 == 0:
            x = ions[len(ions) // 2]
            m = np.sort((x + rng.uniform(-0.005, 0.005, 50)).astype(np.float32))
        else:
            m = np.sort(np.concatenate([ions, (10.0 ** rng.uniform(-3, 6, 80)).astype(np.float32)]))
        peaks.append((m, rng.lognormal(6, 1, len(m)).astype(np.float32)))
        pmz.append(prec_mz_for(pep.mono[t], 2))
    return pep, DB, spectra(peaks, pmz, 2), dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.da(-0.02, 0.02), report_psms=2,
                                                 min_matched_peaks=0)


# ------------------------------------------------------------------------------------------------ count overflow
def _overflow(n_fill):
    """One (query, peptide) pair whose preliminary count passes 65 536: a 255-residue peptide on an even slot of a window of
    `n_fill` + 1 peptides of length 2, with a fragment tolerance wider than the fragment range, so every peak matches every indexed
    fragment of the window. Its odd neighbour matches too. Precursor charge 2: one fragment charge."""
    rng = np.random.default_rng(231 + n_fill)
    big = bytes(rng.choice(AA, 255))
    fill = [bytes(rng.choice(AA, 2)) for _ in range(n_fill)]
    M = F32(28000.0)
    half = n_fill // 2
    half -= 1 - half % 2    # odd: pre_idx_lo is the last of the three leading peptides, so the big peptide's slot (half + 1) is even
    mono = np.concatenate([M - F32(0.5) + np.arange(half, dtype=np.float32) * F32(2.0 ** -12), [M],
                           M + F32(0.01) + np.arange(n_fill - half, dtype=np.float32) * F32(2.0 ** -12)]).astype(np.float32)
    seqs = fill[:half] + [big] + fill[half:]
    lead = [b"GG"] * 3
    lead_mono = np.array([500.0, 600.0, 700.0], np.float32)
    pep = peptides(lead + seqs, mono=np.concatenate([lead_mono, mono]))
    n_peaks = 140
    m = np.sort(rng.uniform(200, 2000, n_peaks).astype(np.float32))
    sp = spectra([(m, rng.lognormal(6, 1, n_peaks).astype(np.float32))], prec_mz_for(M, 2), 2)
    cfg = dict(precursor_tol=Tolerance.da(-0.6, 0.6), fragment_tol=Tolerance.da(-40000.0, 40000.0), report_psms=3, min_matched_peaks=0)
    return pep, dict(DB, min_ion_index=0), sp, cfg


def overflow_warp():
    return _overflow(500)


def overflow_narrow():
    return _overflow(2000)


WORKLOADS = [isobaric_isomers, isotope_defaults_r1, isotope_defaults_r5, isotope_defaults_r64, two_charges_unknown, two_charges_override,
             wide_window_isolation, wide_window_nan_isolation, equal_intensities, ion_index_zero_two_charges, duplicate_peaks, more_candidates_than_reported,
             fmax_intensity_sage, fmax_intensity_openms, zero_intensity_matches, tic_zero, asymmetric_da, asymmetric_ppm, asymmetric_pct,
             one_sided_positive, window_bounds, odd_peaks, window_1024, window_1025, window_8192, window_8193, block_boundaries,
             block_boundaries_wide, negative_fragment_mz, report_psms_64, isotope_range_32, charge_range_16, peptide_lengths, single_peptide_db, fragment_charges_1_to_8,
             peak_counts_0_1, one_lut_cell, overflow_warp, overflow_narrow]
BY_NAME = {f.__name__: f for f in WORKLOADS}
# workloads whose row count is reported and must not be zero


def potentials(pep, db_kw, sp, cfg):
    """pre_idx_hi - pre_idx_lo + 1 of every spectrum's first query: the dense window the counting kernels are chosen by."""
    db = R.build_from_peptides(pep, **db_kw)
    ptol = R.Tol.of(cfg["precursor_tol"])
    out = []
    for s in R.spectra_from_batch(sp):
        z = s.charge if s.charge is not None else cfg.get("min_precursor_charge", 2)
        q = R.db_query(db, (s.prec_mz - R.PROTON) * F32(z), ptol, R.Tol.of(cfg["fragment_tol"]))
        out.append(q.pre_idx_hi - q.pre_idx_lo + 1)
    return out


COUNTED = {"overflow_warp", "overflow_narrow", "window_1024", "window_1025", "window_8192", "window_8193", "report_psms_64", "peptide_lengths"}


# ------------------------------------------------------------------------------------------------ comparison
def restated(pep, db_kw, sp, cfg, counters=False):
    """(features[n * report_psms] FEATURE_DTYPE, counts[n], fragments rows, counters) from the restatement, laid out like score_batch."""
    from oracle.oracle import FEATURE_DTYPE, FRAGMENT_DTYPE
    db = R.build_from_peptides(pep, **db_kw)
    rows, frags, ctr = R.score_batch(db, cfg, sp, counters=counters)
    k = int(cfg.get("report_psms", 1))
    out = np.zeros(len(rows) * k, FEATURE_DTYPE)
    counts = np.array([len(r) for r in rows], np.uint32)
    frag_rows = []
    for i, rs in enumerate(rows):
        for j, r in enumerate(rs):
            o = out[i * k + j]
            o["spectrum"] = i
            for f in R.FEATURE_FIELDS:
                out[f][i * k + j] = r[f]
            if frags is not None:
                out["frag_offset"][i * k + j] = len(frag_rows)
                out["frag_count"][i * k + j] = len(r["fragments"])
                frag_rows += r["fragments"]
    fr = None
    if frags is not None:
        fr = np.zeros(len(frag_rows), FRAGMENT_DTYPE)
        for t, (kind, c, ordn, it, calc, exp) in enumerate(frag_rows):
            fr[t] = (kind, c, ordn, it, calc, exp)
    return out, counts, fr, ctr


F32_FIELDS = ["expmass", "calcmass", "delta_mass", "isotope_error", "average_ppm", "longest_y_pct", "matched_intensity_pct", "ms2_intensity"]
INT_FIELDS = ["peptide_idx", "peptide_len", "rank", "label", "charge", "matched_peaks", "longest_b", "longest_y", "missed_cleavages", "scored_candidates"]
F64_FIELDS = ["hyperscore", "delta_next", "delta_best", "poisson"]


def _nan_or_same(x, y, bits):
    """Equal bit patterns, or NaN on both sides: the reference does not fix a NaN's sign or payload (x86 gives 0xFFC00000 for 0/0,
    the device the canonical 0x7FFFFFFF)."""
    return (np.ascontiguousarray(x).view(bits) == np.ascontiguousarray(y).view(bits)) | (np.isnan(x) & np.isnan(y))


def assert_rows_bits_equal(a, ca, b, cb, report_psms, what="", f64=True):
    """Counts, then every Feature field bit for bit (f32 and f64 by their bit patterns; any NaN equals any NaN); f64=False leaves out the
    four f64 scores. Returns the number of rows compared."""
    assert np.array_equal(np.asarray(ca), np.asarray(cb)), f"{what}: PSM counts differ at spectra {np.nonzero(np.asarray(ca) != np.asarray(cb))[0][:10]}"
    sel = (np.arange(len(a)) % report_psms) < np.repeat(np.asarray(ca), report_psms)
    x, y = a[sel], b[sel]
    for f in INT_FIELDS:
        bad = np.nonzero(x[f].astype(np.int64) != y[f].astype(np.int64))[0]
        assert len(bad) == 0, f"{what}: {f} differs at rows {bad[:5]}: {x[f][bad[:5]]} vs {y[f][bad[:5]]}"
    for f in F32_FIELDS:
        bad = np.nonzero(~_nan_or_same(x[f], y[f], np.uint32))[0]
        assert len(bad) == 0, f"{what}: {f} differs at rows {bad[:5]}: {x[f][bad[:5]]} vs {y[f][bad[:5]]}"
    for f in (F64_FIELDS if f64 else []):
        bad = np.nonzero(~_nan_or_same(x[f], y[f], np.uint64))[0]
        assert len(bad) == 0, f"{what}: {f} differs at rows {bad[:5]}: {[float(v).hex() for v in x[f][bad[:5]]]} vs {[float(v).hex() for v in y[f][bad[:5]]]}"
    return int(sel.sum())


def _frag_fields(rows):
    names = rows.dtype.names
    return ("frag_offset", "frag_count") if "frag_offset" in names else ("fragment_offset", "fragment_count")


def assert_fragments_equal(a, ca, fa, b, cb, fb, report_psms, what=""):
    """The Fragments of every reported row: kind, charge, ordinal, intensity, calculated and experimental m/z, in order, bit for bit."""
    sel_a = (np.arange(len(a)) % report_psms) < np.repeat(np.asarray(ca), report_psms)
    sel_b = (np.arange(len(b)) % report_psms) < np.repeat(np.asarray(cb), report_psms)
    (oa, na), (ob, nb) = _frag_fields(a), _frag_fields(b)
    for ra, rb in zip(a[sel_a], b[sel_b]):
        assert ra[na] == rb[nb], f"{what}: fragment counts differ"
        xa = fa[int(ra[oa]):int(ra[oa]) + int(ra[na])]
        xb = fb[int(rb[ob]):int(rb[ob]) + int(rb[nb])]
        for f in ("kind", "charge", "ordinal"):
            assert np.array_equal(xa[f], xb[f]), f"{what}: fragment {f} differs"
        for f in ("intensity", "mz_calculated", "mz_experimental"):
            assert np.all(_nan_or_same(xa[f], xb[f], np.uint32)), f"{what}: fragment {f} differs"
