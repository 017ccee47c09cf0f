"""Synthetic workloads of the shapes BASELINE.json names (SURVEY.md §8d): a human-tryptic-scale peptide table and
200-peak MS2 spectra. Product-side (bench.py, tests, smoke) — independent of oracle/.

Peptides follow the reference's digest conventions (trypsin KR|P, 1 missed cleavage, length 5-50, mass 500-5000,
reversed decoys `Peptide::reverse`, sort by (monoisotopic, sequence), dedup) but nothing here needs to be bit-faithful
to the reference's digest: both the oracle and the CUDA path consume exactly these arrays.
"""
from __future__ import annotations

import itertools
import os

import numpy as np

from .api import Peptides, SpectraBatch

H2O = np.float32(18.010565)
PROTON = np.float32(1.0072764)
# mass.rs:64-76
MONO = np.zeros(256, np.float32)
for _aa, _m in zip("ACDEFGHIKLMNPQRSTVWY", [71.03711, 103.00919, 115.02694, 129.04259, 147.0684, 57.02146, 137.05891, 113.08406, 128.09496,
                                           113.08406, 131.0405, 114.04293, 97.05276, 128.05858, 156.1011, 87.03203, 101.04768, 99.06841,
                                           186.07932, 163.06332]):
    MONO[ord(_aa)] = _m
# approximate SwissProt residue frequencies (%), order ACDEFGHIKLMNPQRSTVWY
_FREQ = np.array([8.25, 1.37, 5.45, 6.75, 3.86, 7.07, 2.27, 5.96, 5.84, 9.66, 2.42, 4.06, 4.70, 3.93, 5.53, 6.56, 5.34, 6.87, 1.08, 2.92])
_AA = np.frombuffer(b"ACDEFGHIKLMNPQRSTVWY", np.uint8)
MAX_LEN = 50


def _digest(prot: np.ndarray, prot_off: np.ndarray, missed: int, min_len: int, max_len: int):
    """Tryptic (KR, not before P) segments with up to `missed` missed cleavages -> (start, end, n_missed)."""
    n = len(prot)
    is_end = np.zeros(n, bool)
    is_end[prot_off[1:] - 1] = True
    nxt_p = np.zeros(n, bool)
    nxt_p[:-1] = prot[1:] == ord("P")
    cut = (((prot == ord("K")) | (prot == ord("R"))) & ~nxt_p) | is_end  # cleave after these positions
    ends = np.nonzero(cut)[0] + 1
    starts = np.concatenate([[0], ends[:-1]])
    seg_prot = np.searchsorted(prot_off, starts, side="right") - 1
    S, E, M = [starts], [ends], [np.zeros(len(starts), np.uint8)]
    for m in range(1, missed + 1):
        ok = seg_prot[:-m] == seg_prot[m:]
        S.append(starts[:-m][ok])
        E.append(ends[m:][ok])
        M.append(np.full(int(ok.sum()), m, np.uint8))
    s, e, mm = np.concatenate(S), np.concatenate(E), np.concatenate(M)
    ln = e - s
    keep = (ln >= min_len) & (ln <= max_len)
    return s[keep], e[keep], mm[keep]


def _gather(prot, s, e):
    ln = (e - s).astype(np.int64)
    idx = s[:, None] + np.arange(MAX_LEN)[None, :]
    mat = prot[np.minimum(idx, len(prot) - 1)]
    mat[np.arange(MAX_LEN)[None, :] >= ln[:, None]] = 0
    return mat, ln


def _reverse_inner(mat, ln):
    """Peptide::reverse (peptide.rs:307-318): reverse residues 1..len-1, keep first and last."""
    out = mat.copy()
    j = np.arange(MAX_LEN)[None, :]
    src = np.where((j >= 1) & (j < ln[:, None] - 1), ln[:, None] - 1 - j, j)
    inner = ln > 2
    out[inner] = np.take_along_axis(mat[inner], src[inner], axis=1)
    return out


def _expand_variable_mods(site_mass, max_variable_mods):
    """Peptide::apply (peptide.rs:258-305): every combination of up to `max_variable_mods` variable modifications on distinct sites
    (site_mass != 0 marks a site). Returns the base row of every form (the unmodified forms first) and the (form, column) pairs to modify."""
    n = len(site_mass)
    is_site = site_mass != 0
    nsite = is_site.sum(axis=1)
    maxs = int(nsite.max()) if n else 0
    order = np.argsort(~is_site, axis=1, kind="stable")[:, :max(maxs, 1)]   # order[i, k] = column of the k-th site of row i
    base_rows, add_rows, add_cols = [np.arange(n)], [], []
    form_count = n
    for k in range(1, max_variable_mods + 1):
        for slots in itertools.combinations(range(maxs), k):
            rows = np.nonzero(nsite > slots[-1])[0]
            if len(rows) == 0:
                continue
            base_rows.append(rows)
            ids = form_count + np.arange(len(rows))
            for sl in slots:
                add_rows.append(ids)
                add_cols.append(order[rows, sl])
            form_count += len(rows)
    base = np.concatenate(base_rows)
    if add_rows:
        return base, np.concatenate(add_rows), np.concatenate(add_cols)
    return base, np.zeros(0, np.int64), np.zeros(0, np.int64)


_NATIVE = None


def _native():
    """libsage_synth.so (sage_b200/csrc/synth_expand.cpp, built by sage_b200.build): same result as the numpy path, ~100x faster."""
    global _NATIVE
    if _NATIVE is None:
        import ctypes as C
        from .build import synth_library_path
        path = synth_library_path()
        if os.environ.get("SAGE_B200_SYNTH_NUMPY") == "1" or not os.path.exists(path):
            _NATIVE = False
        else:
            lib = C.CDLL(path)
            lib.synth_expand.restype = C.c_void_p
            lib.synth_expand.argtypes = [C.c_uint64, C.c_uint32] + [C.c_void_p] * 7 + [C.c_uint32, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
            lib.synth_expand_fetch.argtypes = [C.c_void_p] * 7
            lib.synth_expand_free.argtypes = [C.c_void_p]
            _NATIVE = lib
    return _NATIVE or None


def _expand_native(lib, mat, ln, static, site_mass, base_mono, decoy, missed, max_mods):
    import ctypes as C
    mat, ln = np.ascontiguousarray(mat, np.uint8), np.ascontiguousarray(ln, np.int64)
    static, site_mass, base_mono = (np.ascontiguousarray(x, np.float32) for x in (static, site_mass, base_mono))
    decoy, missed = np.ascontiguousarray(decoy, np.uint8), np.ascontiguousarray(missed, np.uint8)
    n_out, n_res = C.c_uint64(0), C.c_uint64(0)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    h = lib.synth_expand(len(mat), mat.shape[1], p(mat), p(ln), p(static), p(site_mass), p(base_mono), p(decoy), p(missed), max_mods,
                         C.c_float(500.0), C.c_float(5000.0), C.byref(n_out), C.byref(n_res))
    if not h:
        raise RuntimeError("synth_expand failed (too many forms / residues for u32 offsets)")
    n, r = n_out.value, n_res.value
    seq_off, seq, mods = np.zeros(n + 1, np.uint32), np.zeros(r, np.uint8), np.zeros(r, np.float32)
    mono, dec, mis = np.zeros(n, np.float32), np.zeros(n, np.uint8), np.zeros(n, np.uint8)
    lib.synth_expand_fetch(h, p(seq_off), p(seq), p(mods), p(mono), p(dec), p(mis))
    lib.synth_expand_free(h)
    return Peptides(seq_off=seq_off, seq=seq, mods=mods, nterm=np.full(n, np.nan, np.float32), mono=mono, decoy=dec, missed=mis)


def make_peptides(n_target: int = 2_000_000, seed: int = 0x5A6E, missed: int = 1, static_c: bool = False, il_twin_fraction: float = 0.02,
                  var_mod_m: bool = False, var_mods=(), max_variable_mods: int = 2) -> Peptides:
    """Peptide table sorted like reorder_peptides (database.rs:221-258). `n_target` ~ rows (targets + reversed decoys) BEFORE the variable
    modifications are enumerated; var_mods = ((residues, mass), ...) adds every combination of up to max_variable_mods modified sites
    (peptide.rs:258-305), e.g. (("M", 15.9949), ("STY", 79.9663)) turns ~1.9 M rows into ~15 M. var_mod_m is shorthand for M+15.9949 with
    at most one modified site per form."""
    rng = np.random.default_rng(seed)
    if var_mod_m and not var_mods:
        var_mods, max_variable_mods = (("M", 15.9949),), 1
    # ~1 unique peptide (0+1 missed, len 5-50, after dedup) per 5.3 residues; decoys double it
    n_res = int(n_target * 2.75) + 4096
    lens = np.maximum(30, rng.lognormal(np.log(375.0), 0.6, size=max(8, n_res // 430))).astype(np.int64)
    prot_off = np.concatenate([[0], np.cumsum(lens)])
    prot = rng.choice(_AA, size=int(prot_off[-1]), p=_FREQ / _FREQ.sum())
    if il_twin_fraction > 0:  # I/L-swapped protein copies -> isobaric twin peptides (exercise tie order)
        k = max(1, int(len(lens) * il_twin_fraction))
        extra, extra_len = [], []
        for pi in rng.choice(len(lens), size=k, replace=False):
            seg = prot[prot_off[pi]:prot_off[pi + 1]].copy()
            il = np.nonzero((seg == ord("I")) | (seg == ord("L")))[0]
            flip = il[rng.random(len(il)) < 0.3]
            seg[flip] = np.where(seg[flip] == ord("I"), ord("L"), ord("I")).astype(np.uint8)
            extra.append(seg)
            extra_len.append(len(seg))
        prot = np.concatenate([prot] + extra)
        prot_off = np.concatenate([prot_off, prot_off[-1] + np.cumsum(extra_len)])
    s, e, mm = _digest(prot, prot_off, missed, 5, MAX_LEN)
    mat, ln = _gather(prot, s, e)
    # unique target sequences
    key = np.ascontiguousarray(mat).view(f"S{MAX_LEN}").ravel()
    _, first = np.unique(key, return_index=True)
    mat, ln, mm = mat[first], ln[first], mm[first]
    tkey = np.ascontiguousarray(mat).view(f"S{MAX_LEN}").ravel()
    dmat = _reverse_inner(mat, ln)
    dkey = np.ascontiguousarray(dmat).view(f"S{MAX_LEN}").ravel()
    _, dfirst = np.unique(dkey, return_index=True)
    dkeep = dfirst[~np.isin(dkey[dfirst], tkey)]  # decoys equal to a target sequence are dropped (database.rs:212)
    allmat = np.concatenate([mat, dmat[dkeep]])
    allln = np.concatenate([ln, ln[dkeep]])
    allmm = np.concatenate([mm, mm[dkeep]])
    decoy = np.concatenate([np.zeros(len(mat), np.uint8), np.ones(len(dkeep), np.uint8)])
    # rows in sequence order: the final stable sort by mass then yields (monoisotopic, sequence, modifications-in-enumeration-order)
    sorder = np.argsort(np.ascontiguousarray(allmat).view(f"S{MAX_LEN}").ravel(), kind="stable")
    allmat, allln, allmm, decoy = allmat[sorder], allln[sorder], allmm[sorder], decoy[sorder]
    res = MONO[allmat]
    base = np.cumsum(np.concatenate([np.full((len(allmat), 1), H2O, np.float32), res], axis=1), axis=1, dtype=np.float32)[:, -1]
    valid = np.arange(MAX_LEN)[None, :] < allln[:, None]
    static = np.zeros(allmat.shape, np.float32)
    if static_c:
        static[allmat == ord("C")] = np.float32(57.0216)
    if var_mods:
        # variable mods first, then static mods on the sites still unmodified (peptide.rs:293-300); disjoint residue sets here
        site_mass = np.zeros(allmat.shape, np.float32)
        for residues, mass in var_mods:
            for r in residues:
                site_mass[(allmat == ord(r)) & (static == 0) & valid] = np.float32(mass)
        lib = _native()
        if lib is not None:
            return _expand_native(lib, allmat, allln, static, site_mass, base, decoy, allmm, int(max_variable_mods))
        form_base, ar, ac = _expand_variable_mods(site_mass, int(max_variable_mods))
        nforms = len(form_base)
        if nforms > 4_000_000:
            raise RuntimeError("variable-modification tables of this size need the native helper (python -m sage_b200.build)")
        fmods = static[form_base]
        fmods[ar, ac] = site_mass[form_base[ar], ac]
        # modification_mass (peptide.rs:129-133): sequential f32 sum over the residues
        mono = (base[form_base] + np.cumsum(fmods, axis=1, dtype=np.float32)[:, -1]).astype(np.float32)
        keep = np.nonzero((mono >= np.float32(500.0)) & (mono <= np.float32(5000.0)))[0]
        # reorder_peptides: (monoisotopic, sequence == base row, modifications lexicographic); mods >= 0, so big-endian bit patterns sort like values
        mkey = np.ascontiguousarray(fmods[keep].view(np.uint32).astype(">u4")).view(f"S{4 * MAX_LEN}").ravel()
        order = keep[np.lexsort((mkey, form_base[keep], mono[keep]))]
        fb = form_base[order]
        fvalid = valid[fb]
        seq_off = np.concatenate([[0], np.cumsum(allln[fb])]).astype(np.uint32)
        return Peptides(seq_off=seq_off, seq=allmat[fb][fvalid].astype(np.uint8), mods=fmods[order][fvalid].astype(np.float32),
                        nterm=np.full(len(order), np.nan, np.float32), mono=mono[order], decoy=decoy[fb], missed=allmm[fb])
    mods = static
    # monoisotopic = H2O + sum(residues) (sequential f32, peptide.rs:361-373) + modification_mass (peptide.rs:129-133)
    modsum = np.cumsum(mods, axis=1, dtype=np.float32)[:, -1]
    mono = (base + modsum).astype(np.float32)
    keep = (mono >= np.float32(500.0)) & (mono <= np.float32(5000.0))
    allmat, allln, allmm, decoy, mods, mono = allmat[keep], allln[keep], allmm[keep], decoy[keep], mods[keep], mono[keep]
    order = np.argsort(mono, kind="stable")   # rows are in sequence order already: (monoisotopic, sequence)
    allmat, allln, allmm, decoy, mods, mono = allmat[order], allln[order], allmm[order], decoy[order], mods[order], mono[order]
    valid = np.arange(MAX_LEN)[None, :] < allln[:, None]
    seq_off = np.concatenate([[0], np.cumsum(allln)]).astype(np.uint32)
    return Peptides(seq_off=seq_off, seq=allmat[valid].astype(np.uint8), mods=mods[valid].astype(np.float32),
                    nterm=np.full(len(mono), np.nan, np.float32), mono=mono, decoy=decoy, missed=allmm)


def make_spectra(pep: Peptides, n: int = 50_000, seed: int = 0xB202, n_peaks: int = 200, chimeric: bool = False, charge_known: bool = True) -> SpectraBatch:
    """Synthetic MS2 spectra (SURVEY.md §8d): a target peptide's b/y ions at z=1 (and z=2 for 30% of 3+ precursors), 50% dropout,
    4 ppm jitter, padded with uniform noise to exactly n_peaks; lognormal intensities (signal x3); masses sorted ascending."""
    rng = np.random.default_rng(seed)
    targets = np.nonzero(pep.decoy == 0)[0]
    ln_all = np.diff(pep.seq_off.astype(np.int64))

    def one_component(choice):
        ln = ln_all[choice]
        idx = pep.seq_off[choice].astype(np.int64)[:, None] + np.arange(MAX_LEN)[None, :]
        valid = np.arange(MAX_LEN)[None, :] < ln[:, None]
        idx = np.minimum(idx, len(pep.seq) - 1)
        rm = np.where(valid, MONO[pep.seq[idx]] + pep.mods[idx], np.float32(0)).astype(np.float32)
        b = np.cumsum(rm, axis=1, dtype=np.float32)  # b_i, i = 1..L (last one is not an ion)
        mono = pep.mono[choice]
        y = mono[:, None] - b
        ion_ok = np.arange(MAX_LEN)[None, :] < (ln[:, None] - 1)
        return b, y, ion_ok, mono

    choice = rng.choice(targets, size=n)
    z = np.where(rng.random(n) < 0.6, 2, 3).astype(np.uint8)
    b, y, ion_ok, mono = one_component(choice)
    prec_mz = ((mono.astype(np.float64) + z * float(PROTON)) / z * (1.0 + rng.normal(0, 3e-6, n))).astype(np.float32)
    comps = [(b, y, ion_ok, np.ones(n, bool))]
    if chimeric:  # second, co-isolated peptide whose precursor m/z is within 1 Th (a neighbour in the mass-sorted table)
        mass_rank = np.searchsorted(pep.mono[targets], mono)
        other = targets[np.clip(mass_rank + rng.integers(-200, 200, n), 0, len(targets) - 1)]
        b2, y2, ok2, _ = one_component(other)
        comps.append((b2, y2, ok2, np.ones(n, bool)))
    sig_m, sig_ok, sig_w = [], [], []
    for ci, (bb, yy, ok, _) in enumerate(comps):
        z2 = (z == 3) & (rng.random(n) < 0.3)
        for ions in (bb, yy):
            for fc, allow in ((1, np.ones(n, bool)), (2, z2)):
                keep = ok & allow[:, None] & (rng.random(ions.shape) < 0.5)
                m = ions.astype(np.float64) / fc * (1.0 + rng.normal(0, 4e-6, ions.shape))
                sig_m.append(m)
                sig_ok.append(keep & (m > 50.0))
                sig_w.append(np.full(ions.shape, 3.0 * (0.6 if (chimeric and ci == 0) else (0.4 if chimeric else 1.0)) / (1.0 if not chimeric else 0.6)))
    sig_m, sig_ok, sig_w = np.concatenate(sig_m, axis=1), np.concatenate(sig_ok, axis=1), np.concatenate(sig_w, axis=1)
    hi = np.minimum(2000.0, mono.astype(np.float64))
    masses = (150.0 + rng.random((n, n_peaks)) * (hi - 150.0)[:, None]) - float(PROTON)
    intens = rng.lognormal(8.0, 1.2, (n, n_peaks))
    # overwrite the first k_i slots of each row with that row's signal peaks
    rank = np.cumsum(sig_ok, axis=1) - 1
    take = sig_ok & (rank < n_peaks)
    rows = np.nonzero(take)[0]
    cols = rank[take]
    masses[rows, cols] = sig_m[take]
    intens[rows, cols] = intens[rows, cols] * sig_w[take]
    masses = masses.astype(np.float32)
    intens = intens.astype(np.float32)
    order = np.argsort(masses, axis=1, kind="stable")
    masses = np.take_along_axis(masses, order, axis=1)
    intens = np.take_along_axis(intens, order, axis=1)
    tic = np.cumsum(intens, axis=1, dtype=np.float32)[:, -1]  # sequential f32 sum (spectrum.rs:398)
    peak_off = (np.arange(n + 1, dtype=np.uint64) * np.uint64(n_peaks))
    chg = z if charge_known else np.zeros(n, np.uint8)
    return SpectraBatch(peak_off=peak_off, masses=masses.ravel(), intensities=intens.ravel(), prec_mz=prec_mz, prec_charge=chg,
                        iso_lo=np.full(n, np.nan, np.float32), iso_hi=np.full(n, np.nan, np.float32), tic=tic, level=np.full(n, 2, np.uint8),
                        rt=(np.arange(n, dtype=np.float32) * np.float32(0.01)), ims=np.full(n, np.nan, np.float32))


NEUTRON = np.float32(1.00335)
# carbon count per residue (mass.rs:78-104), for an approximate isotope envelope
_CARBON = np.zeros(256, np.int64)
for _aa, _c in zip("ACDEFGHIKLMNPQRSTVWYUO", [3, 3, 4, 5, 9, 2, 6, 6, 6, 6, 5, 4, 5, 5, 6, 3, 4, 5, 11, 9, 3, 12]):
    _CARBON[ord(_aa)] = _c


def make_ms1_runs(pep: Peptides, n_ids: int = 30_000, n_files: int = 4, spectra_per_file: int = 3000, peaks_per_spectrum: int = 1500, seed: int = 0x1F0,
                  mobility: bool = False, charges=(2, 3), absent_fraction: float = 0.15, ppm_jitter: float = 2.0, sigma: float = 0.0015,
                  rt_range=(0.05, 0.95), scan_range=None, rt_offset_bins=None, distort: bool = True, ref_file=None, silent_files=()):
    """Synthetic label-free quantification input: `n_ids` target peptides "identified" at an aligned RT (normalized run time, uniform in
    `rt_range`), a charge and a file; per-file linear RT distortion (returned as the alignments that undo it); Gaussian elution profiles (sd
    `sigma` in aligned RT) of 3-isotope envelopes from each peptide's carbon count, with ppm jitter; every peptide absent from a random
    `absent_fraction` of the other files; noise peaks up to `peaks_per_spectrum`; optionally per-peak mobilities. The Feature rows also hold
    filtered-out rows (q-value too high, decoys) and lower-confidence repeats of identified peptides, as a real confidence-sorted Feature table does.
    Options that shape the time warps quantification finds (the defaults leave the output unchanged):
      scan_range      (lo, hi): the spectra sample this aligned-RT interval evenly instead of the whole run;
      rt_offset_bins  one int per file: that file's elution is late by this many grid bins (RT_TOL * 2 / 100 = 1e-4 of aligned RT each);
      distort=False   identity alignments (max_rt 100, slope 1, intercept 0): every file samples the same aligned RTs;
      ref_file        every identified peptide's best PSM is in this file (the grid's reference file);
      silent_files    files with no peptide signal at all.
    Returns dict(features, alignments, batch: Ms1Batch of every file's spectra in acquisition order, file by file)."""
    from .api import ALIGNMENT_DTYPE, Ms1Batch
    rng = np.random.default_rng(seed)
    targets = np.nonzero(pep.decoy == 0)[0]
    decoys = np.nonzero(pep.decoy != 0)[0]
    ids = rng.choice(targets, size=min(n_ids, len(targets)), replace=False).astype(np.uint32)
    n = len(ids)
    t_rt = rng.uniform(rt_range[0], rt_range[1], n).astype(np.float32)
    charge = rng.choice(np.asarray(charges), n).astype(np.int64)
    file_of = rng.integers(0, n_files, n).astype(np.uint32)
    if ref_file is not None:
        file_of[:] = ref_file
    shift = np.zeros(n_files) if rt_offset_bins is None else np.asarray(rt_offset_bins, np.float64) * 1e-4
    ims = rng.uniform(0.7, 1.3, n).astype(np.float32) if mobility else np.zeros(n, np.float32)
    mono = pep.mono[ids].astype(np.float32)
    off = pep.seq_off.astype(np.int64)
    carbon = np.add.reduceat(_CARBON[pep.seq], off[:-1])[ids] if len(pep.seq) else np.zeros(n, np.int64)
    lam = carbon * 0.011
    env = np.stack([np.ones(n), lam, lam * lam / 2.0], axis=1)
    env /= env.max(axis=1, keepdims=True)
    present = rng.random((n_files, n)) >= absent_fraction
    present[file_of, np.arange(n)] = True
    present[list(silent_files)] = False
    abundance = np.exp(rng.normal(13.0, 1.5, n))

    # features: identified rows, then lower-confidence repeats, rows above the q-value cut and decoy rows, shuffled after the first block
    n_rep, n_bad, n_dec = n // 5, n // 10, n // 10
    rep = rng.choice(n, n_rep)
    bad = rng.choice(targets, n_bad).astype(np.uint32)
    dec = rng.choice(decoys, n_dec).astype(np.uint32) if len(decoys) else np.zeros(0, np.uint32)
    tail_pep = np.concatenate([ids[rep], bad, dec])
    m = len(tail_pep)
    feats = np.zeros(n + m, dtype=[("peptide_idx", "<u4"), ("peptide_q", "<f4"), ("label", "<i4"), ("aligned_rt", "<f4"), ("calcmass", "<f4"),
                                   ("file_id", "<u4"), ("ims", "<f4")])
    feats["peptide_idx"] = np.concatenate([ids, tail_pep])
    feats["peptide_q"] = np.concatenate([rng.uniform(0, 0.01, n), rng.uniform(0, 0.01, n_rep), rng.uniform(0.0101, 0.5, n_bad), rng.uniform(0, 0.01, n_dec)])
    feats["label"] = np.concatenate([np.ones(n + n_rep + n_bad, np.int32), -np.ones(n_dec, np.int32)])
    feats["aligned_rt"] = np.concatenate([t_rt + rng.normal(0, sigma / 4, n).astype(np.float32), rng.uniform(0, 1, m).astype(np.float32)])
    feats["calcmass"] = pep.mono[feats["peptide_idx"]]
    feats["file_id"] = np.concatenate([file_of, rng.integers(0, n_files, m).astype(np.uint32)])
    feats["ims"] = np.concatenate([ims, rng.uniform(0.7, 1.3, m).astype(np.float32) if mobility else np.zeros(m, np.float32)])
    tail = n + rng.permutation(m)
    feats = np.concatenate([feats[:n], feats[tail]])

    align = np.zeros(n_files, ALIGNMENT_DTYPE)
    align["max_rt"] = rng.uniform(60.0, 120.0, n_files)
    align["slope"] = rng.uniform(0.95, 1.05, n_files)
    align["intercept"] = rng.uniform(-0.02, 0.02, n_files)
    if not distort:
        align["max_rt"], align["slope"], align["intercept"] = 100.0, 1.0, 0.0

    offs, masses, intens, fids, ssts, mobs = [np.zeros(1, np.uint64)], [], [], [], [], []
    total = 0
    for f in range(n_files):
        sel = np.nonzero(present[f])[0]
        sel = sel[np.argsort(t_rt[sel])]
        if scan_range is None:
            sst = (np.arange(spectra_per_file, dtype=np.float64) + 0.5) / spectra_per_file * float(align["max_rt"][f])
        else:
            want = scan_range[0] + (np.arange(spectra_per_file, dtype=np.float64) + 0.5) / spectra_per_file * (scan_range[1] - scan_range[0])
            sst = (want - float(align["intercept"][f])) / float(align["slope"][f]) * float(align["max_rt"][f])
        arts = (sst / float(align["max_rt"][f])) * float(align["slope"][f]) + float(align["intercept"][f])
        for s in range(spectra_per_file):
            a, b = np.searchsorted(t_rt[sel], [arts[s] - shift[f] - 4 * sigma, arts[s] - shift[f] + 4 * sigma])
            el = sel[a:b]
            prof = abundance[el] * np.exp(-0.5 * ((arts[s] - shift[f] - t_rt[el]) / sigma) ** 2)
            sig_m = ((mono[el, None] + np.arange(3)[None, :] * NEUTRON) / charge[el, None]).ravel()
            sig_m = sig_m * (1.0 + rng.normal(0, ppm_jitter * 1e-6, len(sig_m)))
            sig_i = (prof[:, None] * env[el]).ravel()
            sig_mob = np.repeat(ims[el], 3) * (1.0 + rng.normal(0, 0.002, 3 * len(el)))
            k = max(peaks_per_spectrum - len(sig_m), 0)
            mm = np.concatenate([sig_m, rng.uniform(300.0, 1500.0, k)]).astype(np.float32)
            ii = np.concatenate([sig_i, np.exp(rng.normal(9.0, 1.0, k))]).astype(np.float32)
            mo = np.concatenate([sig_mob, rng.uniform(0.7, 1.3, k)]).astype(np.float32)
            order = np.argsort(mm, kind="stable")
            masses.append(mm[order])
            intens.append(ii[order])
            mobs.append(mo[order])
            total += len(mm)
            offs.append(np.array([total], np.uint64))
            fids.append(f)
            ssts.append(sst[s])
    batch = Ms1Batch(np.concatenate(offs), np.concatenate(masses), np.concatenate(intens), np.array(fids, np.uint32), np.array(ssts, np.float32),
                     np.concatenate(mobs) if mobility else None)
    return dict(features=feats, alignments=align, batch=batch, ids=ids, charge=charge)


def make_psms(n: int, seed: int = 0x0FD2, decoy_fraction: float = 0.3, true_fraction: float = 0.5, ppm: float = 20.0, ims: bool = False,
              rt_range: float = 60.0) -> np.ndarray:
    """Seeded Feature rows (FEATURE_DTYPE) shaped like a search's output, for rescoring (spectrum_fdr). A `decoy_fraction` of the rows are decoys;
    the targets are a mix of true matches (`true_fraction` of them: higher hyperscore, more matched peaks, a mass error centred on 0) and
    false matches drawn like decoys. Mass errors are within +-`ppm`; `ims` fills the mobility column (else 0, as without mobility data)."""
    from .api import FEATURE_DTYPE
    rng = np.random.default_rng(seed)
    out = np.zeros(n, FEATURE_DTYPE)
    decoy = rng.random(n) < decoy_fraction
    true = ~decoy & (rng.random(n) < true_fraction)
    plen = rng.integers(7, 31, n).astype(np.uint32)
    matched = np.where(true, rng.integers(6, 30, n), rng.integers(1, 12, n)).astype(np.uint32)
    longest_b = np.minimum(rng.integers(0, 10, n) + true * rng.integers(0, 8, n), plen - 1).astype(np.uint32)
    longest_y = np.minimum(rng.integers(0, 10, n) + true * rng.integers(0, 12, n), plen - 1).astype(np.uint32)
    hyper = np.where(true, rng.normal(40.0, 8.0, n), rng.normal(18.0, 6.0, n)).clip(0.5, None)
    delta_next = (hyper * np.where(true, rng.uniform(0.05, 0.6, n), rng.uniform(0.0, 0.15, n)))
    charge = rng.integers(2, 5, n).astype(np.uint32)
    calc = rng.uniform(700.0, 4000.0, n).astype(np.float32)
    dppm = np.where(true, rng.normal(0.0, ppm / 8.0, n), rng.uniform(-ppm, ppm, n)).clip(-ppm, ppm).astype(np.float32)
    exp = (calc.astype(np.float64) * (1.0 + dppm.astype(np.float64) * 1e-6)).astype(np.float32)
    out["spectrum"] = np.arange(n, dtype=np.uint32)
    out["peptide_idx"] = rng.integers(0, 1 << 20, n).astype(np.uint32)
    out["peptide_len"] = plen
    out["rank"] = np.where(rng.random(n) < 0.8, 1, 2).astype(np.uint32)
    out["label"] = np.where(decoy, -1, 1).astype(np.int32)
    out["expmass"], out["calcmass"] = exp, calc
    out["charge"] = charge
    out["rt"] = rng.uniform(0.0, rt_range, n).astype(np.float32)
    out["ims"] = rng.uniform(0.6, 1.4, n).astype(np.float32) if ims else np.float32(0)
    out["delta_mass"] = np.abs(dppm)
    out["isotope_error"] = np.where(rng.random(n) < 0.05, 1.0, 0.0).astype(np.float32)
    out["average_ppm"] = np.abs(np.where(true, rng.normal(0.0, 3.0, n), rng.uniform(-10.0, 10.0, n))).astype(np.float32)
    out["hyperscore"] = hyper
    out["delta_next"] = delta_next
    out["delta_best"] = np.where(out["rank"] == 1, 0.0, delta_next * 0.5)
    out["matched_peaks"] = matched
    out["longest_b"], out["longest_y"] = longest_b, longest_y
    out["longest_y_pct"] = (longest_y.astype(np.float32) / plen.astype(np.float32)).astype(np.float32)
    out["missed_cleavages"] = rng.integers(0, 2, n).astype(np.uint32)
    out["matched_intensity_pct"] = np.where(true, rng.uniform(20.0, 80.0, n), rng.uniform(1.0, 30.0, n)).astype(np.float32)
    out["scored_candidates"] = rng.integers(1, 5000, n).astype(np.uint32)
    out["ms2_intensity"] = rng.uniform(1e3, 1e6, n).astype(np.float32)
    out["poisson"] = np.where(true, -rng.uniform(5.0, 20.0, n), -rng.uniform(0.0, 4.0, n))
    return out


def make_rt_psms(pep: Peptides, n: int, n_files: int, seed: int = 0x5E7, mobility: bool = False, with_truth: bool = False):
    """Seeded Feature rows (FEATURE_DTYPE) and their file ids for the predict_rt stage (runner.rs:513-531). A quarter of the rows are decoys; 60 %
    of the targets are true matches (poisson -20 .. -5) and the rest false (poisson -4 .. 0, like the decoys). A true match's normalised RT is a
    hidden linear function of its peptide's residue counts and length (the RT model's features) plus noise; file f then applies its own linear
    distortion x = (rt - b_f) / a_f and scale rt = x * T_f (T_f uniform in 60 .. 120). False matches and decoys get uniform RTs. With
    `mobility`, every row's ims is linear in the mobility model's features (residue fractions, 1 / charge, mass) plus noise; otherwise 0.
    Returns (rows, file_id), plus a dict of the hidden values (rt_true, is_true, T, a, b per file) when `with_truth`."""
    from .api import FEATURE_DTYPE
    rng = np.random.default_rng(seed)
    rows = make_psms(n, seed=seed)
    decoy = rng.random(n) < 0.25
    true = ~decoy & (rng.random(n) < 0.6)
    targets, decoys = np.nonzero(pep.decoy == 0)[0], np.nonzero(pep.decoy != 0)[0]
    pidx = rng.choice(targets, n).astype(np.uint32)
    if len(decoys):
        pidx[decoy] = rng.choice(decoys, int(decoy.sum())).astype(np.uint32)
    off = pep.seq_off.astype(np.int64)
    lens = np.diff(off)
    coef = np.zeros(256)
    coef[np.frombuffer(b"ACDEFGHIKLMNPQRSTVWYUO", np.uint8)] = rng.uniform(-0.02, 0.04, 22)
    raw = np.add.reduceat(coef[pep.seq], off[:-1]) + 0.004 * lens if len(pep.seq) else np.zeros(len(lens))
    lo, hi = raw.min(), raw.max()
    pep_rt = 0.05 + 0.9 * (raw - lo) / max(hi - lo, 1e-12)
    rt_true = pep_rt[pidx] + rng.normal(0.0, 0.004, n)
    fid = rng.integers(0, n_files, n).astype(np.uint32)
    T, a, b = rng.uniform(60.0, 120.0, n_files), rng.uniform(0.9, 1.1, n_files), rng.uniform(-0.05, 0.05, n_files)
    x = np.where(true, (rt_true - b[fid]) / a[fid], rng.uniform(0.0, 1.0, n))
    rows["peptide_idx"] = pidx
    rows["peptide_len"] = lens[pidx].astype(np.uint32)
    rows["label"] = np.where(decoy, -1, 1).astype(np.int32)
    rows["poisson"] = np.where(true, -rng.uniform(5.0, 20.0, n), -rng.uniform(0.0, 4.0, n))
    rows["rt"] = (x * T[fid]).astype(np.float32)
    charge = rows["charge"].astype(np.float64)
    if mobility:
        cim = np.zeros(256)
        cim[np.frombuffer(b"ACDEFGHIKLMNPQRSTVWYUO", np.uint8)] = rng.uniform(-0.3, 0.3, 22)
        pep_ims = (np.add.reduceat(cim[pep.seq], off[:-1]) / lens if len(pep.seq) else np.zeros(len(lens))) + 0.1 * pep.mono.astype(np.float64) / 1000.0
        rows["ims"] = (0.6 + pep_ims[pidx] + 0.6 / charge + rng.normal(0.0, 0.003, n)).astype(np.float32)
    else:
        rows["ims"] = np.float32(0)
    if with_truth:
        return rows, fid, dict(rt_true=rt_true, is_true=true, T=T, a=a, b=b)
    return rows, fid


def make_raw_spectra(n: int, peaks=(0, 400), levels=(1, 2, 3), order: str = "shuffled", mobility: bool = False, duplicate_fraction: float = 0.1,
                     mz_range=(100.0, 2000.0), seed: int = 0x5A7):
    """Synthetic RawSpectrum batch (any levels) for SpectrumProcessor::process: n spectra with a peak count uniform in [peaks[0], peaks[1]],
    a level drawn from `levels`, log-normal intensities, `duplicate_fraction` of each spectrum's m/z repeating an earlier one of it (with
    its own intensity, so a stable sort is visible), and peaks in `order`: "sorted" (ascending m/z), "reversed" or "shuffled". With
    `mobility`, every peak has one (RawSpectrum::mobility is Some for the whole batch). Precursor charges are 0 (None) to 4."""
    from .api import RawSpectra
    rng = np.random.default_rng(seed)
    cnt = rng.integers(peaks[0], peaks[1] + 1, n)
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum(cnt)
    mzs, its = [], []
    for c in cnt:
        mz = rng.uniform(mz_range[0], mz_range[1], c).astype(np.float32)
        dup = np.nonzero(rng.random(c) < duplicate_fraction)[0]
        dup = dup[dup > 0]
        mz[dup] = mz[rng.integers(0, np.maximum(dup, 1))]
        if order == "sorted":
            mz = np.sort(mz, kind="stable")
        elif order == "reversed":
            mz = np.sort(mz, kind="stable")[::-1].copy()
        elif order != "shuffled":
            raise ValueError(f"order must be sorted, reversed or shuffled, not {order!r}")
        mzs.append(mz)
        its.append(np.exp(rng.normal(9.0, 1.5, c)).astype(np.float32))
    cat = (lambda x: np.concatenate(x).astype(np.float32) if n else np.zeros(0, np.float32))
    total = int(off[-1])
    return RawSpectra(off, cat(mzs), cat(its), rng.choice(np.asarray(levels, np.uint8), n).astype(np.uint8), rng.integers(0, 5, n).astype(np.uint8),
                      rng.uniform(0.6, 1.4, total).astype(np.float32) if mobility else None, np.zeros(n, np.uint32), np.arange(n, dtype=np.float32))


def ms1_to_raw(batch, shuffle: bool = False, seed: int = 0x5A8):
    """The raw MS1 spectra behind an Ms1Batch of make_ms1_runs: m/z = mass + PROTON in f32, every peak's intensity and mobility with it,
    optionally shuffled inside each spectrum. (Processing them again gives masses within an ulp of the batch's, not the same bits.)"""
    from .api import RawSpectra
    off = np.asarray(batch.peak_off, np.uint64)
    mz = (np.asarray(batch.masses, np.float32) + PROTON).astype(np.float32)
    it = np.asarray(batch.intensities, np.float32).copy()
    mob = None if batch.mobilities is None else np.asarray(batch.mobilities, np.float32).copy()
    if shuffle:
        rng = np.random.default_rng(seed)
        perm = np.arange(len(mz))
        for s in range(len(off) - 1):
            a, b = int(off[s]), int(off[s + 1])
            perm[a:b] = a + rng.permutation(b - a)
        mz, it = mz[perm], it[perm]
        mob = None if mob is None else mob[perm]
    n = len(off) - 1
    return RawSpectra(off.copy(), mz, it, np.ones(n, np.uint8), None, mob, np.asarray(batch.file_id, np.uint32).copy(),
                      np.asarray(batch.scan_start_time, np.float32).copy())


def write_mgf(batch: SpectraBatch, title: str = "synth", rt=None) -> bytes:
    """A SpectraBatch as MGF text: one record per spectrum with TITLE, PEPMASS (precursor m/z), CHARGE, RTINSECONDS (when rt is given, f32
    seconds) and one "mz intensity" line per peak. Every f32 is written in its shortest round-trip form, so MgfReader::parse reads the
    arrays back bit for bit."""
    n = len(batch)
    off = np.asarray(batch.peak_off, np.int64)
    mz = np.asarray(batch.masses, np.float32).astype("U")
    it = np.asarray(batch.intensities, np.float32).astype("U")
    pmz = np.asarray(batch.prec_mz, np.float32).astype("U")
    rts = None if rt is None else np.asarray(rt, np.float32).astype("U")
    peaks = np.char.add(np.char.add(mz, " "), it)
    out = []
    for s in range(n):
        head = f"BEGIN IONS\nTITLE={title}.{s}\nPEPMASS={pmz[s]}\nCHARGE={int(batch.prec_charge[s])}+\n"
        if rts is not None:
            head += f"RTINSECONDS={rts[s]}\n"
        out.append(head + "\n".join(peaks[off[s] - off[0]:off[s + 1] - off[0]].tolist()) + "\nEND IONS\n")
    return "".join(out).encode()
