"""Python mirror of the reference interface for the hot path, bound to libsage_b200.so through the C ABI
(include/sage_b200.h) with ctypes. Names and argument meaning follow sage-core:

    Tolerance          crates/sage/src/mass.rs:10-16
    Precursor / ProcessedSpectrum   crates/sage/src/spectrum.rs:47-79
    IndexedDatabase    crates/sage/src/database.rs:384-395   (device-resident here)
    Scorer             crates/sage/src/scoring.rs:210-232    (.score(spectrum) -> [Feature], plus .score_batch)

There is no CPU fallback: loading fails if the CUDA library is missing and every call fails if no GPU is present.
"""
from __future__ import annotations

import ctypes as C
import os
import time
from dataclasses import dataclass, field

import numpy as np

from .build import build_library, library_path

PPM, PCT, DA = 0, 1, 2
KIND = {"a": 0, "b": 1, "c": 2, "x": 3, "y": 4, "z": 5}


class SageB200Error(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"sage_b200 error {code}: {message}")
        self.code = code
        self.message = message


# ------------------------------------------------------------------------------------------------ C structs
class CTol(C.Structure):
    _fields_ = [("kind", C.c_int32), ("lo", C.c_float), ("hi", C.c_float)]


class CPeptides(C.Structure):
    _fields_ = [("n_peptides", C.c_uint64), ("residue_offsets", C.c_void_p), ("sequence", C.c_void_p), ("modifications", C.c_void_p),
                ("nterm", C.c_void_p), ("monoisotopic", C.c_void_p), ("decoy", C.c_void_p), ("missed_cleavages", C.c_void_p)]


class CIndex(C.Structure):
    _fields_ = [("n_fragments", C.c_uint64), ("fragment_peptide", C.c_void_p), ("fragment_mz", C.c_void_p), ("n_buckets", C.c_uint64),
                ("bucket_min", C.c_void_p), ("bucket_size", C.c_uint64), ("ion_kinds", C.c_void_p), ("n_ion_kinds", C.c_uint64)]


class CDbInfo(C.Structure):
    _fields_ = [("n_peptides", C.c_uint64), ("n_fragments", C.c_uint64), ("n_buckets", C.c_uint64), ("bucket_size", C.c_uint64),
                ("n_ion_kinds", C.c_uint64), ("total_residues", C.c_uint64), ("device_bytes", C.c_uint64), ("device", C.c_int32)]


class CScorerParams(C.Structure):
    _fields_ = [("precursor_tol", CTol), ("fragment_tol", CTol), ("min_matched_peaks", C.c_uint16), ("min_isotope_err", C.c_int8),
                ("max_isotope_err", C.c_int8), ("min_precursor_charge", C.c_uint8), ("max_precursor_charge", C.c_uint8),
                ("override_precursor_charge", C.c_uint8), ("max_fragment_charge", C.c_int8), ("chimera", C.c_uint8), ("wide_window", C.c_uint8),
                ("annotate_matches", C.c_uint8), ("score_type", C.c_uint8), ("report_psms", C.c_uint32)]


class CSpectra(C.Structure):
    _fields_ = [("n", C.c_uint64), ("peak_offsets", C.c_void_p), ("masses", C.c_void_p), ("intensities", C.c_void_p), ("precursor_mz", C.c_void_p),
                ("precursor_charge", C.c_void_p), ("isolation_lo", C.c_void_p), ("isolation_hi", C.c_void_p), ("total_ion_current", C.c_void_p),
                ("level", C.c_void_p), ("scan_start_time", C.c_void_p), ("inverse_ion_mobility", C.c_void_p)]


COUNTER_U64 = ["spectra", "peaks", "queries", "tasks", "pages", "entries_scanned", "matched_fragments", "candidates_scored", "peptide_record_floats",
               "psms", "wide_queries", "pep_queries", "pep_fallbacks", "wide_overflows", "algorithmic_bytes", "prelim_bytes", "score_bytes", "h2d_bytes", "d2h_bytes", "kernel_launches", "chunk_retries"]
COUNTER_F32 = ["ms_total", "ms_h2d", "ms_setup", "ms_prelim", "ms_score", "ms_d2h", "ms_prelim_count", "ms_wall"]


class CCounters(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in COUNTER_U64] + [(n, C.c_float) for n in COUNTER_F32]


# layout == sage_b200_feature (include/sage_b200.h)
FEATURE_DTYPE = np.dtype([
    ("spectrum", "<u4"), ("peptide_idx", "<u4"), ("peptide_len", "<u4"), ("rank", "<u4"), ("label", "<i4"), ("expmass", "<f4"), ("calcmass", "<f4"),
    ("charge", "<u4"), ("rt", "<f4"), ("ims", "<f4"), ("delta_mass", "<f4"), ("isotope_error", "<f4"), ("average_ppm", "<f4"), ("_pad0", "<u4"),
    ("hyperscore", "<f8"), ("delta_next", "<f8"), ("delta_best", "<f8"), ("matched_peaks", "<u4"), ("longest_b", "<u4"), ("longest_y", "<u4"),
    ("longest_y_pct", "<f4"), ("missed_cleavages", "<u4"), ("matched_intensity_pct", "<f4"), ("scored_candidates", "<u4"), ("ms2_intensity", "<f4"),
    ("poisson", "<f8"), ("fragment_offset", "<u4"), ("fragment_count", "<u4"),
])
assert FEATURE_DTYPE.itemsize == 128
FRAGMENT_DTYPE = np.dtype([("kind", "<i4"), ("charge", "<i4"), ("ordinal", "<i4"), ("intensity", "<f4"), ("mz_calculated", "<f4"),
                           ("mz_experimental", "<f4")])

EXPORTED_SYMBOLS = [
    "sage_b200_device_count", "sage_b200_db_create", "sage_b200_db_build", "sage_b200_db_get_info", "sage_b200_db_export_index", "sage_b200_db_destroy",
    "sage_b200_scorer_create", "sage_b200_scorer_destroy", "sage_b200_scorer_set_option", "sage_b200_score_batch", "sage_b200_batch_upload", "sage_b200_batch_run",
    "sage_b200_batch_download", "sage_b200_score_batch_multi", "sage_b200_quick_score", "sage_b200_initial_hits", "sage_b200_counters_get",
    "sage_b200_process_spectra", "sage_b200_find_reporter_ions", "sage_b200_host_alloc", "sage_b200_host_free", "sage_b200_last_error",
    "sage_b200_host_log_variant", "sage_b200_host_log1pf_exact", "sage_b200_device_log", "sage_b200_bind_thread_to_device", "sage_b200_host_alloc_blocks",
    "sage_b200_lfq_create", "sage_b200_lfq_add_ms1", "sage_b200_lfq_integrate", "sage_b200_lfq_get_info", "sage_b200_lfq_export", "sage_b200_lfq_destroy",
    "sage_b200_spectrum_fdr", "sage_b200_kde_build", "sage_b200_device_math", "sage_b200_predict_rt",
    "sage_b200_picked_fdr", "sage_b200_picked_precursor", "sage_b200_competition_keys", "sage_b200_protein_groups", "sage_b200_bipartite_cover",
    "sage_b200_digest_create", "sage_b200_digest_get_info", "sage_b200_digest_export", "sage_b200_digest_destroy",
    "sage_b200_prefilter_create", "sage_b200_prefilter_get_info", "sage_b200_prefilter_chunk_counts", "sage_b200_prefilter_export",
    "sage_b200_prefilter_take_db", "sage_b200_prefilter_destroy", "sage_b200_process_raw", "sage_b200_lfq_add_raw_ms1",
    "sage_b200_write_tsv", "sage_b200_format_hashes",
    "sage_b200_mgf_create", "sage_b200_mgf_get_info", "sage_b200_mgf_export", "sage_b200_mgf_process", "sage_b200_mgf_destroy", "sage_b200_parse_f32",
]

_lib = None


def load_library(build: bool = True):
    """Loads the in-tree CUDA library. Raises (never falls back) if it cannot be built/loaded."""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.exists(path):
        if not build:
            raise FileNotFoundError(f"{path} not built; run `python -m sage_b200.build`")
        build_library()
    lib = C.CDLL(path)
    for s in EXPORTED_SYMBOLS:
        getattr(lib, s)
    lib.sage_b200_host_alloc.restype = C.c_void_p
    lib.sage_b200_host_alloc.argtypes = [C.c_size_t]
    lib.sage_b200_host_free.argtypes = [C.c_void_p]
    lib.sage_b200_host_alloc_blocks.restype = C.c_void_p
    lib.sage_b200_host_alloc_blocks.argtypes = [C.c_size_t, C.c_void_p, C.c_int]
    lib.sage_b200_last_error.restype = C.c_size_t
    lib.sage_b200_initial_hits.restype = C.c_int64
    lib.sage_b200_db_destroy.argtypes = [C.c_void_p]
    lib.sage_b200_scorer_destroy.argtypes = [C.c_void_p]
    lib.sage_b200_lfq_destroy.argtypes = [C.c_void_p]
    lib.sage_b200_digest_destroy.argtypes = [C.c_void_p]
    lib.sage_b200_prefilter_destroy.argtypes = [C.c_void_p]
    lib.sage_b200_mgf_destroy.argtypes = [C.c_void_p]
    _lib = lib
    return lib


def _last_error() -> str:
    buf = C.create_string_buffer(2048)
    load_library().sage_b200_last_error(buf, C.c_size_t(2048))
    return buf.value.decode(errors="replace")


def _check(rc: int):
    if rc != 0:
        raise SageB200Error(int(rc), _last_error())


def device_count() -> int:
    return int(load_library().sage_b200_device_count())


def bind_thread_to_device(device: int) -> int:
    """Pins the calling thread to the CPUs of the GPU's NUMA node (-1: topology unknown, nothing changed)."""
    return int(load_library().sage_b200_bind_thread_to_device(C.c_int(device)))


def host_log_variant() -> int:
    """Which build of glibc's log() the host libm is (0 FMA-contracted, 1 plain, -1 unknown); the kernels reproduce that one (glibc_log.cuh)."""
    return int(load_library().sage_b200_host_log_variant())


def host_log1pf_exact() -> bool:
    """True when the host libm's log1pf is the function the kernels reproduce for the OpenMS score type."""
    return bool(load_library().sage_b200_host_log1pf_exact())


def device_log(x: np.ndarray, variant: int, device: int = 0) -> np.ndarray:
    """The device's evaluation of f64 log for every x (test hook for the glibc log() emulation)."""
    x = np.ascontiguousarray(x, np.float64)
    out = np.zeros_like(x)
    _check(load_library().sage_b200_device_log(C.c_int(device), C.c_int(variant), _ptr(x), C.c_uint64(len(x)), _ptr(out)))
    return out


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def pinned_empty(shape, dtype) -> np.ndarray:
    """numpy array backed by page-locked memory from sage_b200_host_alloc (release with pinned_free)."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) * dtype.itemsize
    p = load_library().sage_b200_host_alloc(C.c_size_t(max(n, 16)))
    if not p:
        raise SageB200Error(-2, _last_error())
    buf = (C.c_ubyte * max(n, 16)).from_address(p)
    arr = np.frombuffer(buf, dtype=np.uint8, count=n).view(dtype).reshape(shape)
    _PINNED[arr.ctypes.data] = p
    return arr


def pinned_empty_blocks(shape, dtype, devices) -> np.ndarray:
    """Page-locked array whose i-th of len(devices) equal parts sits on the NUMA node next to devices[i] (sage_b200_host_alloc_blocks): the
    input / output buffers of a score_batch_multi call."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) * dtype.itemsize
    dev = (C.c_int * len(devices))(*[int(d) for d in devices])
    p = load_library().sage_b200_host_alloc_blocks(C.c_size_t(max(n, 16)), dev, C.c_int(len(devices)))
    if not p:
        raise SageB200Error(-2, _last_error())
    buf = (C.c_ubyte * max(n, 16)).from_address(p)
    arr = np.frombuffer(buf, dtype=np.uint8, count=n).view(dtype).reshape(shape)
    _PINNED[arr.ctypes.data] = p
    return arr


_PINNED: dict = {}


def pinned_free(arr: np.ndarray):
    p = _PINNED.pop(arr.ctypes.data, None)
    if p is not None:
        load_library().sage_b200_host_free(C.c_void_p(p))


# ------------------------------------------------------------------------------------------------ reference-shaped types
@dataclass(frozen=True)
class Tolerance:
    """mass.rs:10-16. Tolerance.ppm(-10, 10) / .da(-500, 100) / .pct(..)."""
    kind: int
    lo: float
    hi: float

    @staticmethod
    def ppm(lo, hi):
        return Tolerance(PPM, float(lo), float(hi))

    @staticmethod
    def da(lo, hi):
        return Tolerance(DA, float(lo), float(hi))

    @staticmethod
    def pct(lo, hi):
        return Tolerance(PCT, float(lo), float(hi))

    def as_tuple(self):
        return (self.kind, self.lo, self.hi)

    def _c(self):
        return CTol(self.kind, self.lo, self.hi)


@dataclass
class Precursor:
    """spectrum.rs:47-55"""
    mz: float = 0.0
    charge: int | None = None
    isolation_window: Tolerance | None = None
    inverse_ion_mobility: float | None = None


@dataclass
class ProcessedSpectrum:
    """spectrum.rs:58-79"""
    level: int = 2
    id: str = ""
    file_id: int = 0
    scan_start_time: float = 0.0
    precursors: list = field(default_factory=list)
    masses: np.ndarray = field(default_factory=lambda: np.zeros(0, np.float32))
    intensities: np.ndarray = field(default_factory=lambda: np.zeros(0, np.float32))
    total_ion_current: float = 0.0


@dataclass
class SpectraBatch:
    """&[ProcessedSpectrum] flattened to the SoA the C ABI takes (sage_b200_spectra)."""
    peak_off: np.ndarray
    masses: np.ndarray
    intensities: np.ndarray
    prec_mz: np.ndarray
    prec_charge: np.ndarray
    iso_lo: np.ndarray
    iso_hi: np.ndarray
    tic: np.ndarray
    level: np.ndarray | None = None
    rt: np.ndarray | None = None
    ims: np.ndarray | None = None

    def __len__(self):
        return len(self.prec_mz)

    @staticmethod
    def from_spectra(spectra) -> "SpectraBatch":
        n = len(spectra)
        off = np.zeros(n + 1, np.uint64)
        for i, s in enumerate(spectra):
            off[i + 1] = off[i] + len(s.masses)
        masses = np.concatenate([np.asarray(s.masses, np.float32) for s in spectra]) if n else np.zeros(0, np.float32)
        intens = np.concatenate([np.asarray(s.intensities, np.float32) for s in spectra]) if n else np.zeros(0, np.float32)
        pmz, chg = np.full(n, np.nan, np.float32), np.zeros(n, np.uint8)
        ilo, ihi, ims = np.full(n, np.nan, np.float32), np.full(n, np.nan, np.float32), np.full(n, np.nan, np.float32)
        for i, s in enumerate(spectra):
            if s.precursors:
                p = s.precursors[0]
                pmz[i] = p.mz
                chg[i] = p.charge or 0
                if p.isolation_window is not None:
                    assert p.isolation_window.kind == DA
                    ilo[i], ihi[i] = p.isolation_window.lo, p.isolation_window.hi
                if p.inverse_ion_mobility is not None:
                    ims[i] = p.inverse_ion_mobility
        return SpectraBatch(off, masses, intens, pmz, chg, ilo, ihi, np.array([s.total_ion_current for s in spectra], np.float32),
                            np.array([s.level for s in spectra], np.uint8), np.array([s.scan_start_time for s in spectra], np.float32), ims)

    def as_dict(self) -> dict:
        return dict(peak_off=self.peak_off, masses=self.masses, intensities=self.intensities, prec_mz=self.prec_mz, prec_charge=self.prec_charge,
                    iso_lo=self.iso_lo, iso_hi=self.iso_hi, tic=self.tic, level=self.level, ims=self.ims)

    def slice(self, a: int, b: int) -> "SpectraBatch":
        p0, p1 = int(self.peak_off[a]), int(self.peak_off[b])
        opt = lambda x: None if x is None else x[a:b]  # noqa: E731
        return SpectraBatch(self.peak_off[a:b + 1] - self.peak_off[a], self.masses[p0:p1], self.intensities[p0:p1], self.prec_mz[a:b],
                            self.prec_charge[a:b], self.iso_lo[a:b], self.iso_hi[a:b], self.tic[a:b], opt(self.level), opt(self.rt), opt(self.ims))

    def _c(self, keep: list) -> CSpectra:
        def arr(x, dt):
            if x is None:
                return None
            a = np.ascontiguousarray(x, dtype=dt)
            keep.append(a)
            return _ptr(a)
        cs = CSpectra()
        cs.n = len(self)
        cs.peak_offsets = arr(self.peak_off, np.uint64)
        cs.masses = arr(self.masses, np.float32)
        cs.intensities = arr(self.intensities, np.float32)
        cs.precursor_mz = arr(self.prec_mz, np.float32)
        cs.precursor_charge = arr(self.prec_charge, np.uint8)
        cs.isolation_lo = arr(self.iso_lo, np.float32)
        cs.isolation_hi = arr(self.iso_hi, np.float32)
        cs.total_ion_current = arr(self.tic, np.float32)
        cs.level = arr(self.level, np.uint8)
        cs.scan_start_time = arr(self.rt, np.float32)
        cs.inverse_ion_mobility = arr(self.ims, np.float32)
        return cs


@dataclass
class Peptides:
    """The Peptide fields the hot path reads (peptide.rs:13-31), flattened. Row index == PeptideIx."""
    seq_off: np.ndarray
    seq: np.ndarray
    mods: np.ndarray
    nterm: np.ndarray
    mono: np.ndarray
    decoy: np.ndarray
    missed: np.ndarray

    def __len__(self):
        return len(self.mono)

    def sequence(self, i: int) -> str:
        return bytes(self.seq[self.seq_off[i]:self.seq_off[i + 1]]).decode()

    def _c(self, keep: list) -> CPeptides:
        def arr(x, dt):
            a = np.ascontiguousarray(x, dtype=dt)
            keep.append(a)
            return _ptr(a)
        cp = CPeptides()
        cp.n_peptides = len(self.mono)
        cp.residue_offsets = arr(self.seq_off, np.uint32)
        cp.sequence = arr(self.seq, np.uint8)
        cp.modifications = arr(self.mods, np.float32)
        cp.nterm = arr(self.nterm, np.float32)
        cp.monoisotopic = arr(self.mono, np.float32)
        cp.decoy = arr(self.decoy, np.uint8)
        cp.missed_cleavages = arr(self.missed, np.uint8)
        return cp


def _kinds(ion_kinds):
    return np.array([KIND[k] if isinstance(k, str) else int(k) for k in ion_kinds], dtype=np.uint8)


class IndexedDatabase:
    """Device-resident IndexedDatabase (database.rs:384-395)."""

    def __init__(self, handle, peptides: Peptides):
        self._h = C.c_void_p(handle)
        self.peptides = peptides
        info = CDbInfo()
        _check(load_library().sage_b200_db_get_info(self._h, C.byref(info)))
        self.info = {k: getattr(info, k) for k, _ in CDbInfo._fields_}

    def device_bytes(self) -> int:
        """HBM held by the index right now, including the block-major copies scorers have built on first use."""
        info = CDbInfo()
        _check(load_library().sage_b200_db_get_info(self._h, C.byref(info)))
        return int(info.device_bytes)

    def __del__(self):
        try:
            if self._h:
                load_library().sage_b200_db_destroy(self._h)
                self._h = None
        except Exception:
            pass

    @staticmethod
    def from_reference_layout(peptides: Peptides, frag_pep, frag_mz, bucket_min, bucket_size, ion_kinds=("b", "y"), device=0) -> "IndexedDatabase":
        """Upload an index already built by the reference's Parameters::build (database.rs:260)."""
        keep: list = []
        cp = peptides._c(keep)
        ci = CIndex()
        fp = np.ascontiguousarray(frag_pep, np.uint32)
        fm = np.ascontiguousarray(frag_mz, np.float32)
        bm = np.ascontiguousarray(bucket_min, np.float32)
        kinds = _kinds(ion_kinds)
        ci.n_fragments, ci.fragment_peptide, ci.fragment_mz = len(fp), _ptr(fp), _ptr(fm)
        ci.n_buckets, ci.bucket_min, ci.bucket_size = len(bm), _ptr(bm), int(bucket_size)
        ci.ion_kinds, ci.n_ion_kinds = _ptr(kinds), len(kinds)
        h = C.c_void_p()
        _check(load_library().sage_b200_db_create(C.byref(cp), C.byref(ci), C.c_int(device), C.byref(h)))
        return IndexedDatabase(h.value, peptides)

    @staticmethod
    def build_from_peptides(peptides: Peptides, bucket_size=8192, ion_kinds=("b", "y"), min_ion_index=2, device=0) -> "IndexedDatabase":
        """Parameters::build_from_peptides (database.rs:265-365) executed on the device."""
        keep: list = []
        cp = peptides._c(keep)
        kinds = _kinds(ion_kinds)
        h = C.c_void_p()
        _check(load_library().sage_b200_db_build(C.byref(cp), C.c_uint64(int(bucket_size)), _ptr(kinds), C.c_uint64(len(kinds)),
                                                 C.c_uint64(int(min_ion_index)), C.c_int(device), C.byref(h)))
        return IndexedDatabase(h.value, peptides)

    @staticmethod
    def from_fasta(fasta, *, bucket_size=8192, ion_kinds=("b", "y"), min_ion_index=2, device=0, prefilter=False, spectra=None, scorer=None,
                   prefilter_chunk_size=0, prefilter_low_memory=True, min_peaks=15, **digest_args) -> "IndexedDatabase":
        """Builder::make_parameters + Parameters::build (database.rs:96-115, 260) from FASTA text: digest_fasta, then build_from_peptides on
        the digested table. `bucket_size` is rounded up to a power of two. The digest result stays on the db as `.digest` (protein lists,
        cterm, semi_enzymatic for picked_fdr, protein_groups and the writers).
        prefilter=True: the database prefilter of runner.rs:104-128 (prefilter_fasta) with `spectra` (a SpectraBatch) and `scorer` (a dict of
        the Scorer keywords, precursor_tol and fragment_tol required); `.digest` is then the PrefilterResult."""
        if prefilter:
            if spectra is None or scorer is None:
                raise ValueError("prefilter=True needs spectra and scorer")
            r = prefilter_fasta(fasta, spectra, bucket_size=bucket_size, ion_kinds=ion_kinds, min_ion_index=min_ion_index, device=device,
                                prefilter_chunk_size=prefilter_chunk_size, prefilter_low_memory=prefilter_low_memory, min_peaks=min_peaks,
                                **dict(scorer), **digest_args)
            r.db.digest = r
            return r.db
        if isinstance(bucket_size, bool) or not isinstance(bucket_size, (int, np.integer)) or not 1 <= int(bucket_size) <= 1 << 30:
            raise ValueError(f"bucket_size must be an integer in 1..2^30, got {bucket_size!r}")
        bs = 1 << (int(bucket_size) - 1).bit_length()
        d = digest_fasta(fasta, device=device, **digest_args)
        db = IndexedDatabase.build_from_peptides(d.peptides, bucket_size=bs, ion_kinds=ion_kinds, min_ion_index=min_ion_index, device=device)
        db.digest = d
        return db

    def export_index(self):
        nf, nb = self.info["n_fragments"], self.info["n_buckets"]
        fp, fm, bm = np.empty(nf, np.uint32), np.empty(nf, np.float32), np.empty(nb, np.float32)
        _check(load_library().sage_b200_db_export_index(self._h, _ptr(fp), _ptr(fm), _ptr(bm)))
        return fp, fm, bm


class Scorer:
    """Scorer (scoring.rs:210-232): same public fields; `db` is a device-resident IndexedDatabase."""

    def __init__(self, db: IndexedDatabase, precursor_tol: Tolerance, fragment_tol: Tolerance, min_matched_peaks=4, min_isotope_err=0,
                 max_isotope_err=0, min_precursor_charge=2, max_precursor_charge=4, override_precursor_charge=False, max_fragment_charge=None,
                 chimera=False, report_psms=1, wide_window=False, annotate_matches=False, score_type=0):
        self.db = db
        self.report_psms = int(report_psms)
        self.fragment_capacity = None   # annotate_matches: size of the fragments array (default: generous estimate)
        self.last_fragments = None      # Fragments rows of the last score_batch (Feature.fragment_offset/count index into it)
        p = CScorerParams()
        p.precursor_tol, p.fragment_tol = precursor_tol._c(), fragment_tol._c()
        p.min_matched_peaks = min_matched_peaks
        p.min_isotope_err, p.max_isotope_err = min_isotope_err, max_isotope_err
        p.min_precursor_charge, p.max_precursor_charge = min_precursor_charge, max_precursor_charge
        p.override_precursor_charge = int(override_precursor_charge)
        p.max_fragment_charge = -1 if max_fragment_charge is None else int(max_fragment_charge)
        p.chimera, p.wide_window, p.annotate_matches = int(chimera), int(wide_window), int(annotate_matches)
        p.score_type = int(score_type)
        p.report_psms = self.report_psms
        self._params = p
        h = C.c_void_p()
        _check(load_library().sage_b200_scorer_create(db._h, C.byref(p), C.byref(h)))
        self._h = h

    def set_option(self, name: str, value: int):
        _check(load_library().sage_b200_scorer_set_option(self._h, name.encode(), C.c_int64(int(value))))

    def __del__(self):
        try:
            if self._h:
                load_library().sage_b200_scorer_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def score_batch(self, batch: SpectraBatch, out: np.ndarray | None = None, counts: np.ndarray | None = None):
        """`spectra.par_iter().flat_map(|s| scorer.score(s))` (runner.rs:311-325). Returns (features[n*report_psms], counts[n])."""
        n = len(batch)
        if out is None:
            out = np.zeros(n * self.report_psms, FEATURE_DTYPE)
        if counts is None:
            counts = np.zeros(n, np.uint32)
        keep: list = []
        cs = batch._c(keep)
        used = C.c_uint64(0)
        if self._params.annotate_matches:
            cap = int(self.fragment_capacity or (n * self.report_psms * 128 + 1024))
            frags = np.zeros(cap, FRAGMENT_DTYPE)
            _check(load_library().sage_b200_score_batch(self._h, C.byref(cs), _ptr(out), _ptr(counts), _ptr(frags), C.c_uint64(cap), C.byref(used)))
            self.last_fragments = frags[:used.value]
            return out, counts
        _check(load_library().sage_b200_score_batch(self._h, C.byref(cs), _ptr(out), _ptr(counts), None, C.c_uint64(0), C.byref(used)))
        return out, counts

    # device-resident phases of score_batch (one chunk): upload once, run many times, download
    def upload(self, batch: SpectraBatch):
        keep: list = []
        cs = batch._c(keep)
        self._resident_n = len(batch)
        _check(load_library().sage_b200_batch_upload(self._h, C.byref(cs)))

    def run(self):
        _check(load_library().sage_b200_batch_run(self._h))

    def download(self, out: np.ndarray | None = None, counts: np.ndarray | None = None):
        n = self._resident_n
        if out is None:
            out = np.zeros(n * self.report_psms, FEATURE_DTYPE)
        if counts is None:
            counts = np.zeros(n, np.uint32)
        _check(load_library().sage_b200_batch_download(self._h, _ptr(out), _ptr(counts)))
        return out, counts

    def quick_score(self, batch: SpectraBatch, prefilter_low_memory: bool, keep: np.ndarray | None = None) -> np.ndarray:
        """Scorer::quick_score (scoring.rs:255-298) over a batch: keep[PeptideIx] (uint8) is OR-ed and returned."""
        if keep is None:
            keep = np.zeros(self.db.info["n_peptides"], np.uint8)
        keep_c = np.ascontiguousarray(keep, dtype=np.uint8)
        kl: list = []
        cs = batch._c(kl)
        _check(load_library().sage_b200_quick_score(self._h, C.byref(cs), C.c_int(int(prefilter_low_memory)), _ptr(keep_c)))
        return keep_c

    def score(self, spectrum: ProcessedSpectrum):
        """Scorer::score (scoring.rs:300): one spectrum -> list of Feature rows."""
        out, counts = self.score_batch(SpectraBatch.from_spectra([spectrum]))
        return out[:counts[0]]

    def initial_hits(self, batch: SpectraBatch):
        assert len(batch) == 1
        cap = 256
        m, p = np.zeros(cap, np.uint16), np.zeros(cap, np.uint32)
        c, i = np.zeros(cap, np.uint8), np.zeros(cap, np.int8)
        mp, scd = C.c_uint64(0), C.c_uint64(0)
        keep: list = []
        cs = batch._c(keep)
        n = load_library().sage_b200_initial_hits(self._h, C.byref(cs), _ptr(m), _ptr(p), _ptr(c), _ptr(i), C.c_uint64(cap), C.byref(mp), C.byref(scd))
        if n < 0:
            raise SageB200Error(int(n), _last_error())
        return dict(matched=m[:n].copy(), peptide=p[:n].copy(), charge=c[:n].copy(), iso=i[:n].copy(), matched_peaks=mp.value, scored_candidates=scd.value)

    def counters(self) -> dict:
        cc = CCounters()
        _check(load_library().sage_b200_counters_get(self._h, C.byref(cc)))
        return {k: getattr(cc, k) for k, _ in CCounters._fields_}


def score_batch_multi(scorers, batch: SpectraBatch, out: np.ndarray | None = None, counts: np.ndarray | None = None):
    """sage_b200_score_batch_multi: one process, one Scorer per GPU (same settings), spectra split into contiguous blocks."""
    n, r = len(batch), scorers[0].report_psms
    if out is None:
        out = np.zeros(n * r, FEATURE_DTYPE)
    if counts is None:
        counts = np.zeros(n, np.uint32)
    keep: list = []
    cs = batch._c(keep)
    arr = (C.c_void_p * len(scorers))(*[s._h for s in scorers])
    _check(load_library().sage_b200_score_batch_multi(arr, C.c_int(len(scorers)), C.byref(cs), _ptr(out), _ptr(counts)))
    return out, counts


class CProcessorParams(C.Structure):
    _fields_ = [("take_top_n", C.c_uint64), ("deisotope", C.c_uint8), ("min_deisotope_mz", C.c_float)]


class CRawSpectra(C.Structure):
    _fields_ = [("n", C.c_uint64), ("peak_offsets", C.c_void_p), ("mz", C.c_void_p), ("intensity", C.c_void_p), ("precursor_charge", C.c_void_p),
                ("level", C.c_void_p)]


class SpectrumProcessor:
    """SpectrumProcessor::new(take_top_n, deisotope, min_deisotope_mz) (spectrum.rs:271); process() runs on the device."""

    def __init__(self, take_top_n: int, deisotope: bool, min_deisotope_mz: float, device: int = 0):
        self.take_top_n, self.deisotope, self.min_deisotope_mz, self.device = int(take_top_n), bool(deisotope), float(min_deisotope_mz), device

    def process_batch(self, peak_off, mz, intensity, precursor_charge):
        """Raw centroided MS2 spectra (CSR) -> (peak_off[n+1], masses, intensities, tic[n]) of the ProcessedSpectrum batch."""
        peak_off = np.ascontiguousarray(peak_off, np.uint64)
        mz, intensity = np.ascontiguousarray(mz, np.float32), np.ascontiguousarray(intensity, np.float32)
        chg = np.ascontiguousarray(precursor_charge, np.uint8)
        n = len(chg)
        pp = CProcessorParams(self.take_top_n, int(self.deisotope), self.min_deisotope_mz)
        raw = CRawSpectra(n, _ptr(peak_off), _ptr(mz), _ptr(intensity), _ptr(chg), None)
        out_off = np.zeros(n + 1, np.uint64)
        om, oi, tic = np.zeros(max(1, len(mz)), np.float32), np.zeros(max(1, len(mz)), np.float32), np.zeros(n, np.float32)
        _check(load_library().sage_b200_process_spectra(C.c_int(self.device), C.byref(pp), C.byref(raw), _ptr(out_off), _ptr(om), _ptr(oi), _ptr(tic)))
        k = int(out_off[-1])
        return out_off, om[:k].copy(), oi[:k].copy(), tic

    def process_raw(self, batch: "RawSpectra") -> "ProcessedBatch":
        """process() (spectrum.rs:338-412) of a batch of any MS levels: level 2 as process_batch, other levels keep every peak, sorted."""
        keep: list = []
        raw = batch._c(keep)
        n = len(batch)
        npk = max(1, int(batch.peak_off[-1] - batch.peak_off[0])) if n else 1
        pp = CProcessorParams(self.take_top_n, int(self.deisotope), self.min_deisotope_mz)
        out_off = np.zeros(n + 1, np.uint64)
        om, oi, ob, tic = np.zeros(npk, np.float32), np.zeros(npk, np.float32), np.zeros(npk, np.float32), np.zeros(n, np.float32)
        _check(load_library().sage_b200_process_raw(C.c_int(self.device), C.byref(pp), C.byref(raw), _ptr(out_off), _ptr(om), _ptr(oi), _ptr(ob),
                                                    _ptr(tic)))
        k = int(out_off[-1])
        level = np.ascontiguousarray(batch.level, np.uint8).copy()
        return ProcessedBatch(out_off, om[:k].copy(), oi[:k].copy(), ob[:k].copy(), (level == 1) & (batch.mobility is not None), tic, level)


class CRawBatch(C.Structure):
    _fields_ = [("n", C.c_uint64), ("peak_offsets", C.c_void_p), ("mz", C.c_void_p), ("intensity", C.c_void_p), ("level", C.c_void_p),
                ("precursor_charge", C.c_void_p), ("mobility", C.c_void_p)]


class CRawMs1(C.Structure):
    _fields_ = [("n", C.c_uint64), ("peak_offsets", C.c_void_p), ("mz", C.c_void_p), ("intensity", C.c_void_p), ("file_id", C.c_void_p),
                ("scan_start_time", C.c_void_p), ("mobility", C.c_void_p)]


def _keep_arr(keep: list, x, dt):
    if x is None:
        return None
    a = np.ascontiguousarray(x, dtype=dt)
    keep.append(a)
    return _ptr(a)


@dataclass
class RawSpectra:
    """A batch of RawSpectrum (spectrum.rs:81-106) of any MS levels, flattened: peaks in any order. precursor_charge (0 = None) is read for
    level 2 only; mobility (per peak) may be None: then no spectrum of the batch has mobility. file_id and scan_start_time are needed by
    FeatureMap.add_raw_ms1 only."""
    peak_off: np.ndarray
    mz: np.ndarray
    intensity: np.ndarray
    level: np.ndarray
    precursor_charge: np.ndarray | None = None
    mobility: np.ndarray | None = None
    file_id: np.ndarray | None = None
    scan_start_time: np.ndarray | None = None

    def __len__(self):
        return len(self.level)

    def slice(self, a: int, b: int) -> "RawSpectra":
        p0, p1 = int(self.peak_off[a]), int(self.peak_off[b])
        cut = (lambda x, lo, hi: None if x is None else x[lo:hi])
        return RawSpectra(self.peak_off[a:b + 1] - self.peak_off[a], self.mz[p0:p1], self.intensity[p0:p1], self.level[a:b],
                          cut(self.precursor_charge, a, b), cut(self.mobility, p0, p1), cut(self.file_id, a, b), cut(self.scan_start_time, a, b))

    def _c(self, keep: list) -> CRawBatch:
        return CRawBatch(len(self), _keep_arr(keep, self.peak_off, np.uint64), _keep_arr(keep, self.mz, np.float32),
                         _keep_arr(keep, self.intensity, np.float32), _keep_arr(keep, self.level, np.uint8),
                         _keep_arr(keep, self.precursor_charge, np.uint8), _keep_arr(keep, self.mobility, np.float32))


@dataclass
class ProcessedBatch:
    """A batch of ProcessedSpectrum (spectrum.rs:58-79) flattened. mobilities runs parallel to masses and is NaN for a spectrum whose
    ProcessedSpectrum::mobilities is empty (has_mobilities False: every level but 1, and level 1 without mobility)."""
    peak_off: np.ndarray
    masses: np.ndarray
    intensities: np.ndarray
    mobilities: np.ndarray
    has_mobilities: np.ndarray
    tic: np.ndarray
    level: np.ndarray

    def __len__(self):
        return len(self.level)


TMT6PLEX = np.float32([126.127726, 127.124761, 128.134436, 129.131471, 130.141145, 131.138180])   # tmt.rs:213-215
TMT11PLEX = np.float32([126.127726, 127.124761, 127.131081, 128.128116, 128.134436, 129.131471, 129.137790, 130.134825, 130.141145, 131.138180,
                        131.144499])   # tmt.rs:217-220
TMT18PLEX = np.float32([126.127726, 127.124761, 127.131081, 128.128116, 128.134436, 129.131471, 129.137790, 130.134825, 130.141145, 131.138180,
                        131.144500, 132.141535, 132.147855, 133.144890, 133.151210, 134.148245, 134.154565, 135.15160])   # tmt.rs:222-226
# Isobaric::reporter_masses (tmt.rs:24-34): Tmt10 is the first 10 of the 11-plex, Tmt16 the first 16 of the 18-plex
ISOBARIC = {"Tmt6": TMT6PLEX, "Tmt10": TMT11PLEX[:10].copy(), "Tmt11": TMT11PLEX, "Tmt16": TMT18PLEX[:16].copy(), "Tmt18": TMT18PLEX}


def tmt_min_deisotope_mz(isobaric: str, level: int) -> float:
    """runner.rs:398-404: with TMT at level 2, the last reporter mass * (1.0 + 20E-6), in f32; 0.0 otherwise (the unwrap_or(0.0))."""
    if level != 2:
        return 0.0
    return float(ISOBARIC[isobaric][-1] * (np.float32(1.0) + np.float32(20e-6)))


def tmt_quantify(processed: ProcessedBatch, isobaric: str, level: int, tolerance: Tolerance | None = None, device: int = 0):
    """tmt::quantify (tmt.rs:314-352): the spectra of `level` (none for level 1) and their reporter intensities through find_reporter_ions
    (0 where no peak is within tolerance, the unwrap_or_default). Returns (row indices into `processed`, float32 [rows, labels])."""
    labels = ISOBARIC[isobaric]
    tolerance = Tolerance.ppm(-20, 20) if tolerance is None else tolerance
    rows = np.nonzero(np.asarray(processed.level) == level)[0] if level != 1 else np.zeros(0, np.int64)
    if len(rows) == 0:
        return rows, np.zeros((0, len(labels)), np.float32)
    off = np.asarray(processed.peak_off, np.uint64)
    lens = (off[rows + 1] - off[rows]).astype(np.int64)
    sub_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    take = np.concatenate([np.arange(int(off[r]), int(off[r + 1])) for r in rows]) if lens.sum() else np.zeros(0, np.int64)
    return rows, find_reporter_ions(sub_off, processed.masses[take], processed.intensities[take], labels, tolerance, device)


def find_reporter_ions(peak_off, masses, intensities, labels, label_tolerance: Tolerance, device: int = 0) -> np.ndarray:
    """tmt::find_reporter_ions (tmt.rs:193-211) over a batch of ProcessedSpectrum -> float32 [n, n_labels]."""
    peak_off = np.ascontiguousarray(peak_off, np.uint64)
    masses, intensities, labels = (np.ascontiguousarray(x, np.float32) for x in (masses, intensities, labels))
    n = len(peak_off) - 1
    out = np.zeros((n, len(labels)), np.float32)
    _check(load_library().sage_b200_find_reporter_ions(C.c_int(device), C.c_uint64(n), _ptr(peak_off), _ptr(masses), _ptr(intensities), _ptr(labels),
                                                       C.c_uint64(len(labels)), label_tolerance._c(), _ptr(out)))
    return out


# ------------------------------------------------------------------------------------------------ label-free quantification (lfq.rs)
PEAK_SCORING = {"RetentionTime": 0, "SpectralAngle": 1, "Intensity": 2, "Hybrid": 3}   # PeakScoringStrategy, lfq.rs:25-31
INTEGRATION = {"Apex": 0, "Sum": 1}                                                   # IntegrationStrategy, lfq.rs:33-37


class CLfqParams(C.Structure):
    _fields_ = [("peak_scoring", C.c_int32), ("integration", C.c_int32), ("spectral_angle", C.c_double), ("ppm_tolerance", C.c_float),
                ("mobility_pct_tolerance", C.c_float), ("peptide_q_value", C.c_float), ("combine_charge_states", C.c_uint8),
                ("min_precursor_charge", C.c_uint8), ("max_precursor_charge", C.c_uint8)]


class CLfqFeatures(C.Structure):
    _fields_ = [("n", C.c_uint64), ("peptide_idx", C.c_void_p), ("peptide_q", C.c_void_p), ("label", C.c_void_p), ("aligned_rt", C.c_void_p),
                ("calcmass", C.c_void_p), ("file_id", C.c_void_p), ("ims", C.c_void_p)]


class CMs1(C.Structure):
    _fields_ = [("n", C.c_uint64), ("peak_offsets", C.c_void_p), ("masses", C.c_void_p), ("intensities", C.c_void_p), ("file_id", C.c_void_p),
                ("scan_start_time", C.c_void_p), ("mobilities", C.c_void_p)]


class CLfqInfo(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("n_peptides", "n_ranges", "n_pages", "n_grids", "n_files", "grids_touched", "ms1_spectra", "ms1_peaks",
                                          "contributions", "device_bytes")] + \
               [(n, C.c_float) for n in ("ms_build", "ms_trace", "ms_integrate", "ms_download")]


ALIGNMENT_DTYPE = np.dtype([("max_rt", "<f4"), ("slope", "<f4"), ("intercept", "<f4")])            # sage_b200_alignment
LFQ_RANGE_DTYPE = np.dtype([("rt", "<f4"), ("mass_lo", "<f4"), ("mass_hi", "<f4"), ("mobility_lo", "<f4"), ("mobility_hi", "<f4"),
                            ("peptide", "<u4"), ("file_id", "<u4"), ("charge", "u1"), ("isotope", "u1"), ("decoy", "u1"), ("_pad", "u1")])
LFQ_ROW_DTYPE = np.dtype([("peptide", "<u4"), ("charge", "u1"), ("decoy", "u1"), ("_pad0", "<u2"), ("rt", "<u4"), ("_pad1", "<u4"),
                          ("spectral_angle", "<f8"), ("score", "<f8")])                                 # sage_b200_lfq_row
LFQ_FEATURE_FIELDS = ("peptide_idx", "peptide_q", "label", "aligned_rt", "calcmass", "file_id", "ims")
_LFQ_FEATURE_TYPES = (np.uint32, np.float32, np.int32, np.float32, np.float32, np.uint32, np.float32)


@dataclass
class LfqSettings:
    """LfqSettings (lfq.rs:45-68), same defaults. peak_scoring / integration take the reference's variant names."""
    peak_scoring: str = "Hybrid"
    integration: str = "Sum"
    spectral_angle: float = 0.70
    ppm_tolerance: float = 5.0
    mobility_pct_tolerance: float = 1.0
    combine_charge_states: bool = True
    peptide_q_value: float = 0.01

    def _c(self, precursor_charge) -> CLfqParams:
        p = CLfqParams()
        p.peak_scoring, p.integration = PEAK_SCORING[self.peak_scoring], INTEGRATION[self.integration]
        p.spectral_angle, p.ppm_tolerance, p.mobility_pct_tolerance = self.spectral_angle, self.ppm_tolerance, self.mobility_pct_tolerance
        p.peptide_q_value, p.combine_charge_states = self.peptide_q_value, int(self.combine_charge_states)
        p.min_precursor_charge, p.max_precursor_charge = int(precursor_charge[0]), int(precursor_charge[1])
        return p


@dataclass
class Ms1Batch:
    """A batch of MS1 ProcessedSpectrum (spectrum.rs:58-79) flattened: masses are mz - PROTON, as SpectrumProcessor gives them.
    mobilities (per peak) may be None: then no spectrum of the batch has mobility."""
    peak_off: np.ndarray
    masses: np.ndarray
    intensities: np.ndarray
    file_id: np.ndarray
    scan_start_time: np.ndarray
    mobilities: np.ndarray | None = None

    def __len__(self):
        return len(self.file_id)

    def slice(self, a: int, b: int) -> "Ms1Batch":
        p0, p1 = int(self.peak_off[a]), int(self.peak_off[b])
        return Ms1Batch(self.peak_off[a:b + 1] - self.peak_off[a], self.masses[p0:p1], self.intensities[p0:p1], self.file_id[a:b], self.scan_start_time[a:b],
                        None if self.mobilities is None else self.mobilities[p0:p1])

    def _c(self, keep: list) -> CMs1:
        def arr(x, dt):
            if x is None:
                return None
            a = np.ascontiguousarray(x, dtype=dt)
            keep.append(a)
            return _ptr(a)
        return CMs1(len(self), arr(self.peak_off, np.uint64), arr(self.masses, np.float32), arr(self.intensities, np.float32), arr(self.file_id, np.uint32),
                    arr(self.scan_start_time, np.float32), arr(self.mobilities, np.float32))


def _lfq_features(features, keep: list) -> CLfqFeatures:
    cols = [np.ascontiguousarray(features[f], dtype=t) for f, t in zip(LFQ_FEATURE_FIELDS, _LFQ_FEATURE_TYPES)]
    keep.extend(cols)
    return CLfqFeatures(len(cols[0]), *[_ptr(c) for c in cols])


class FeatureMap:
    """build_feature_map(...) (lfq.rs:94-193) and FeatureMap::quantify (lfq.rs:226-304) on the device: build, add_ms1 any number of batches, quantify.
    `features` is a structured array or dict with the Feature fields peptide_idx, peptide_q, label, aligned_rt, calcmass, file_id, ims, in the
    caller's confidence order; `alignments` is ALIGNMENT_DTYPE (or [n_files, 3] float32: max_rt, slope, intercept)."""

    def __init__(self, handle, n_files: int, settings: LfqSettings, precursor_charge):
        self._h = C.c_void_p(handle)
        self.n_files = n_files
        self.settings = settings
        self.precursor_charge = tuple(precursor_charge)

    @staticmethod
    def build(db: IndexedDatabase, peptides: Peptides, settings: LfqSettings, precursor_charge, features, alignments) -> "FeatureMap":
        keep: list = []
        cp = peptides._c(keep)
        cf = _lfq_features(features, keep)
        al = np.ascontiguousarray(alignments)
        al = al.view(np.float32).reshape(-1, 3) if al.dtype.names else np.ascontiguousarray(al, np.float32).reshape(-1, 3)
        al = np.ascontiguousarray(al)
        params = settings._c(precursor_charge)
        h = C.c_void_p()
        _check(load_library().sage_b200_lfq_create(db._h, C.byref(cp), C.byref(params), C.byref(cf), C.c_uint64(len(al)), _ptr(al), C.byref(h)))
        return FeatureMap(h.value, len(al), settings, precursor_charge)

    def __del__(self):
        try:
            if self._h:
                load_library().sage_b200_lfq_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def add_ms1(self, batch: Ms1Batch):
        """The tracing loop of quantify (lfq.rs:239-287) over one batch."""
        keep: list = []
        cm = batch._c(keep)
        _check(load_library().sage_b200_lfq_add_ms1(self._h, C.byref(cm)))

    def add_raw_ms1(self, batch: RawSpectra):
        """add_ms1 of process() of a batch of raw MS1 spectra (file_id and scan_start_time set): processed and traced on the device."""
        if len(batch) and not (np.asarray(batch.level) == 1).all():
            raise ValueError("add_raw_ms1 takes MS1 spectra only")
        keep: list = []
        cr = CRawMs1(len(batch), _keep_arr(keep, batch.peak_off, np.uint64), _keep_arr(keep, batch.mz, np.float32), _keep_arr(keep, batch.intensity, np.float32),
                     _keep_arr(keep, batch.file_id, np.uint32), _keep_arr(keep, batch.scan_start_time, np.float32), _keep_arr(keep, batch.mobility, np.float32))
        _check(load_library().sage_b200_lfq_add_raw_ms1(self._h, C.byref(cr)))

    def info(self) -> dict:
        ci = CLfqInfo()
        _check(load_library().sage_b200_lfq_get_info(self._h, C.byref(ci)))
        return {k: getattr(ci, k) for k, _ in CLfqInfo._fields_}

    def quantify(self) -> dict:
        """summarize_traces + integrate for every traced precursor. Rows are ordered by (id, decoy): id is the PeptideIx, plus the charge when
        combine_charge_states is false (charge is 0 otherwise). Returns dict(id, charge, decoy, rt, spectral_angle, score, areas[n, n_files])."""
        cap = max(1, int(self.info()["n_grids"]))
        rows = np.zeros(cap, LFQ_ROW_DTYPE)
        areas = np.zeros((cap, self.n_files), np.float64)
        n = C.c_uint64(0)
        _check(load_library().sage_b200_lfq_integrate(self._h, _ptr(rows), _ptr(areas), C.c_uint64(cap), C.byref(n)))
        r = rows[:n.value]
        return dict(id=r["peptide"].copy(), charge=r["charge"].copy(), decoy=r["decoy"].astype(bool), rt=r["rt"].copy(),
                    spectral_angle=r["spectral_angle"].copy(), score=r["score"].copy(), areas=areas[:n.value].copy())

    def export(self, grids: bool = False) -> dict:
        """Test hook: the sorted ranges, min_rts and (grids=True) the raw grids [n_grids, n_files * 3, 100] with their touched flags."""
        info = self.info()
        ranges = np.zeros(info["n_ranges"], LFQ_RANGE_DTYPE)
        min_rts = np.zeros(info["n_pages"], np.float32)
        g = np.zeros((info["n_grids"], self.n_files * 3, 100), np.float64) if grids else None
        t = np.zeros(info["n_grids"], np.uint8) if grids else None
        _check(load_library().sage_b200_lfq_export(self._h, _ptr(ranges), _ptr(min_rts), _ptr(g), _ptr(t)))
        return dict(ranges=ranges, min_rts=min_rts, grids=g, touched=t)


Feature = FEATURE_DTYPE


# ------------------------------------------------------------------------------------------------ rescoring (spectrum_fdr)
class CFdrParams(C.Structure):
    _fields_ = [("precursor_tol", CTol)]


FDR_STAGES = ["ms_mass_kde", "ms_features", "ms_lda", "ms_discriminant_kde", "ms_sort_q", "ms_total"]


class CFdrOut(C.Structure):
    _fields_ = [("discriminant_score", C.c_void_p), ("posterior_error", C.c_void_p), ("spectrum_q", C.c_void_p), ("order", C.c_void_p),
                ("passing", C.c_uint64), ("lda_fitted", C.c_int32), ("coef", C.c_double * 20), ("eps", C.c_double)] + [(s, C.c_float) for s in FDR_STAGES]


def spectrum_fdr(features: np.ndarray, precursor_tol: Tolerance, aligned_rt=None, delta_rt_model=None, delta_ims_model=None, device: int = 0) -> dict:
    """The runner's spectrum_fdr (runner.rs:280-291) on the device: linear_discriminant::score_psms, the heuristic fallback when it fails, the
    descending sort and spectrum_q_value. `features` are FEATURE_DTYPE rows as Scorer.score_batch returns them; the three optional f32 columns
    default to the Feature defaults (aligned_rt = rt, 0.999). Returns discriminant_score, posterior_error, spectrum_q (indexed like the rows),
    order (row at each sorted position), passing, lda_fitted, coef, eps and the stage times (ms_*)."""
    rows = np.ascontiguousarray(features)
    if rows.dtype != FEATURE_DTYPE:
        raise TypeError("features must have FEATURE_DTYPE")
    n = len(rows)
    cols = [None if c is None else np.ascontiguousarray(c, np.float32) for c in (aligned_rt, delta_rt_model, delta_ims_model)]
    for c in cols:
        if c is not None and len(c) != n:
            raise ValueError("optional columns must have one value per row")
    res = dict(discriminant_score=np.zeros(n, np.float32), posterior_error=np.zeros(n, np.float32), spectrum_q=np.zeros(n, np.float32),
               order=np.zeros(n, np.uint32))
    out = CFdrOut(_ptr(res["discriminant_score"]), _ptr(res["posterior_error"]), _ptr(res["spectrum_q"]), _ptr(res["order"]))
    params = CFdrParams(precursor_tol._c())
    _check(load_library().sage_b200_spectrum_fdr(C.c_int(device), C.byref(params), _ptr(rows), C.c_uint64(n), *[_ptr(c) for c in cols], C.byref(out)))
    res.update(passing=int(out.passing), lda_fitted=bool(out.lda_fitted), coef=np.array(out.coef[:], np.float64), eps=float(out.eps))
    res.update({s: float(getattr(out, s)) for s in FDR_STAGES})
    return res


def kde_build(scores: np.ndarray, decoy: np.ndarray, bins: int = 1000, monotonic: bool = True, bw_factor: float = 1.0, device: int = 0):
    """kde::Builder::build (kde.rs:83-136) on the device with bw_adjust = x * bw_factor: (PEP per bin, min_score, score_step)."""
    s = np.ascontiguousarray(scores, np.float64)
    d = np.ascontiguousarray(decoy, np.uint8)
    out = np.zeros(int(bins), np.float64)
    lo, step = C.c_double(), C.c_double()
    _check(load_library().sage_b200_kde_build(C.c_int(device), _ptr(s), _ptr(d), C.c_uint64(len(s)), C.c_uint64(int(bins)), C.c_int(int(monotonic)),
                                              C.c_double(bw_factor), _ptr(out), C.byref(lo), C.byref(step)))
    return out, lo.value, step.value


MATH_FUNCTIONS = {"exp": 0, "log1p": 1, "log10": 2}


def device_math(function: str, x: np.ndarray, variant: int = -1, device: int = 0) -> np.ndarray:
    """The device's evaluation of glibc's exp / log1p / log10 (variant 0 FMA builds, 1 uncontracted, -1 the one selected for this host)."""
    x = np.ascontiguousarray(x, np.float64)
    out = np.zeros_like(x)
    _check(load_library().sage_b200_device_math(C.c_int(device), C.c_int(MATH_FUNCTIONS[function]), C.c_int(variant), _ptr(x), C.c_uint64(len(x)), _ptr(out)))
    return out


# ------------------------------------------------------------------------------------------------ predict_rt (runner.rs:513-531)
RT_STAGES = ["ms_sort_q", "ms_alignment", "ms_rt_model", "ms_ims_model", "ms_total"]
RT_FEATURES, IMS_FEATURES = 69, 100
RT_COLUMNS = ("aligned_rt", "predicted_rt", "delta_rt_model", "predicted_ims", "delta_ims_model", "spectrum_q")


class CRtOut(C.Structure):
    _fields_ = [(c, C.c_void_p) for c in RT_COLUMNS] + [("alignments", C.c_void_p), ("training_rows", C.c_uint64), ("aligned_peptides", C.c_uint64),
                                                         ("rt_fitted", C.c_int32), ("rt_r2", C.c_double), ("rt_eps", C.c_double),
                                                         ("rt_beta", C.c_double * RT_FEATURES), ("ims_fitted", C.c_int32), ("ims_r2", C.c_double),
                                                         ("ims_eps", C.c_double), ("ims_beta", C.c_double * IMS_FEATURES)] + [(s, C.c_float) for s in RT_STAGES]


def predict_rt(db: IndexedDatabase, peptides: Peptides, features: np.ndarray, file_id, n_files: int) -> dict:
    """The runner's predict_rt stage (runner.rs:513-531) on the device: the ascending poisson sort and interim spectrum q-values,
    global_alignment, retention_model::predict and mobility_model::predict. `features` are FEATURE_DTYPE rows, `file_id` one file per row
    (< n_files), `peptides` the table `db` was built from. The rows are not reordered. Returns aligned_rt, predicted_rt, delta_rt_model,
    predicted_ims, delta_ims_model and the interim spectrum_q (f32, indexed like the rows), alignments (ALIGNMENT_DTYPE[n_files], the input of
    FeatureMap.build), training_rows, aligned_peptides, rt_fitted / rt_r2 / rt_eps / rt_beta, the same for ims, and the stage times (ms_*).
    aligned_rt, delta_rt_model and delta_ims_model feed spectrum_fdr's optional columns."""
    rows = np.ascontiguousarray(features)
    if rows.dtype != FEATURE_DTYPE:
        raise TypeError("features must have FEATURE_DTYPE")
    n = len(rows)
    fid = np.ascontiguousarray(file_id, np.uint32)
    if len(fid) != n:
        raise ValueError("file_id must have one value per row")
    res = {c: np.zeros(n, np.float32) for c in RT_COLUMNS}
    res["alignments"] = np.zeros(int(n_files), ALIGNMENT_DTYPE)
    out = CRtOut(*[_ptr(res[c]) for c in RT_COLUMNS], _ptr(res["alignments"]))
    keep: list = []
    cp = peptides._c(keep)
    _check(load_library().sage_b200_predict_rt(db._h, C.byref(cp), _ptr(rows), _ptr(fid), C.c_uint64(n), C.c_uint64(int(n_files)), C.byref(out)))
    res.update(training_rows=int(out.training_rows), aligned_peptides=int(out.aligned_peptides))
    for m, d in (("rt", RT_FEATURES), ("ims", IMS_FEATURES)):
        res.update({f"{m}_fitted": bool(getattr(out, f"{m}_fitted")), f"{m}_r2": float(getattr(out, f"{m}_r2")),
                    f"{m}_eps": float(getattr(out, f"{m}_eps")), f"{m}_beta": np.array(getattr(out, f"{m}_beta")[:d], np.float64)})
    res.update({s: float(getattr(out, s)) for s in RT_STAGES})
    return res


# ------------------------------------------------------------------------------------------------ picked FDR (fdr.rs)
class CPickedParams(C.Structure):
    _fields_ = [("cterm", C.c_void_p), ("n_proteins", C.c_void_p), ("protein", C.c_void_p), ("generate_decoys", C.c_uint8)]


PICKED_STAGES = ["ms_keys", "ms_peptide", "ms_protein", "ms_total"]


class CPickedOut(C.Structure):
    _fields_ = [("peptide_q", C.c_void_p), ("protein_q", C.c_void_p), ("peptide_passing", C.c_uint64), ("protein_passing", C.c_uint64),
                ("peptide_entries", C.c_uint64), ("protein_entries", C.c_uint64)] + [(s, C.c_float) for s in PICKED_STAGES]


def _picked_params(peptides: Peptides, n_proteins, protein, cterm, generate_decoys, keep: list) -> CPickedParams:
    n = len(peptides)
    cols = []
    for name, x, dt in (("cterm", cterm, np.float32), ("n_proteins", n_proteins, np.uint32), ("protein", protein, np.uint32)):
        if x is None:
            cols.append(None)
            continue
        a = np.ascontiguousarray(x, dt)
        if len(a) != n:
            raise ValueError(f"{name} must have one value per peptide")
        keep.append(a)
        cols.append(_ptr(a))
    return CPickedParams(*cols, int(bool(generate_decoys)))


def picked_fdr(peptides: Peptides, features: np.ndarray, discriminant_score, n_proteins, protein, cterm=None, generate_decoys: bool = True,
               device: int = 0) -> dict:
    """picked_peptide then picked_protein (fdr.rs:123-190, runner.rs:534-537) on the device. `features` are FEATURE_DTYPE rows in the order the
    runner holds them (spectrum_fdr's sorted order: entries are ordered by the first row that reaches them), `discriminant_score` one f32 per
    row, `peptides` the table the rows' PeptideIx index. Per peptide: `n_proteins` (Peptide::proteins.len()), `protein` (an id of the single
    protein name, equal ids for equal names; read where n_proteins == 1) and `cterm` (NaN = None; None = no C-terminal modifications).
    Returns peptide_q and protein_q (f32, indexed like the rows; protein_q is 1.0 where the peptide has != 1 protein), peptide_passing,
    protein_passing, peptide_entries, protein_entries and the stage times (ms_*)."""
    rows = np.ascontiguousarray(features)
    if rows.dtype != FEATURE_DTYPE:
        raise TypeError("features must have FEATURE_DTYPE")
    n = len(rows)
    score = np.ascontiguousarray(discriminant_score, np.float32)
    if len(score) != n:
        raise ValueError("discriminant_score must have one value per row")
    keep: list = []
    cp = peptides._c(keep)
    params = _picked_params(peptides, n_proteins, protein, cterm, generate_decoys, keep)
    res = dict(peptide_q=np.zeros(n, np.float32), protein_q=np.zeros(n, np.float32))
    out = CPickedOut(_ptr(res["peptide_q"]), _ptr(res["protein_q"]))
    _check(load_library().sage_b200_picked_fdr(C.c_int(device), C.byref(cp), C.byref(params), _ptr(rows), _ptr(score), C.c_uint64(n), C.byref(out)))
    res.update({k: int(getattr(out, k)) for k in ("peptide_passing", "protein_passing", "peptide_entries", "protein_entries")})
    res.update({s: float(getattr(out, s)) for s in PICKED_STAGES})
    return res


def picked_precursor(score, decoy, device: int = 0):
    """picked_precursor (fdr.rs:228-287, runner.rs:572) on the device over FeatureMap.quantify()'s rows: `score` (Peak::score, f64) and `decoy`.
    Returns (q_value f32 indexed like the rows, passing = target rows at q <= 0.05)."""
    s = np.ascontiguousarray(score, np.float64)
    d = np.ascontiguousarray(decoy, np.uint8)
    if len(d) != len(s):
        raise ValueError("decoy must have one value per row")
    q = np.zeros(len(s), np.float32)
    passing = C.c_uint64(0)
    _check(load_library().sage_b200_picked_precursor(C.c_int(device), _ptr(s), _ptr(d), C.c_uint64(len(s)), _ptr(q), C.byref(passing)))
    return q, int(passing.value)


def competition_keys(peptides: Peptides, peptide_idx, cterm=None, generate_decoys: bool = True, hash_bits: int = 64, device: int = 0) -> np.ndarray:
    """Test hook: each row's picked_peptide entry rank (first-appearance order). hash_bits < 64 truncates the key hash so that distinct keys
    collide and the exact comparison that separates them runs."""
    idx = np.ascontiguousarray(peptide_idx, np.uint32)
    keep: list = []
    cp = peptides._c(keep)
    params = _picked_params(peptides, None, None, cterm, generate_decoys, keep)
    out = np.zeros(len(idx), np.uint32)
    _check(load_library().sage_b200_competition_keys(C.c_int(device), C.byref(cp), C.byref(params), _ptr(idx), C.c_uint64(len(idx)),
                                                     C.c_uint32(int(hash_bits)), _ptr(out)))
    return out


# ------------------------------------------------------------------------------------------------ protein grouping (protein_grouping.rs)
class CProteinGroupParams(C.Structure):
    _fields_ = [("protein_offsets", C.c_void_p), ("protein_ids", C.c_void_p), ("n_names", C.c_uint64), ("protein_grouping", C.c_uint8),
                ("has_threshold", C.c_uint8), ("generate_decoys", C.c_uint8), ("threshold", C.c_float)]


PROTEIN_GROUP_COUNTS = ["peptides", "proteins", "meta_peptides", "groups", "edges", "covered", "forced", "greedy_picks", "components",
                        "largest_component", "annotated"]
PROTEIN_GROUP_STAGES = ["ms_build", "ms_cover", "ms_lookup"]


class CProteinGroupOut(C.Structure):
    _fields_ = ([(c, C.c_void_p) for c in ("num_protein_groups", "protein_group_q", "pass", "row_group_offsets", "row_groups", "group_offsets",
                                            "group_members", "group_covered", "group_decoy")]
                + [(c, C.c_uint64 * 2) for c in PROTEIN_GROUP_COUNTS] + [("passing", C.c_uint64), ("entries", C.c_uint64)]
                + [(s, C.c_float * 2) for s in PROTEIN_GROUP_STAGES] + [("ms_picked", C.c_float), ("ms_total", C.c_float)])


def protein_groups(peptides: Peptides, features: np.ndarray, peptide_q, discriminant_score, protein_offsets, protein_ids, n_names: int,
                   protein_grouping: bool = True, threshold: float | None = 0.01, generate_decoys: bool = True, device: int = 0) -> dict:
    """generate_protein_groups then picked_protein_group (protein_grouping.rs, fdr.rs:192-226, runner.rs:540-545) on the device.
    `features` are FEATURE_DTYPE rows in spectrum_fdr's sorted order (peptide_idx and label are read), `peptide_q` and `discriminant_score` one
    f32 per row. Peptide p's proteins are the name ids protein_ids[protein_offsets[p]:protein_offsets[p + 1]] in stored order (equal ids for
    equal names, each < n_names). threshold None is the reference's None: pass 2 only.
    Returns num_protein_groups, protein_group_q, pass (1 or 2, 0 = fallback) per row; each row's covered groups as row_group_offsets /
    row_groups; the group table of both passes (group_offsets, group_members as ascending ids, group_covered, group_decoy; pass 2's groups
    follow pass 1's); per-pass counts as 2-element lists (PROTEIN_GROUP_COUNTS); passing, entries and the stage times. protein_group_strings
    builds the reference's strings from it."""
    rows = np.ascontiguousarray(features)
    if rows.dtype != FEATURE_DTYPE:
        raise TypeError("features must have FEATURE_DTYPE")
    n = len(rows)
    pq = np.ascontiguousarray(peptide_q, np.float32)
    score = np.ascontiguousarray(discriminant_score, np.float32)
    if len(pq) != n or len(score) != n:
        raise ValueError("peptide_q and discriminant_score must have one value per row")
    off = np.ascontiguousarray(protein_offsets, np.uint32)
    ids = np.ascontiguousarray(protein_ids, np.uint32)
    if len(off) != len(peptides) + 1:
        raise ValueError("protein_offsets must have one value per peptide, plus one")
    pep_idx = rows["peptide_idx"].astype(np.int64)
    row_cap = int((off[1:].astype(np.int64) - off[:-1])[pep_idx[pep_idx < len(peptides)]].sum()) if n else 0
    group_cap = 2 * min(int(off[-1]), 2 * int(n_names))
    res = dict(num_protein_groups=np.zeros(n, np.uint32), protein_group_q=np.zeros(n, np.float32), row_pass=np.zeros(n, np.uint8),
               row_group_offsets=np.zeros(n + 1, np.uint64), row_groups=np.zeros(row_cap, np.uint32), group_offsets=np.zeros(group_cap + 1, np.uint64),
               group_members=np.zeros(group_cap, np.uint32), group_covered=np.zeros(group_cap, np.uint8), group_decoy=np.zeros(group_cap, np.uint8))
    out = CProteinGroupOut(*[_ptr(res[k]) for k in ("num_protein_groups", "protein_group_q", "row_pass", "row_group_offsets", "row_groups",
                                                    "group_offsets", "group_members", "group_covered", "group_decoy")])
    params = CProteinGroupParams(_ptr(off), _ptr(ids), int(n_names), int(bool(protein_grouping)), int(threshold is not None), int(bool(generate_decoys)),
                                 float("nan") if threshold is None else float(threshold))
    keep: list = []
    cp = peptides._c(keep)
    _check(load_library().sage_b200_protein_groups(C.c_int(device), C.byref(cp), C.byref(params), _ptr(rows), _ptr(pq), _ptr(score), C.c_uint64(n),
                                                   C.byref(out)))
    res["pass"] = res.pop("row_pass")
    res.update({c: [int(v) for v in getattr(out, c)] for c in PROTEIN_GROUP_COUNTS})
    n_groups = sum(res["groups"])
    res["row_groups"] = res["row_groups"][:int(res["row_group_offsets"][-1])]
    res["group_offsets"] = res["group_offsets"][:n_groups + 1]
    res["group_members"] = res["group_members"][:int(res["group_offsets"][-1])]
    res["group_covered"] = res["group_covered"][:n_groups]
    res["group_decoy"] = res["group_decoy"][:n_groups]
    res.update(passing=int(out.passing), entries=int(out.entries), ms_picked=float(out.ms_picked), ms_total=float(out.ms_total))
    res.update({s: [float(v) for v in getattr(out, s)] for s in PROTEIN_GROUP_STAGES})
    return res


def _format_name(name: str, decoy: bool, decoy_tag: str, generate_decoys: bool) -> str:
    return decoy_tag + name if decoy and generate_decoys else name


def group_string(result: dict, g: int, names, decoy_tag: str = "rev_", generate_decoys: bool = True) -> str:
    """ProteinGroup::format of group g of protein_groups' table: its member names, tagged when the group is a decoy, sorted, joined with '/'."""
    a, b = int(result["group_offsets"][g]), int(result["group_offsets"][g + 1])
    dec = bool(result["group_decoy"][g])
    return "/".join(sorted(_format_name(names[i], dec, decoy_tag, generate_decoys) for i in result["group_members"][a:b].tolist()))


def protein_group_strings(result: dict, rows: np.ndarray, peptides: Peptides, protein_offsets, protein_ids, names, decoy_tag: str = "rev_",
                          generate_decoys: bool = True) -> list:
    """The reference's Feature::protein_groups of each row from protein_groups' result (the rule of include/sage_b200.h): a grouped row joins
    its groups' strings, sorted, with ';'; a fallback row is Peptide::proteins(decoy_tag, generate_decoys). names[id] is the name of an id."""
    off = np.asarray(protein_offsets)
    ids = np.asarray(protein_ids)
    roff = result["row_group_offsets"]
    out = []
    for i, p in enumerate(np.asarray(rows["peptide_idx"]).tolist()):
        if result["pass"][i]:
            gs = result["row_groups"][int(roff[i]):int(roff[i + 1])].tolist()
            out.append(";".join(sorted(group_string(result, g, names, decoy_tag, generate_decoys) for g in gs)))
        else:
            dec = bool(peptides.decoy[p])
            out.append(";".join(_format_name(names[k], dec, decoy_tag, generate_decoys) for k in ids[off[p]:off[p + 1]].tolist()))
    return out


def bipartite_cover(left, right, n_left: int, n_right: int, device: int = 0) -> np.ndarray:
    """Test hook: BipartiteGraph::new(edges, n_left, n_right).into_cover() (protein_grouping.rs) on the device: a bool per left node."""
    lft = np.ascontiguousarray(left, np.uint32)
    rgt = np.ascontiguousarray(right, np.uint32)
    if len(lft) != len(rgt):
        raise ValueError("left and right must have one value per edge")
    cover = np.zeros(int(n_left), np.uint8)
    _check(load_library().sage_b200_bipartite_cover(C.c_int(device), _ptr(lft), _ptr(rgt), C.c_uint64(len(lft)), C.c_uint64(int(n_left)),
                                                    C.c_uint64(int(n_right)), _ptr(cover)))
    return cover.astype(bool)


# ------------------------------------------------------------------------------------------------ digest (database.rs:162-258)
class CDigestParams(C.Structure):
    _fields_ = [("missed_cleavages", C.c_uint8), ("min_len", C.c_uint64), ("max_len", C.c_uint64), ("cleave_at", C.c_char_p), ("restrict_", C.c_char_p),
                ("c_terminal", C.c_uint8), ("semi_enzymatic", C.c_uint8), ("peptide_min_mass", C.c_float), ("peptide_max_mass", C.c_float),
                ("static_specs", C.c_void_p), ("static_masses", C.c_void_p), ("n_static", C.c_uint64),
                ("variable_specs", C.c_void_p), ("variable_masses", C.c_void_p), ("n_variable", C.c_uint64),
                ("max_variable_mods", C.c_uint64), ("decoy_tag", C.c_char_p), ("generate_decoys", C.c_uint8)]


DIGEST_COUNTS = ("n_peptides", "n_residues", "n_protein_refs", "n_names", "name_bytes", "n_proteins", "n_windows", "n_groups", "n_candidates", "n_rows",
                 "device_bytes", "peak_device_bytes")
DIGEST_TIMES = ("ms_parse", "ms_upload", "ms_sites", "ms_windows", "ms_group", "ms_expand", "ms_sort", "ms_merge", "ms_total", "ms_wall")


class CDigestInfo(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in DIGEST_COUNTS] + [(n, C.c_float) for n in DIGEST_TIMES]


@dataclass
class DigestResult:
    """The digested peptide table (one row per PeptideIx) and what only the digest knows: cterm (NaN = None), semi_enzymatic, and each
    peptide's proteins as a CSR of ids (protein_offsets, protein_ids) into `names`, the distinct accessions in byte order (id = rank).
    Ids are ascending within a peptide and a repeated accession stays repeated, as Peptide::proteins after its sort."""
    peptides: Peptides
    cterm: np.ndarray
    semi_enzymatic: np.ndarray
    protein_offsets: np.ndarray
    protein_ids: np.ndarray
    names: list
    info: dict

    @property
    def n_proteins(self) -> np.ndarray:
        """Peptide::proteins.len() per peptide, as picked_fdr takes it."""
        return np.diff(self.protein_offsets).astype(np.uint32)

    @property
    def protein(self) -> np.ndarray:
        """The id of each peptide's first protein (0 for a peptide without proteins): picked_fdr reads it where n_proteins == 1."""
        ids = np.append(self.protein_ids, np.uint32(0))
        return np.where(self.n_proteins > 0, ids[self.protein_offsets[:-1]], 0).astype(np.uint32)

    def proteins(self, i: int) -> list:
        """Peptide::proteins of peptide i as accessions (target names; the decoy tag is added when output is formatted)."""
        return [self.names[j] for j in self.protein_ids[self.protein_offsets[i]:self.protein_offsets[i + 1]]]


def _spec_arrays(mods: dict | None, keep: list, variable: bool):
    items = [(k, m) for k, ms in (mods or {}).items() for m in (ms if variable else [ms])]
    specs = (C.c_char_p * max(1, len(items)))(*[k.encode() for k, _ in items])
    masses = np.array([m for _, m in items] or [0.0], np.float32)
    keep += [specs, masses]
    return C.cast(specs, C.c_void_p), _ptr(masses), len(items)


def _digest_params(keep: list, missed_cleavages=0, min_len=5, max_len=50, cleave_at="KR", restrict="P", c_terminal=True, semi_enzymatic=False,
                   peptide_min_mass=500.0, peptide_max_mass=5000.0, static_mods=None, variable_mods=None, max_variable_mods=2, decoy_tag="rev_",
                   generate_decoys=True) -> CDigestParams:
    p = CDigestParams()
    p.missed_cleavages, p.min_len, p.max_len = int(missed_cleavages), int(min_len), int(max_len)
    p.cleave_at, p.restrict_ = cleave_at.encode(), restrict.encode()
    p.c_terminal, p.semi_enzymatic = int(bool(c_terminal)), int(bool(semi_enzymatic))
    p.peptide_min_mass, p.peptide_max_mass = float(peptide_min_mass), float(peptide_max_mass)
    p.static_specs, p.static_masses, p.n_static = _spec_arrays(static_mods, keep, False)
    p.variable_specs, p.variable_masses, p.n_variable = _spec_arrays(variable_mods, keep, True)
    p.max_variable_mods, p.decoy_tag, p.generate_decoys = int(max_variable_mods), decoy_tag.encode(), int(bool(generate_decoys))
    return p


def _export_table(export, h, info: dict) -> tuple:
    """The table of a digest or prefilter handle, exported with `export` into numpy arrays: (Peptides, cterm, semi, prot_off, ids, names)."""
    n, nres, nref = info["n_peptides"], info["n_residues"], info["n_protein_refs"]
    a = dict(seq_off=np.empty(n + 1, np.uint32), seq=np.empty(nres, np.uint8), mods=np.empty(nres, np.float32), nterm=np.empty(n, np.float32),
             cterm=np.empty(n, np.float32), mono=np.empty(n, np.float32), decoy=np.empty(n, np.uint8), missed=np.empty(n, np.uint8),
             semi=np.empty(n, np.uint8), prot_off=np.empty(n + 1, np.uint32), ids=np.empty(nref, np.uint32),
             name_off=np.empty(info["n_names"] + 1, np.uint64), names=np.empty(max(1, info["name_bytes"]), np.uint8))
    t = time.perf_counter()
    _check(export(h, *[_ptr(a[k]) for k in ("seq_off", "seq", "mods", "nterm", "cterm", "mono", "decoy", "missed", "semi", "prot_off", "ids",
                                            "name_off", "names")]))
    info["ms_export"] = (time.perf_counter() - t) * 1e3
    raw = a["names"].tobytes()
    no = a["name_off"]
    names = [raw[no[i]:no[i + 1]].decode("utf-8", errors="surrogateescape") for i in range(len(no) - 1)]
    pep = Peptides(a["seq_off"], a["seq"], a["mods"], a["nterm"], a["mono"], a["decoy"], a["missed"])
    return pep, a["cterm"], a["semi"].astype(bool), a["prot_off"], a["ids"], names


def digest_fasta(fasta, *, device=0, **digest_args) -> DigestResult:
    """Parameters::digest (database.rs:162-258) on the device: FASTA text (str or bytes) to the sorted, merged peptide table. Keywords and
    defaults are Builder::default()'s: missed_cleavages=0, min_len=5, max_len=50, cleave_at="KR", restrict="P", c_terminal=True,
    semi_enzymatic=False, peptide_min_mass=500.0, peptide_max_mass=5000.0, static_mods=None, variable_mods=None, max_variable_mods=2,
    decoy_tag="rev_", generate_decoys=True. static_mods maps a spec ("C", "^", "[Q", ...) to a mass, variable_mods a spec to a list of masses."""
    text = fasta.encode() if isinstance(fasta, str) else bytes(fasta)
    keep: list = []
    p = _digest_params(keep, **digest_args)
    lib = load_library()
    h = C.c_void_p()
    _check(lib.sage_b200_digest_create(C.c_int(device), C.c_char_p(text), C.c_uint64(len(text)), C.byref(p), C.byref(h)))
    try:
        ci = CDigestInfo()
        _check(lib.sage_b200_digest_get_info(h, C.byref(ci)))
        info = {k: getattr(ci, k) for k, _ in CDigestInfo._fields_}
        table = _export_table(lib.sage_b200_digest_export, h, info)
    finally:
        lib.sage_b200_digest_destroy(h)
    return DigestResult(*table, info)


# ------------------------------------------------------------------------------------------------ prefilter (runner.rs:104-128, 161-278)
class CPrefilterParams(C.Structure):
    _fields_ = [("chunk_size", C.c_uint64), ("low_memory", C.c_uint8), ("min_peaks", C.c_uint64)]


PREFILTER_COUNTS = ("chunk_size", "n_chunks", "plain_build", "n_proteins", "unmodified_peptides", "n_spectra", "rows_digested", "rows_kept", "n_peptides",
                    "n_residues", "n_protein_refs", "n_names", "name_bytes", "n_fragments", "device_bytes", "peak_device_bytes")
PREFILTER_TIMES = ("ms_parse", "ms_count", "ms_digest", "ms_index", "ms_quick_score", "ms_compact", "ms_merge", "ms_final_index", "ms_spectra_upload",
                   "ms_wall")


class CPrefilterInfo(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in PREFILTER_COUNTS] + [(n, C.c_float) for n in PREFILTER_TIMES]


@dataclass
class PrefilterResult(DigestResult):
    """The prefiltered peptide table in DigestResult's shape (so picked_fdr and protein_groups take it unchanged; protein ids are ranks in the
    names table of the whole FASTA), the final index over it, and per chunk the rows digested and kept."""
    db: "IndexedDatabase"
    chunk_rows: np.ndarray
    chunk_kept: np.ndarray


def prefilter_fasta(fasta, spectra: SpectraBatch, *, precursor_tol: Tolerance, fragment_tol: Tolerance, min_matched_peaks=4, min_isotope_err=0,
                    max_isotope_err=0, min_precursor_charge=2, max_precursor_charge=4, override_precursor_charge=False, max_fragment_charge=None,
                    chimera=False, report_psms=1, wide_window=False, annotate_matches=False, score_type=0, min_peaks=15, prefilter_chunk_size=0,
                    prefilter_low_memory=True, bucket_size=8192, ion_kinds=("b", "y"), min_ion_index=2, device=0, **digest_args) -> PrefilterResult:
    """The database prefilter (database.prefilter = true, runner.rs:104-128) on the device: the FASTA's proteins in chunks of
    prefilter_chunk_size (0 = Parameters::auto_calculate_prefilter_chunk_size), each chunk digested and indexed, Scorer::quick_score with
    report_psms + 1 for every MS2 spectrum of `spectra` with at least min_peaks peaks, the selected peptides of all chunks merged by
    reorder_peptides, and one index built over them. When the chunk size covers every protein the plain digest and index are built and
    nothing is scored, as the reference does. The Scorer keywords are Scorer's; the digest keywords are digest_fasta's. bucket_size is rounded
    up to a power of two."""
    if isinstance(bucket_size, bool) or not isinstance(bucket_size, (int, np.integer)) or not 1 <= int(bucket_size) <= 1 << 30:
        raise ValueError(f"bucket_size must be an integer in 1..2^30, got {bucket_size!r}")
    bs = 1 << (int(bucket_size) - 1).bit_length()
    text = fasta.encode() if isinstance(fasta, str) else bytes(fasta)
    keep: list = []
    dp = _digest_params(keep, **digest_args)
    sp = CScorerParams()
    sp.precursor_tol, sp.fragment_tol = precursor_tol._c(), fragment_tol._c()
    sp.min_matched_peaks = min_matched_peaks
    sp.min_isotope_err, sp.max_isotope_err = min_isotope_err, max_isotope_err
    sp.min_precursor_charge, sp.max_precursor_charge = min_precursor_charge, max_precursor_charge
    sp.override_precursor_charge = int(override_precursor_charge)
    sp.max_fragment_charge = -1 if max_fragment_charge is None else int(max_fragment_charge)
    sp.chimera, sp.wide_window, sp.annotate_matches = int(chimera), int(wide_window), int(annotate_matches)
    sp.score_type, sp.report_psms = int(score_type), int(report_psms)
    pp = CPrefilterParams(int(prefilter_chunk_size), int(bool(prefilter_low_memory)), int(min_peaks))
    cs = spectra._c(keep)
    kinds = _kinds(ion_kinds)
    lib = load_library()
    h = C.c_void_p()
    _check(lib.sage_b200_prefilter_create(C.c_int(device), C.c_char_p(text), C.c_uint64(len(text)), C.byref(dp), C.byref(sp), C.byref(pp), C.byref(cs),
                                          C.c_uint64(bs), _ptr(kinds), C.c_uint64(len(kinds)), C.c_uint64(int(min_ion_index)), C.byref(h)))
    try:
        ci = CPrefilterInfo()
        _check(lib.sage_b200_prefilter_get_info(h, C.byref(ci)))
        info = {k: getattr(ci, k) for k, _ in CPrefilterInfo._fields_}
        table = _export_table(lib.sage_b200_prefilter_export, h, info)
        rows, kept = np.zeros(info["n_chunks"], np.uint64), np.zeros(info["n_chunks"], np.uint64)
        _check(lib.sage_b200_prefilter_chunk_counts(h, _ptr(rows), _ptr(kept)))
        dbh = C.c_void_p()
        _check(lib.sage_b200_prefilter_take_db(h, C.byref(dbh)))
    finally:
        lib.sage_b200_prefilter_destroy(h)
    db = IndexedDatabase(dbh.value, table[0])
    return PrefilterResult(*table, info, db, rows, kept)


# ------------------------------------------------------------------------------------------------ result files (runner.rs writers)
FILE_RESULTS, FILE_PIN, FILE_FRAGMENTS, FILE_LFQ, FILE_TMT = 1, 2, 3, 4, 5   # SAGE_B200_FILE_*


class CWriteStats(C.Structure):
    _fields_ = [(f, C.c_float) for f in ("ms_upload", "ms_measure", "ms_scan", "ms_write", "ms_d2h", "ms_total")] + [
        (f, C.c_uint64) for f in ("h2d_bytes", "d2h_bytes", "records", "chunks")]


class CWriteInputs(C.Structure):
    _fields_ = [("rows", C.c_void_p), ("psm_id", C.c_void_p), ("n_rows", C.c_uint64), ("fragments", C.c_void_p), ("n_fragments", C.c_uint64),
                ("filename_offsets", C.c_void_p), ("filename_bytes", C.c_void_p), ("n_files", C.c_uint64),
                ("spec_id_offsets", C.c_void_p), ("spec_id_bytes", C.c_void_p), ("n_spec_ids", C.c_uint64),
                ("n_quant", C.c_uint64), ("quant_file_id", C.c_void_p), ("quant_spec_id", C.c_void_p), ("ion_injection_time", C.c_void_p),
                ("peaks", C.c_void_p), ("n_channels", C.c_uint64), ("user_labels", C.c_uint8),
                ("peptides", C.POINTER(CPeptides)), ("cterm", C.c_void_p), ("semi_enzymatic", C.c_void_p), ("protein_offsets", C.c_void_p),
                ("protein_ids", C.c_void_p), ("name_offsets", C.c_void_p), ("name_bytes", C.c_void_p), ("n_names", C.c_uint64),
                ("decoy_tag", C.c_char_p), ("generate_decoys", C.c_uint8), ("file_id", C.c_void_p), ("spec_index", C.c_void_p)] + [
        (f, C.c_void_p) for f in ("discriminant_score", "posterior_error", "spectrum_q", "aligned_rt", "predicted_rt", "delta_rt_model", "predicted_ims",
                                  "delta_ims_model", "peptide_q", "protein_q", "num_protein_groups", "protein_group_q", "group_pass", "row_group_offsets",
                                  "row_groups", "group_offsets", "group_members", "group_decoy")] + [
        ("n_groups", C.c_uint64), ("lfq_rows", C.c_void_p), ("lfq_areas", C.c_void_p), ("lfq_q", C.c_void_p), ("n_lfq", C.c_uint64),
        ("text_budget", C.c_uint64), ("stats", C.POINTER(CWriteStats))]


def _strings(strs, keep: list):
    """A list of str / bytes as a CSR byte table (offsets [n + 1], bytes)."""
    bs = [s.encode() if isinstance(s, str) else bytes(s) for s in strs]
    off = np.concatenate([[0], np.cumsum([len(b) for b in bs], dtype=np.uint64)]).astype(np.uint64)
    data = np.frombuffer(b"".join(bs) + b"\0", np.uint8)
    keep += [off, data]
    return _ptr(off), _ptr(data), len(bs)


def _write(file: int, ci: CWriteInputs, device: int, stats: dict | None) -> bytes:
    lib = load_library()
    st = CWriteStats()
    ci.stats = C.pointer(st)
    size = C.c_uint64()
    _check(lib.sage_b200_write_tsv(C.c_int(device), C.c_int(file), C.byref(ci), None, C.c_uint64(0), C.byref(size)))
    buf = np.empty(max(size.value, 1), np.uint8)
    _check(lib.sage_b200_write_tsv(C.c_int(device), C.c_int(file), C.byref(ci), _ptr(buf), C.c_uint64(size.value), C.byref(size)))
    if stats is not None:
        stats.update({f: getattr(st, f) for f, _ in CWriteStats._fields_})
    return buf[:size.value].tobytes()


def write_fragments(rows: np.ndarray, fragments: np.ndarray, psm_id, *, device: int = 0, text_budget: int = 0, stats: dict | None = None) -> bytes:
    """matched_fragments.sage.tsv (runner.rs write_fragments) on the device: one record per fragment of each row, in row order. rows:
    FEATURE_DTYPE as Scorer.score_batch returns them with annotate_matches (fragment_offset / fragment_count index `fragments`, FRAGMENT_DTYPE);
    psm_id: Feature::psm_id of each row. text_budget: device bytes of text per chunk (0 = the library's default)."""
    rows = np.ascontiguousarray(rows, FEATURE_DTYPE)
    fragments = np.ascontiguousarray(fragments, FRAGMENT_DTYPE)
    pid = np.ascontiguousarray(psm_id, np.uint64)
    if len(pid) != len(rows):
        raise ValueError("psm_id needs one entry per row")
    ci = CWriteInputs(rows=_ptr(rows), psm_id=_ptr(pid), n_rows=len(rows), fragments=_ptr(fragments), n_fragments=len(fragments), text_budget=text_budget)
    return _write(FILE_FRAGMENTS, ci, device, stats)


def write_tmt(filenames, spec_ids, file_id, spec, ion_injection_time, peaks, *, user_labels: bool = False, device: int = 0, text_budget: int = 0,
              stats: dict | None = None) -> bytes:
    """tmt.tsv (runner.rs write_tmt) on the device. filenames / spec_ids: str or bytes; per quantified spectrum (the rows tmt_quantify returns,
    in order): file_id into filenames, spec into spec_ids, its ion injection time and peaks [n, channels] (tmt_quantify's intensities).
    user_labels: the columns are user_1..n (Isobaric::User) instead of tmt_1..n."""
    keep: list = []
    fo, fb, nf = _strings(filenames, keep)
    so, sb, ns = _strings(spec_ids, keep)
    fi, si = np.ascontiguousarray(file_id, np.uint32), np.ascontiguousarray(spec, np.uint32)
    inj = np.ascontiguousarray(ion_injection_time, np.float32)
    pk = np.ascontiguousarray(peaks, np.float32)
    if pk.ndim != 2 or not (len(fi) == len(si) == len(inj) == pk.shape[0]):
        raise ValueError("file_id, spec, ion_injection_time and peaks need one entry (row) per quantified spectrum")
    ci = CWriteInputs(filename_offsets=fo, filename_bytes=fb, n_files=nf, spec_id_offsets=so, spec_id_bytes=sb, n_spec_ids=ns, n_quant=len(fi),
                      quant_file_id=_ptr(fi), quant_spec_id=_ptr(si), ion_injection_time=_ptr(inj), peaks=_ptr(pk), n_channels=pk.shape[1],
                      user_labels=int(user_labels), text_budget=text_budget)
    return _write(FILE_TMT, ci, device, stats)


def _digest_table(ci: CWriteInputs, digest: "DigestResult", decoy_tag: str, generate_decoys: bool, keep: list):
    """The peptide table, its protein lists and names into the inputs (results, pin, lfq)."""
    cp = digest.peptides._c(keep)
    keep.append(cp)
    ci.peptides = C.pointer(cp)
    cols = [np.ascontiguousarray(digest.cterm, np.float32), np.ascontiguousarray(digest.semi_enzymatic, np.uint8),
            np.ascontiguousarray(digest.protein_offsets, np.uint32), np.ascontiguousarray(digest.protein_ids, np.uint32)]
    keep += cols
    ci.cterm, ci.semi_enzymatic, ci.protein_offsets, ci.protein_ids = (_ptr(c) for c in cols)
    ci.name_offsets, ci.name_bytes, ci.n_names = _strings(digest.names, keep)
    tag = decoy_tag.encode()
    keep.append(tag)
    ci.decoy_tag, ci.generate_decoys = tag, int(bool(generate_decoys))


def _column(ci: CWriteInputs, field: str, d: dict | None, key: str, dt, n: int, keep: list):
    if d is None or d.get(key) is None:
        return
    a = np.ascontiguousarray(d[key], dt)
    if len(a) != n:
        raise ValueError(f"{key} needs one value per row")
    keep.append(a)
    setattr(ci, field, _ptr(a))


def _rows_inputs(digest, rows, psm_id, file_id, spec_index, filenames, spec_ids, fdr, rt, picked, decoy_tag, generate_decoys, text_budget, keep):
    rows = np.ascontiguousarray(rows, FEATURE_DTYPE)
    n = len(rows)
    arrs = [np.ascontiguousarray(x, dt) for x, dt in ((psm_id, np.uint64), (file_id, np.uint32), (spec_index, np.uint32))]
    if any(len(a) != n for a in arrs):
        raise ValueError("psm_id, file_id and spec_index need one entry per row")
    keep += [rows] + arrs
    ci = CWriteInputs(rows=_ptr(rows), psm_id=_ptr(arrs[0]), n_rows=n, file_id=_ptr(arrs[1]), spec_index=_ptr(arrs[2]), text_budget=text_budget)
    ci.filename_offsets, ci.filename_bytes, ci.n_files = _strings(filenames, keep)
    ci.spec_id_offsets, ci.spec_id_bytes, ci.n_spec_ids = _strings(spec_ids, keep)
    _digest_table(ci, digest, decoy_tag, generate_decoys, keep)
    for field, d, key in (("discriminant_score", fdr, "discriminant_score"), ("posterior_error", fdr, "posterior_error"), ("spectrum_q", fdr, "spectrum_q"),
                          ("aligned_rt", rt, "aligned_rt"), ("predicted_rt", rt, "predicted_rt"), ("delta_rt_model", rt, "delta_rt_model"),
                          ("predicted_ims", rt, "predicted_ims"), ("delta_ims_model", rt, "delta_ims_model"), ("peptide_q", picked, "peptide_q"),
                          ("protein_q", picked, "protein_q")):
        _column(ci, field, d, key, np.float32, n, keep)
    return ci


def write_results(digest: "DigestResult", rows: np.ndarray, psm_id, file_id, spec_index, filenames, spec_ids, *, fdr: dict | None = None,
                  rt: dict | None = None, picked: dict | None = None, groups: dict | None = None, decoy_tag: str = "rev_", generate_decoys: bool = True,
                  device: int = 0, text_budget: int = 0, stats: dict | None = None) -> bytes:
    """results.sage.tsv (runner.rs write_features) on the device, one record per row in the given order. digest: the table the rows'
    PeptideIx index; file_id / spec_index: each row's entry in filenames / spec_ids (Feature::file_id, spec_id); psm_id: Feature::psm_id.
    fdr, rt, picked, groups: the dicts of spectrum_fdr, predict_rt, picked_fdr and protein_groups over the same rows (None: Feature's defaults;
    without groups protein_groups is empty and num_protein_groups 0)."""
    keep: list = []
    ci = _rows_inputs(digest, rows, psm_id, file_id, spec_index, filenames, spec_ids, fdr, rt, picked, decoy_tag, generate_decoys, text_budget, keep)
    n = ci.n_rows
    if groups is not None:
        _column(ci, "num_protein_groups", groups, "num_protein_groups", np.uint32, n, keep)
        _column(ci, "protein_group_q", groups, "protein_group_q", np.float32, n, keep)
        _column(ci, "group_pass", groups, "pass", np.uint8, n, keep)
        g = [np.ascontiguousarray(groups[k], dt) for k, dt in (("row_group_offsets", np.uint64), ("row_groups", np.uint32), ("group_offsets", np.uint64),
                                                               ("group_members", np.uint32), ("group_decoy", np.uint8))]
        keep += g
        ci.row_group_offsets, ci.row_groups, ci.group_offsets, ci.group_members, ci.group_decoy = (_ptr(a) for a in g)
        ci.n_groups = len(g[4])
    return _write(FILE_RESULTS, ci, device, stats)


def write_pin(digest: "DigestResult", rows: np.ndarray, psm_id, file_id, spec_index, filenames, spec_ids, *, fdr: dict | None = None,
              rt: dict | None = None, decoy_tag: str = "rev_", generate_decoys: bool = True, device: int = 0, text_budget: int = 0,
              stats: dict | None = None) -> bytes:
    """results.sage.pin (runner.rs write_pin) on the device; the arguments are write_results' (the .pin reads no q-values or groups)."""
    keep: list = []
    ci = _rows_inputs(digest, rows, psm_id, file_id, spec_index, filenames, spec_ids, fdr, rt, None, decoy_tag, generate_decoys, text_budget, keep)
    return _write(FILE_PIN, ci, device, stats)


def write_lfq(digest: "DigestResult", quant: dict, q_value, filenames, *, decoy_tag: str = "rev_", generate_decoys: bool = True, device: int = 0,
              text_budget: int = 0, stats: dict | None = None) -> bytes:
    """lfq.tsv (runner.rs write_lfq) on the device: quant is FeatureMap.quantify()'s dict, q_value picked_precursor's q-values over its rows.
    Decoy rows are skipped and Combined rows (charge 0) write charge -1; rows keep quantify's order."""
    keep: list = []
    n = len(quant["id"])
    rows = np.zeros(n, LFQ_ROW_DTYPE)
    rows["peptide"], rows["charge"], rows["decoy"] = quant["id"], quant["charge"], quant["decoy"]
    rows["rt"], rows["spectral_angle"], rows["score"] = quant["rt"], quant["spectral_angle"], quant["score"]
    areas = np.ascontiguousarray(quant["areas"], np.float64).reshape(n, len(filenames))
    q = np.ascontiguousarray(q_value, np.float32)
    if len(q) != n:
        raise ValueError("q_value needs one value per row")
    keep += [rows, areas, q]
    ci = CWriteInputs(lfq_rows=_ptr(rows), lfq_areas=_ptr(areas), lfq_q=_ptr(q), n_lfq=n, text_budget=text_budget)
    ci.filename_offsets, ci.filename_bytes, ci.n_files = _strings(filenames, keep)
    _digest_table(ci, digest, decoy_tag, generate_decoys, keep)
    return _write(FILE_LFQ, ci, device, stats)


def format_hashes(fmt: int, first: int = 0, values=None, n: int = 0, block: int = 1 << 16, device: int = 0) -> np.ndarray:
    """Test hook: per-block FNV-1a 64 of values formatted on the device, each followed by '\n'. fmt 0: ryu layout of the f32 with bits
    first + i (i < n); 1: `{:+}` of that f32; 2: ryu layout of the f64 values."""
    v = None if values is None else np.ascontiguousarray(values, np.float64)
    n = len(v) if v is not None else n
    out = np.zeros(n // block, np.uint64)
    _check(load_library().sage_b200_format_hashes(C.c_int(device), C.c_int(fmt), C.c_uint64(first), _ptr(v) if v is not None else None, C.c_uint64(n),
                                                  C.c_uint64(block), _ptr(out)))
    return out


# ------------------------------------------------------------------------------------------------ MGF reader (mgf.rs)
class CMgfInfo(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("n_bytes", "n_lines", "n_records", "n_spectra", "n_peaks", "n_precursors", "id_bytes", "dropped_records",
                                          "malformed_lines", "file_id", "device_bytes", "peak_device_bytes")] + [("ms_h2d", C.c_float), ("ms_read", C.c_float)]


MGF_ISOLATION = {0: None, 1: "Da", 2: "ppm"}


class MgfSpectra:
    """MgfReader::parse of one MGF file, read on the device (sage_b200_mgf_*). The spectra stay resident for process(); the arrays below are
    their exported copies, in the layout of sage_b200_mgf_export: peak_off / mz / intensity, scan_start_time, tic, and the precursor CSR
    (precursors: prec_off, mz, intensity with intensity_some, charge with charge_some, iso_kind 0 None / 1 Da / 2 ppm, iso_lo, iso_hi)."""

    def __init__(self, handle, info: dict, arrays: dict, device: int):
        self._h, self.info, self.device = handle, info, device
        for k, v in arrays.items():
            setattr(self, k, v)
        self.precursors = {k: arrays[k] for k in ("prec_off", "prec_mz", "prec_intensity", "prec_intensity_some", "prec_charge", "prec_charge_some",
                                                  "iso_kind", "iso_lo", "iso_hi")}
        b = arrays["id_bytes"].tobytes()
        off = arrays["id_off"]
        self.ids = [b[int(off[i]):int(off[i + 1])].decode() for i in range(len(off) - 1)]

    def __len__(self):
        return int(self.info["n_spectra"])

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h and _lib is not None:
            _lib.sage_b200_mgf_destroy(C.c_void_p(h))

    def first_charge(self) -> np.ndarray:
        """precursors.first().charge per spectrum as the processor takes it: None -> 0."""
        first = self.prec_off[:-1].astype(np.int64)
        return np.where(self.prec_charge_some[first] != 0, self.prec_charge[first], 0).astype(np.uint8)

    def raw(self) -> "RawSpectra":
        """The spectra as a RawSpectra batch (level 2) for SpectrumProcessor.process_raw."""
        n = len(self)
        return RawSpectra(self.peak_off.copy(), self.mz.copy(), self.intensity.copy(), np.full(n, 2, np.uint8), self.first_charge(), None,
                          np.full(n, self.info["file_id"], np.uint64), self.scan_start_time.copy())

    def process(self, processor: "SpectrumProcessor") -> SpectraBatch:
        """SpectrumProcessor::process of every spectrum where it is on the device -> a SpectraBatch for Scorer.score_batch. The first
        precursor gives m/z, charge and the isolation window, which must be in Da (the batch has no other kind)."""
        n = len(self)
        first = self.prec_off[:-1].astype(np.int64)
        ppm = np.nonzero(self.iso_kind[first] == 2)[0]
        if len(ppm):
            raise AssertionError(f"spectrum {int(ppm[0])} ({self.ids[int(ppm[0])]!r}) has a ppm isolation window; SpectraBatch holds Da windows only")
        pp = CProcessorParams(processor.take_top_n, int(processor.deisotope), processor.min_deisotope_mz)
        npk = max(1, int(self.info["n_peaks"]))
        off, om, oi, tic = np.zeros(n + 1, np.uint64), np.zeros(npk, np.float32), np.zeros(npk, np.float32), np.zeros(n, np.float32)
        _check(load_library().sage_b200_mgf_process(C.c_void_p(self._h), C.byref(pp), _ptr(off), _ptr(om), _ptr(oi), _ptr(tic)))
        k = int(off[-1])
        da = self.iso_kind[first] == 1
        nan = np.float32(np.nan)
        return SpectraBatch(off, om[:k].copy(), oi[:k].copy(), self.prec_mz[first].copy(), self.first_charge(),
                            np.where(da, self.iso_lo[first], nan).astype(np.float32), np.where(da, self.iso_hi[first], nan).astype(np.float32), tic,
                            np.full(n, 2, np.uint8), self.scan_start_time.copy(), np.full(n, nan, np.float32))


def read_mgf(text, file_id: int = 0, device: int = 0) -> MgfSpectra:
    """MgfReader::with_file_id(file_id).parse(text) on the device. text: the file's contents as str or bytes (UTF-8)."""
    data = text.encode("utf-8") if isinstance(text, str) else bytes(text)
    lib = load_library()
    h = C.c_void_p()
    _check(lib.sage_b200_mgf_create(C.c_int(device), data, C.c_uint64(len(data)), C.c_uint64(file_id), C.byref(h)))
    try:
        ci = CMgfInfo()
        _check(lib.sage_b200_mgf_get_info(h, C.byref(ci)))
        info = {n: getattr(ci, n) for n, _ in CMgfInfo._fields_}
        n, npk, npr, nid = info["n_spectra"], info["n_peaks"], info["n_precursors"], info["id_bytes"]
        a = dict(peak_off=np.zeros(n + 1, np.uint64), mz=np.zeros(npk, np.float32), intensity=np.zeros(npk, np.float32),
                 scan_start_time=np.zeros(n, np.float32), tic=np.zeros(n, np.float32), prec_off=np.zeros(n + 1, np.uint64),
                 prec_mz=np.zeros(npr, np.float32), prec_intensity=np.zeros(npr, np.float32), prec_intensity_some=np.zeros(npr, np.uint8),
                 prec_charge=np.zeros(npr, np.uint8), prec_charge_some=np.zeros(npr, np.uint8), iso_kind=np.zeros(npr, np.uint8),
                 iso_lo=np.zeros(npr, np.float32), iso_hi=np.zeros(npr, np.float32), id_off=np.zeros(n + 1, np.uint64),
                 id_bytes=np.zeros(nid, np.uint8))
        _check(lib.sage_b200_mgf_export(h, *[_ptr(a[k]) for k in ("peak_off", "mz", "intensity", "scan_start_time", "tic", "prec_off", "prec_mz",
                                                                   "prec_intensity", "prec_intensity_some", "prec_charge", "prec_charge_some",
                                                                   "iso_kind", "iso_lo", "iso_hi", "id_off", "id_bytes")]))
    except BaseException:
        lib.sage_b200_mgf_destroy(h)
        raise
    return MgfSpectra(h.value, info, a, device)


def parse_f32(tokens, device: int = 0) -> tuple[np.ndarray, np.ndarray]:
    """str::parse::<f32> of each token (str or bytes) on the device -> (values as u32 bits, ok as bool); a failed parse gives bits 0."""
    bs = [t.encode() if isinstance(t, str) else bytes(t) for t in tokens]
    n = len(bs)
    off = np.zeros(n + 1, np.uint64)
    if n:
        off[1:] = np.cumsum([len(b) for b in bs])
    out, ok = np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.uint8)
    _check(load_library().sage_b200_parse_f32(C.c_int(device), b"".join(bs), _ptr(off), C.c_uint64(n), _ptr(out), _ptr(ok)))
    return out[:n].view(np.uint32), ok[:n].astype(bool)
