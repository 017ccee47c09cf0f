"""A numpy restatement of Sage's search-and-score path, from the peptide table to `Feature` rows: the second CPU authority for
`k_setup_queries`, the counting kernels, `k_replay`, `k_score` and the split scoring kernels.

Written from the reference's Rust (paths relative to crates/sage/src); it shares no code with oracle/sage_oracle.cpp or with the
device library and imports neither. Inputs are plain arrays: the `Peptides` fields (seq_off, seq, mods, nterm (NaN = None), mono,
decoy, missed) and the `SpectraBatch` fields (peak_off, masses, intensities, prec_mz (NaN = no precursor), prec_charge (0 = None),
iso_lo / iso_hi (NaN = None), tic, level, ims).

Numerics: every f32 operation is one np.float32 scalar or array operation in the Rust association; `ln` is libm's `log` and
`f32::ln_1p` is libm's `log1pf`, both through ctypes; order-sensitive folds (ion ladders, intensity and ppm sums, the TIC re-sum,
heaps) are explicit loops, and only independent probes or candidates are vectorised.
"""
from __future__ import annotations

import ctypes
import ctypes.util
from dataclasses import dataclass, field

import numpy as np

F32 = np.float32
_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.log.restype, _libm.log.argtypes = ctypes.c_double, [ctypes.c_double]
_libm.log1pf.restype, _libm.log1pf.argtypes = ctypes.c_float, [ctypes.c_float]


def ln(x: float) -> float:
    """f64::ln = the platform libm's log()."""
    return _libm.log(float(x))


def ln_1p_f32(x) -> np.float32:
    """f32::ln_1p = libm's log1pf()."""
    return F32(_libm.log1pf(ctypes.c_float(x)))


# mass.rs:5-8, evaluated as f32 constants
PROTON = F32(1.0072764)
NEUTRON = F32(1.00335)
TWO_E6 = F32(2e6)
LN_10 = 2.302585092994046   # std::f64::consts::LN_10
PEPTIDE_IX_DEFAULT = 0xFFFFFFFF   # PeptideIx::default() (database.rs:372-376)
PPM, PCT, DA = 0, 1, 2
KINDS = {"a": 0, "b": 1, "c": 2, "x": 3, "y": 4, "z": 5}   # ion_series.rs:8-15

# mass.rs:64-68
MONOISOTOPIC_MASSES = np.array([
    71.03711, 0.0, 103.00919, 115.02694, 129.04259, 147.0684, 57.02146, 137.05891, 113.08406, 0.0,
    128.09496, 113.08406, 131.0405, 114.04293, 237.14774, 97.05276, 128.05858, 156.1011, 87.03203,
    101.04768, 150.95363, 99.06841, 186.07932, 0.0, 163.06332, 0.0], dtype=np.float32)


def residue_mass(aa: np.ndarray) -> np.ndarray:
    """mass.rs:70-76: the table for 'A'..'Z', 0.0 for anything else."""
    aa = np.asarray(aa, np.int64)
    up = (aa >= ord("A")) & (aa <= ord("Z"))
    return np.where(up, MONOISOTOPIC_MASSES[np.clip(aa - ord("A"), 0, 25)], F32(0.0)).astype(np.float32)


def is_nterm_kind(kind: int) -> bool:
    return kind <= 2   # Kind::A | Kind::B | Kind::C


# ------------------------------------------------------------------------------------------------ total_cmp and binary search
def f32_key(x) -> np.ndarray:
    """f32::total_cmp as an order-preserving i32 image."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.int32)
    return b ^ ((b >> 31).view(np.uint32) >> np.uint32(1)).view(np.int32)


def f64_key(x: float) -> int:
    """f64::total_cmp as an order-preserving integer."""
    b = int(np.float64(x).view(np.int64))
    return b ^ 0x7FFFFFFFFFFFFFFF if b < 0 else b


def partition_point(n: int, pred) -> int:
    """slice::partition_point as a lower-bound bisection (the form the oracle and the device also use)."""
    lo, hi = 0, n
    while lo < hi:
        mid = lo + (hi - lo) // 2
        if pred(mid):
            lo = mid + 1
        else:
            hi = mid
    return lo


def binary_search_slice(keys: np.ndarray, low, high, is_sorted: bool | None = None):
    """database.rs:549-561 over an array of total_cmp keys (or integers): partition_point(key < low).saturating_sub(1), then
    partition_point(key <= high) over slice[left..]. Vectorised over many (low, high) when the keys are sorted; a literal bisection
    otherwise (unsorted spectra), whose answer then depends on the bisection's probe order."""
    keys = np.asarray(keys)
    low, high = np.atleast_1d(low), np.atleast_1d(high)
    if is_sorted is None:
        is_sorted = bool(np.all(keys[1:] >= keys[:-1])) if len(keys) > 1 else True
    if is_sorted:
        left = np.maximum(np.searchsorted(keys, low, "left").astype(np.int64) - 1, 0)
        right = np.maximum(left, np.searchsorted(keys, high, "right").astype(np.int64))
        return left, right
    left = np.empty(len(low), np.int64)
    right = np.empty(len(low), np.int64)
    n = len(keys)
    for t in range(len(low)):
        lo_k, hi_k = low[t], high[t]
        l_ = max(partition_point(n, lambda i: keys[i] < lo_k) - 1, 0)
        r_ = l_ + partition_point(n - l_, lambda i: keys[l_ + i] <= hi_k)
        left[t], right[t] = l_, r_
    return left, right


# ------------------------------------------------------------------------------------------------ Tolerance (mass.rs:10-57)
@dataclass(frozen=True)
class Tol:
    kind: int
    lo: np.float32
    hi: np.float32

    @staticmethod
    def of(t) -> "Tol":
        """From a (kind, lo, hi) tuple or an object with as_tuple(); the C ABI carries lo / hi as f32."""
        if hasattr(t, "as_tuple"):
            t = t.as_tuple()
        return Tol(int(t[0]), F32(t[1]), F32(t[2]))

    def bounds(self, center):
        """mass.rs:21-35."""
        c = np.asarray(center, dtype=np.float32)
        with np.errstate(all="ignore"):
            if self.kind == PPM:
                return c + (c * self.lo) / F32(1e6), c + (c * self.hi) / F32(1e6)
            if self.kind == PCT:
                return c + (c * self.lo) / F32(100.0), c + (c * self.hi) / F32(100.0)
            return c + self.lo, c + self.hi

    def __mul__(self, rhs) -> "Tol":
        """mass.rs:47-57."""
        with np.errstate(all="ignore"):
            return Tol(self.kind, F32(self.lo * F32(rhs)), F32(self.hi * F32(rhs)))


# ------------------------------------------------------------------------------------------------ heap.rs
def sift_down(s: list, length: int, index: int, lt) -> None:
    """heap.rs:40-60 on s[:length]."""
    while index * 2 + 1 < length:
        smallest = index
        left = index * 2 + 1
        if lt(s[left], s[smallest]):
            smallest = left
        right = index * 2 + 2
        if right < length and lt(s[right], s[smallest]):
            smallest = right
        if smallest != index:
            s[smallest], s[index] = s[index], s[smallest]
            index = smallest
        else:
            break


def bounded_min_heapify(s: list, k: int, lt=None) -> None:
    """heap.rs:7-28, in place; `lt(a, b)` is `a < b` (and `a > b` is `lt(b, a)`)."""
    if lt is None:
        lt = _tuple_lt
    if len(s) <= k:
        return
    for i in range(k // 2 - 1, -1, -1):
        sift_down(s, k, i, lt)
    for i in range(k, len(s)):
        if lt(s[0], s[i]):   # slice[i] > slice[0]
            s[i], s[0] = s[0], s[i]
            sift_down(s, k, 0, lt)


def _tuple_lt(a, b) -> bool:
    return a < b


def check_heap(s: list, lt=None) -> bool:
    """heap.rs:30-38."""
    lt = lt or _tuple_lt
    return all(not lt(s[i], s[(i - 1) // 2]) for i in range(1, len(s)))


# ------------------------------------------------------------------------------------------------ scoring.rs:239-247, 770-793
def max_fragment_charge(opt, precursor_charge: int) -> int:
    """None -> precursor_charge; Some(c) -> c + 1 (u8); then min with the precursor charge and max with 2."""
    m = precursor_charge if opt is None else (int(opt) + 1) & 0xFF
    return max(min(precursor_charge, m), 2)


class Run:
    """scoring.rs:771-793: `last` starts at 0, so index 0 never starts a ladder."""
    __slots__ = ("start", "length", "last", "longest")

    def __init__(self):
        self.start = self.length = self.last = self.longest = 0

    def matched(self, index: int) -> None:
        if self.last == index:
            return
        if self.start + self.length == index:
            self.length += 1
            self.longest = max(self.longest, self.length)
        else:
            self.start = index
            self.length = 1
            self.longest = max(self.longest, self.length)
        self.last = index


def lnfact(n: int) -> float:
    """scoring.rs:170-177 (n is a u16)."""
    if n == 0:
        return 1.0
    x = float(n)
    return x * ln(x) - x + 0.5 * ln(x) + 0.5 * ln(np.pi * 2.0 * x)


def score_type_score(score_type: int, matched_b: int, matched_y: int, summed_b, summed_y) -> float:
    """scoring.rs:179-201, including the 255.0 that replaces a non-finite score."""
    summed_b, summed_y = F32(summed_b), F32(summed_y)
    with np.errstate(all="ignore"):
        if score_type == 0:
            i = float(summed_b + F32(1.0)) * float(summed_y + F32(1.0))
            s = ln(i) + lnfact(matched_b) + lnfact(matched_y)
        else:
            s = float(ln_1p_f32(summed_b + summed_y)) + lnfact(matched_b) + lnfact(matched_y)
    return s if np.isfinite(s) else 255.0


# ------------------------------------------------------------------------------------------------ ion_series.rs:36-85
_C, _O, _H, _PRO, _N = F32(12.0), F32(15.994914), F32(1.007825), F32(1.0072764), F32(14.003074)
_NH3 = (_N + _H * F32(2.0)) + _PRO
_X_OFFSET = (((_C + _O) - _NH3) + _N) + _H


def ion_start(kind: int, mono, nterm):
    """IonSeries::new's cumulative_mass (nterm: Option<f32>, NaN = None -> unwrap_or_default)."""
    nt = np.where(np.isnan(nterm), F32(0.0), nterm).astype(np.float32)
    mono = np.asarray(mono, np.float32)
    return [nt - (_C + _O), nt, nt + _NH3, (mono - nt) + _X_OFFSET, mono - nt, (mono - nt) - _NH3][kind]


def ion_tables(pep, kinds) -> dict:
    """Every ion of every kind of every peptide: {kind: (n_peptides, max_len - 1) f32}, column idx = the iterator's idx. The
    cumulative sum is a loop over residue positions (the Rust fold), vectorised only across peptides."""
    seq_off = np.asarray(pep.seq_off, np.int64)
    lens = np.diff(seq_off)
    n = len(lens)
    width = max(int(lens.max()) - 1, 0) if n else 0
    pos = np.arange(width)
    valid = pos[None, :] < (lens - 1)[:, None]
    flat = seq_off[:-1, None] + pos[None, :]
    flat = np.where(valid, flat, 0)
    seq = np.asarray(pep.seq, np.uint8)
    mods = np.asarray(pep.mods, np.float32)
    delta = np.zeros((n, width), np.float32)
    if width and len(seq):
        delta = np.where(valid, residue_mass(seq[flat]) + mods[flat], F32(0.0)).astype(np.float32)   # monoisotopic(r) + m
    out = {}
    for kind in kinds:
        cum = ion_start(kind, pep.mono, pep.nterm).astype(np.float32)
        tab = np.zeros((n, width), np.float32)
        for p in range(width):
            step = delta[:, p] if is_nterm_kind(kind) else -delta[:, p]
            cum = np.where(valid[:, p], cum + step, cum).astype(np.float32)
            tab[:, p] = cum
        out[kind] = tab
    return out


# ------------------------------------------------------------------------------------------------ database.rs:265-365
def next_power_of_two(n: int) -> int:
    """Builder::make_parameters rounds bucket_size up (database.rs:97)."""
    return 1 if n <= 1 else 1 << (int(n) - 1).bit_length()


@dataclass
class Index:
    """IndexedDatabase (database.rs:384-395) plus the per-peptide ion tables the scorer regenerates."""
    pep: object
    lens: np.ndarray
    ions: dict
    frag_pep: np.ndarray
    frag_mz: np.ndarray
    bucket_min: np.ndarray
    bucket_size: int
    ion_kinds: list
    mono: np.ndarray = field(default=None)
    mono_key: np.ndarray = field(default=None)
    mono_sorted: bool = True

    def __post_init__(self):
        self.mono = np.asarray(self.pep.mono, np.float32)
        self.mono_key = f32_key(self.mono).astype(np.int64)
        self.mono_sorted = bool(np.all(self.mono_key[1:] >= self.mono_key[:-1])) if len(self.mono) > 1 else True
        self.bucket_key = f32_key(self.bucket_min).astype(np.int64)
        page = np.arange(len(self.frag_pep), dtype=np.int64) // self.bucket_size
        self.gkey = (page << 33) + self.frag_pep.astype(np.int64)   # (page, PeptideIx): ascending over the whole array

    @property
    def n_peptides(self) -> int:
        return len(self.mono)

    def ion_list(self, peptide: int):
        """[(kind, idx, mass)] of IonSeries::new(peptide, kind).enumerate() over db.ion_kinds (scoring.rs:693-697)."""
        L = int(self.lens[peptide])
        return [(k, i, self.ions[k][peptide, i]) for k in self.ion_kinds for i in range(L - 1)]


def build_from_peptides(pep, bucket_size: int = 8192, ion_kinds=("b", "y"), min_ion_index: int = 2) -> Index:
    """database.rs:265-365. `par_sort_unstable_by` on fragment m/z and the per-bucket `par_sort_unstable_by` on PeptideIx leave
    equal keys in an unspecified order; the order used here (and by the device's stable radix sorts and the oracle) is by m/z
    (total_cmp) then PeptideIx, then a stable PeptideIx sort inside each bucket. Entries that tie on both are identical."""
    kinds = [KINDS[k] if isinstance(k, str) else int(k) for k in ion_kinds]
    lens = np.diff(np.asarray(pep.seq_off, np.int64))
    ions = ion_tables(pep, kinds)
    peps, mzs = [], []
    for kind in kinds:
        tab = ions[kind]
        idx = np.arange(tab.shape[1])[None, :]
        valid = idx < (lens - 1)[:, None]
        if is_nterm_kind(kind):
            keep = valid & ((idx + 1) > min_ion_index)
        else:
            keep = valid & (((lens - 1)[:, None] - idx) > min_ion_index)   # sequence.len().saturating_sub(1) - ion_idx
        r, c = np.nonzero(keep)
        peps.append(r.astype(np.uint32))
        mzs.append(tab[r, c])
    frag_pep = np.concatenate(peps) if peps else np.zeros(0, np.uint32)
    frag_mz = np.concatenate(mzs).astype(np.float32) if mzs else np.zeros(0, np.float32)
    o = np.lexsort((frag_pep, f32_key(frag_mz)))
    frag_pep, frag_mz = frag_pep[o], frag_mz[o]
    chunk = np.arange(len(frag_pep)) // bucket_size
    bucket_min = frag_mz[::bucket_size].copy()   # chunk[0].fragment_mz of every par_chunks_mut(bucket_size)
    o = np.lexsort((np.arange(len(frag_pep)), frag_pep, chunk))
    return Index(pep, lens, ions, frag_pep[o].astype(np.uint32), frag_mz[o].astype(np.float32), bucket_min.astype(np.float32),
                 int(bucket_size), kinds)


# ------------------------------------------------------------------------------------------------ database.rs:402-536
@dataclass
class Query:
    precursor_mass: np.float32
    ptol: Tol
    ftol: Tol
    pre_idx_lo: int
    pre_idx_hi: int
    plo: np.float32
    phi: np.float32


def db_query(db: Index, precursor_mass, ptol: Tol, ftol: Tol) -> Query:
    """IndexedDatabase::query (database.rs:402-425)."""
    plo, phi = ptol.bounds(F32(precursor_mass))
    lo, hi = binary_search_slice(db.mono_key, f32_key(plo), f32_key(phi), db.mono_sorted)
    return Query(F32(precursor_mass), ptol, ftol, int(lo[0]), int(hi[0]), F32(plo), F32(phi))


@dataclass
class Counters:
    pages: int = 0
    entries_scanned: int = 0


def page_search_counts(db: Index, q: Query, masses: np.ndarray, ctr: Counters | None = None):
    """IndexedQuery::page_search (database.rs:480-536) for a batch of independent probe masses: returns (probe, PeptideIx) of
    every matching fragment. Pages: binary_search_slice over min_value; per page binary_search_slice over PeptideIx; then the
    edge filter at pre_idx_lo / pre_idx_hi (the monoisotopic check only for those two PeptideIx) and the fragment bounds."""
    flo, fhi = q.ftol.bounds(np.asarray(masses, np.float32))
    left, right = binary_search_slice(db.bucket_key, f32_key(flo).astype(np.int64), f32_key(fhi).astype(np.int64), True)
    npages = right - left
    probe = np.repeat(np.arange(len(masses)), npages)
    page = np.repeat(left, npages) + (np.arange(int(npages.sum())) - np.repeat(np.cumsum(npages) - npages, npages))
    nf = len(db.frag_pep)
    pstart = page * db.bucket_size
    pp = np.searchsorted(db.gkey, (page << 33) + q.pre_idx_lo, "left")
    il = np.maximum(pp - 1, pstart)                                               # saturating_sub(1) inside the page
    ir = np.maximum(il, np.searchsorted(db.gkey, (page << 33) + q.pre_idx_hi, "right"))
    ir = np.minimum(ir, np.minimum((page + 1) * db.bucket_size, nf))
    if ctr is not None:
        ctr.pages += int(len(page))
        ctr.entries_scanned += int((ir - il).sum())
    cnt = ir - il
    e = np.repeat(il, cnt) + (np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt))
    pr = np.repeat(probe, cnt)
    fp = db.frag_pep[e].astype(np.int64)
    fm = db.frag_mz[e]
    lo32, hi32 = q.pre_idx_lo, q.pre_idx_hi
    mono_at = db.mono[np.minimum(fp, max(db.n_peptides - 1, 0))] if db.n_peptides else np.zeros(len(fp), np.float32)
    ok = ((fp > lo32) | ((fp == lo32) & (mono_at >= q.plo))) & ((fp < hi32) | ((fp == hi32) & (mono_at <= q.phi))) \
        & (fm >= flo[pr]) & (fm <= fhi[pr])
    return pr[ok], fp[ok]


# ------------------------------------------------------------------------------------------------ scoring.rs
@dataclass
class InitialHits:
    """scoring.rs:52-67; preliminary holds PreScore tuples (matched u16, peptide u32, precursor_charge u8, isotope_error i8)."""
    matched_peaks: int = 0
    scored_candidates: int = 0
    preliminary: list = field(default_factory=list)

    def __iadd__(self, rhs: "InitialHits"):
        self.matched_peaks += rhs.matched_peaks
        self.scored_candidates += rhs.scored_candidates
        self.preliminary.extend(rhs.preliminary)
        return self


PRESCORE_DEFAULT = (0, PEPTIDE_IX_DEFAULT, 0, 0)


@dataclass
class Spectrum:
    """ProcessedSpectrum + its first Precursor (spectrum.rs:47-79)."""
    masses: np.ndarray
    intensities: np.ndarray
    prec_mz: np.float32
    charge: int | None
    isolation: tuple | None
    tic: np.float32
    level: int = 2
    ims: np.float32 | None = None

    def __post_init__(self):
        self.keys = f32_key(self.masses).astype(np.int64)
        self.sorted = bool(np.all(self.keys[1:] >= self.keys[:-1])) if len(self.keys) > 1 else True


def spectra_from_batch(b) -> list:
    """SpectraBatch fields (object or dict) -> [Spectrum]; None for a spectrum without a precursor (prec_mz NaN)."""
    g = (lambda k: b.get(k)) if isinstance(b, dict) else (lambda k: getattr(b, k, None))
    off = np.asarray(g("peak_off"), np.int64)
    masses, intens = np.asarray(g("masses"), np.float32), np.asarray(g("intensities"), np.float32)
    level, ims = g("level"), g("ims")
    out = []
    for i in range(len(off) - 1):
        pm = F32(g("prec_mz")[i])
        lo, hi = F32(g("iso_lo")[i]), F32(g("iso_hi")[i])
        z = int(g("prec_charge")[i])
        out.append(Spectrum(masses[off[i]:off[i + 1]].copy(), intens[off[i]:off[i + 1]].copy(), pm, z if z else None,
                            None if (np.isnan(lo) or np.isnan(hi)) else (lo, hi), F32(g("tic")[i]),
                            2 if level is None else int(level[i]), None if ims is None or np.isnan(ims[i]) else F32(ims[i])))
    return out


def select_most_intense_peaks(s: Spectrum, centers: np.ndarray, tol: Tol) -> np.ndarray:
    """spectrum.rs:134-159 for independent centers: binary_search_slice, then among masses inside [lo, hi] the LAST peak whose
    intensity is >= the running maximum that starts at 0.0 (so equal intensities pick the last one, a zero-intensity peak can be
    picked, negative and NaN intensities never). Returns the peak index per center, -1 for None."""
    centers = np.asarray(centers, np.float32)
    best = np.full(len(centers), -1, np.int64)
    if len(centers) == 0 or len(s.masses) == 0:
        return best
    lo, hi = tol.bounds(centers)
    i, j = binary_search_slice(s.keys, f32_key(lo).astype(np.int64), f32_key(hi).astype(np.int64), s.sorted)
    cnt = j - i
    pair = np.repeat(np.arange(len(centers)), cnt)
    idx = np.repeat(i, cnt) + (np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt))
    m, it = s.masses[idx], s.intensities[idx]
    acc = (m >= lo[pair]) & (m <= hi[pair]) & (it >= F32(0.0))
    pair, idx, it = pair[acc], idx[acc], it[acc]
    if len(pair) == 0:
        return best
    mx = np.full(len(centers), -np.inf, np.float32)
    np.maximum.at(mx, pair, it)
    top = it == mx[pair]
    np.maximum.at(best, pair[top], idx[top])
    return best


class Scorer:
    """scoring.rs:210-232 over an `Index`."""

    def __init__(self, db: Index, precursor_tol, fragment_tol, min_matched_peaks=4, min_isotope_err=0, max_isotope_err=0,
                 min_precursor_charge=2, max_precursor_charge=4, override_precursor_charge=False, max_fragment_charge=None, chimera=False,
                 report_psms=1, wide_window=False, annotate_matches=False, score_type=0):
        self.db = db
        self.precursor_tol, self.fragment_tol = Tol.of(precursor_tol), Tol.of(fragment_tol)
        self.min_matched_peaks = int(min_matched_peaks)
        self.min_isotope_err, self.max_isotope_err = int(min_isotope_err), int(max_isotope_err)
        self.min_precursor_charge, self.max_precursor_charge = int(min_precursor_charge), int(max_precursor_charge)
        self.override_precursor_charge = bool(override_precursor_charge)
        self.max_fragment_charge = max_fragment_charge
        self.chimera, self.report_psms, self.wide_window = bool(chimera), int(report_psms), bool(wide_window)
        self.annotate_matches, self.score_type = bool(annotate_matches), int(score_type)
        self.counters = Counters()

    # :322-329
    def trim_hits(self, hits: InitialHits) -> None:
        n = len(hits.preliminary)
        lo, hi = min(self.report_psms * 2, n), n
        k = lo if 50 < lo else (hi if 50 > hi else 50)   # 50.clamp(lo, hi)
        bounded_min_heapify(hits.preliminary, k)
        del hits.preliminary[k:]

    # :335-382
    def matched_peaks_with_isotope(self, s: Spectrum, precursor_mass, precursor_charge: int, ptol: Tol, isotope_error: int) -> InitialHits:
        q = db_query(self.db, F32(precursor_mass) - F32(isotope_error) * NEUTRON, ptol, self.fragment_tol)
        mfc = max_fragment_charge(self.max_fragment_charge, precursor_charge)
        potential = q.pre_idx_hi - q.pre_idx_lo + 1
        charges = np.arange(1, mfc, dtype=np.int64)
        with np.errstate(all="ignore"):
            probes = (s.masses[:, None] * charges.astype(np.float32)[None, :]).reshape(-1).astype(np.float32)   # peak_mass * charge
        _, peps = page_search_counts(self.db, q, probes, self.counters)
        total = np.bincount(peps - q.pre_idx_lo, minlength=potential).astype(np.int64) if len(peps) else np.zeros(potential, np.int64)
        hits = InitialHits(int(total.sum()), 0, [PRESCORE_DEFAULT] * potential)
        # PreScore::matched is a u16 and the release profile does not check overflow: the count wraps, and every match that finds
        # it at 0 (the first, and the one after each wrap) re-enters `if sc.matched == 0` and counts the candidate again
        hits.scored_candidates = int(((total + 0xFFFF) // 0x10000).sum())
        for slot in np.nonzero(total)[0]:
            hits.preliminary[slot] = (int(total[slot]) & 0xFFFF, int(q.pre_idx_lo + slot), precursor_charge, isotope_error)
        if hits.matched_peaks == 0:
            return hits   # :376-378: the untrimmed all-default list
        self.trim_hits(hits)
        return hits

    # :384-416
    def matched_peaks(self, s: Spectrum, precursor_mass, precursor_charge: int, ptol: Tol) -> InitialHits:
        if self.min_isotope_err != self.max_isotope_err:
            hits = InitialHits()
            for iso in range(self.min_isotope_err, self.max_isotope_err + 1):
                hits += self.matched_peaks_with_isotope(s, precursor_mass, precursor_charge, ptol, iso)
            self.trim_hits(hits)
            return hits
        return self.matched_peaks_with_isotope(s, precursor_mass, precursor_charge, ptol, 0)

    # :418-462
    def initial_hits(self, s: Spectrum) -> InitialHits:
        mz = s.prec_mz - PROTON
        with np.errstate(all="ignore"):
            if self.wide_window:
                hits = InitialHits()
                for z in range(self.min_precursor_charge, self.max_precursor_charge + 1):
                    iso = Tol(DA, s.isolation[0], s.isolation[1]) if s.isolation is not None else Tol(DA, F32(-2.4), F32(2.4))
                    hits += self.matched_peaks(s, mz * F32(z), z, iso * F32(z))
            elif s.charge is not None and not self.override_precursor_charge:
                hits = self.matched_peaks(s, mz * F32(s.charge), s.charge, self.precursor_tol)
            else:
                hits = InitialHits()
                for z in range(self.min_precursor_charge, self.max_precursor_charge + 1):
                    hits += self.matched_peaks(s, mz * F32(z), z, self.precursor_tol)
        self.trim_hits(hits)
        return hits

    # :675-767
    def score_candidate(self, s: Spectrum, pre: tuple):
        """Returns (Score dict, fragments list | None)."""
        peptide, charge, iso = pre[1], pre[2], pre[3]
        mfc = max_fragment_charge(self.max_fragment_charge, charge)
        ions = self.db.ion_list(peptide)
        charges = list(range(1, mfc))
        with np.errstate(all="ignore"):
            mzs = np.array([m / F32(c) for (_, _, m) in ions for c in charges], np.float32)   # frag.monoisotopic_mass / charge
        best = select_most_intense_peaks(s, mzs, self.fragment_tol)
        mb = my = 0
        sb = sy = ppm = F32(0.0)
        b_run, y_run = Run(), Run()
        frags = [] if self.annotate_matches else None
        L = int(self.db.lens[peptide])
        t = 0
        with np.errstate(all="ignore"):
            for (kind, idx, _) in ions:
                for c in charges:
                    pk = best[t]
                    mz = mzs[t]
                    t += 1
                    if pk < 0:
                        continue
                    pm, pi = s.masses[pk], s.intensities[pk]
                    ppm = ppm + ((pi * abs(mz - pm)) * TWO_E6) / (mz + pm)
                    if is_nterm_kind(kind):
                        mb = (mb + 1) & 0xFFFF
                        sb = sb + pi
                        b_run.matched(idx)
                    else:
                        my = (my + 1) & 0xFFFF
                        sy = sy + pi
                        y_run.matched(idx)
                    if frags is not None:
                        ordinal = idx + 1 if is_nterm_kind(kind) else max(L - 1, 0) - idx
                        frags.append((kind, c, ordinal, pi, mz + PROTON, pm + PROTON))
            hyperscore = score_type_score(self.score_type, mb, my, sb, sy)
            ppm = ppm / (sb + sy)
        return dict(peptide=peptide, matched_b=mb, matched_y=my, summed_b=F32(sb), summed_y=F32(sy), longest_b=b_run.longest,
                    longest_y=y_run.longest, hyperscore=hyperscore, ppm_difference=F32(ppm), precursor_charge=charge, isotope_error=iso), frags

    # :478-595
    def build_features(self, s: Spectrum, hits: InitialHits, report_psms: int, features: list) -> None:
        sv = []
        for pre in hits.preliminary:
            if pre[1] == PEPTIDE_IX_DEFAULT:
                continue
            sc, fr = self.score_candidate(s, pre)
            if ((sc["matched_b"] + sc["matched_y"]) & 0xFFFF) >= self.min_matched_peaks:
                sv.append((sc, fr))
        sv.sort(key=lambda e: -f64_key(e[0]["hyperscore"]))   # stable sort_by(b.total_cmp(a))
        mp, scd = hits.matched_peaks, hits.scored_candidates
        lam = mp / scd if scd else (float("nan") if mp == 0 else float("inf"))
        mz = s.prec_mz - PROTON
        pep = self.db.pep
        for idx in range(min(report_psms, len(sv))):
            sc, fr = sv[idx]
            p = sc["peptide"]
            mono = self.db.mono[p]
            with np.errstate(all="ignore"):
                precursor_mass = mz * F32(sc["precursor_charge"])
                nxt = sv[idx + 1][0]["hyperscore"] if idx + 1 < len(sv) else 0.0
                best = sv[0][0]["hyperscore"]
                k = (sc["matched_b"] + sc["matched_y"]) & 0xFFFF
                log10_poisson = (float(k) * ln(lam) - lam - lnfact(k)) / LN_10
                iso_e = F32(sc["isotope_error"]) * NEUTRON
                delta_mass = (((precursor_mass - mono) - iso_e) * TWO_E6) / ((precursor_mass - iso_e) + mono)
                summed = sc["summed_b"] + sc["summed_y"]
                L = int(self.db.lens[p])
                features.append(dict(
                    peptide_idx=p, peptide_len=L, rank=idx + 1, label=-1 if pep.decoy[p] else 1, expmass=F32(precursor_mass), calcmass=mono,
                    charge=sc["precursor_charge"], delta_mass=F32(delta_mass), isotope_error=F32(iso_e), average_ppm=sc["ppm_difference"],
                    hyperscore=sc["hyperscore"], delta_next=sc["hyperscore"] - nxt, delta_best=best - sc["hyperscore"], matched_peaks=k,
                    longest_b=sc["longest_b"], longest_y=sc["longest_y"], longest_y_pct=F32(F32(sc["longest_y"]) / F32(L)),
                    missed_cleavages=int(pep.missed[p]), matched_intensity_pct=F32((F32(100.0) * summed) / s.tic),
                    scored_candidates=scd & 0xFFFFFFFF, poisson=log10_poisson if np.isfinite(log10_poisson) else float("-inf"),
                    ms2_intensity=F32(summed), fragments=fr))

    # :598-644
    def remove_matched_peaks(self, s: Spectrum, psm: dict) -> Spectrum:
        mfc = max_fragment_charge(self.max_fragment_charge, psm["charge"])
        with np.errstate(all="ignore"):
            centers = np.array([m / F32(c) for (_, _, m) in self.db.ion_list(psm["peptide_idx"]) for c in range(1, mfc)], np.float32)
        best = select_most_intense_peaks(s, centers, self.fragment_tol)
        picked = best[best >= 0]
        rm_m, rm_i = s.masses[picked], s.intensities[picked]
        # Vec::contains on (f32, f32): PartialEq, so NaN never equals and -0.0 == 0.0
        hit = (s.masses[:, None] == rm_m[None, :]) & (s.intensities[:, None] == rm_i[None, :])
        keep = ~hit.any(axis=1) if len(rm_m) else np.ones(len(s.masses), bool)
        masses, intens = s.masses[keep].copy(), s.intensities[keep].copy()
        tic = F32(0.0)
        with np.errstate(all="ignore"):
            for x in intens:   # iter().sum::<f32>()
                tic = tic + x
        return Spectrum(masses, intens, s.prec_mz, s.charge, s.isolation, tic, s.level, s.ims)

    # :648-672
    def score_chimera_fast(self, s: Spectrum) -> list:
        hits = self.initial_hits(s)
        cands: list = []
        prev = 0
        while len(cands) < self.report_psms:
            self.build_features(s, hits, 1, cands)
            if len(cands) > prev:
                s = self.remove_matched_peaks(s, cands[prev])
                cands[prev]["rank"] = prev + 1
                prev = len(cands)
            else:
                break
        return cands

    # :300-309, 465-474
    def score(self, s: Spectrum) -> list:
        if s.level != 2 or np.isnan(s.prec_mz):
            raise ValueError("the reference panics on a non-MS2 scan or a missing precursor")
        if self.chimera:
            return self.score_chimera_fast(s)
        out: list = []
        self.build_features(s, self.initial_hits(s), self.report_psms, out)
        return out

    # :255-298
    def quick_score(self, s: Spectrum, prefilter_low_memory: bool, keep: np.ndarray) -> None:
        hits = self.initial_hits(s)
        if prefilter_low_memory:
            sv = []
            for pre in hits.preliminary:
                if pre[1] == PEPTIDE_IX_DEFAULT:
                    continue
                sc, _ = self.score_candidate(s, pre)
                if ((sc["matched_b"] + sc["matched_y"]) & 0xFFFF) < self.min_matched_peaks:
                    continue
                sv.append(sc)
            k = min(self.report_psms, len(sv))
            bounded_min_heapify(sv, k, score_partial_lt)
            for sc in sv[:k]:
                keep[sc["peptide"]] = 1
        else:
            for pre in hits.preliminary:
                if pre[1] != PEPTIDE_IX_DEFAULT:
                    keep[pre[1]] = 1


_SCORE_FIELDS = ("peptide", "matched_b", "matched_y", "summed_b", "summed_y", "longest_b", "longest_y", "hyperscore", "ppm_difference",
                 "precursor_charge", "isotope_error")


def score_partial_lt(a: dict, b: dict) -> bool:
    """`a < b` under Score's DERIVED PartialOrd (scoring.rs:17-30: field order, peptide first), which heap.rs's `<` / `>` use — not
    the hyperscore `Ord`. A NaN field makes partial_cmp None, and `<` is then false."""
    for f in _SCORE_FIELDS:
        x, y = a[f], b[f]
        if x < y:
            return True
        if x > y:
            return False
        if not x == y:
            return False
    return False


# ------------------------------------------------------------------------------------------------ batch drivers
FEATURE_FIELDS = ("peptide_idx", "peptide_len", "rank", "label", "expmass", "calcmass", "charge", "delta_mass", "isotope_error", "average_ppm",
                  "hyperscore", "delta_next", "delta_best", "matched_peaks", "longest_b", "longest_y", "longest_y_pct", "missed_cleavages",
                  "matched_intensity_pct", "scored_candidates", "poisson", "ms2_intensity")


def score_batch(db: Index, cfg: dict, spectra, counters: bool = False):
    """`spectra.iter().map(|s| scorer.score(s))` -> (rows per spectrum, fragments per row | None, counters | None)."""
    sc = Scorer(db, **cfg)
    rows = []
    for s in spectra_from_batch(spectra):
        rows.append(sc.score(s))
    frags = [[r["fragments"] for r in rs] for rs in rows] if sc.annotate_matches else None
    return rows, frags, (dict(pages=sc.counters.pages, entries_scanned=sc.counters.entries_scanned) if counters else None)


def quick_score_batch(db: Index, cfg: dict, spectra, low_memory: bool) -> np.ndarray:
    sc = Scorer(db, **cfg)
    keep = np.zeros(db.n_peptides, np.uint8)
    for s in spectra_from_batch(spectra):
        sc.quick_score(s, low_memory, keep)
    return keep


def initial_hits_one(db: Index, cfg: dict, spectra) -> InitialHits:
    """The trimmed preliminary list of the first spectrum, in heap order."""
    return Scorer(db, **cfg).initial_hits(spectra_from_batch(spectra)[0])
