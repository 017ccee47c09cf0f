"""An independent numpy restatement of sage's label-free quantification, written from crates/sage/src/lfq.rs, isotopes.rs and mass.rs (cited as
file:line). TEST INFRASTRUCTURE ONLY: it shares no code with the CPU oracle (oracle_lfq/) or the device kernels, so a misreading of lfq.rs that
those two share shows up as a difference here.

Where lfq.rs leaves an order unspecified (DashMap, rayon, par_sort_unstable_by) this module uses the order the device path defines (DESIGN.md §9):
ranges before sorting in ascending (PeptideIx, charge, isotope, forward before decoy), both sorts stable, and each grid cell summed in (add_ms1
call, spectrum, peak, map position, lo before hi) order.

Every f32 operation is one numpy float32 operation (one IEEE rounding, no contraction). expf comes from the C library through ctypes (numpy's
float32 exp is its own SIMD code); acos, exp and pow come from Python's math module, which calls the C library. Sums whose association matters
are explicit loops, vectorised only across independent sums, never np.sum or np.add.reduceat (both pairwise).
"""
from __future__ import annotations

import ctypes
import ctypes.util
import math

import numpy as np

from sage_b200.api import LFQ_RANGE_DTYPE

f32 = np.float32
RT_TOL = f32(0.0050)        # lfq.rs:15
K_WIDTH = 10                # lfq.rs:17
GRID_SIZE = 100             # lfq.rs:21
N_ISOTOPES = 3              # lfq.rs:23
SLACK = 75                  # lfq.rs:350
BIN_SIZE = 16 * 1024        # lfq.rs:176, 190
NEUTRON = f32(1.00335)      # mass.rs:7
DECOY_SHIFT = f32(11.06)    # lfq.rs:156

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.expf.restype = ctypes.c_float
_libm.expf.argtypes = [ctypes.c_float]


def expf(x):
    """f32::exp of every element: the C library's expf, called once per distinct value."""
    x = np.asarray(x, f32)
    u, inv = np.unique(x, return_inverse=True)
    return np.array([_libm.expf(float(v)) for v in u], f32)[inv].reshape(x.shape)


def _acos(x: float) -> float:
    return math.acos(x) if -1.0 <= x <= 1.0 else math.nan   # libm acos: NaN outside [-1, 1] (math.acos raises instead)


def acos(x):
    x = np.asarray(x, np.float64)
    u, inv = np.unique(x, return_inverse=True)
    return np.array([_acos(float(v)) for v in u], np.float64)[inv].reshape(x.shape)


def total_key(x):
    """f32::total_cmp as a signed integer key."""
    b = np.asarray(x, f32).view(np.int32).astype(np.int64)
    return b ^ ((b >> 31) & 0x7FFFFFFF)


def search_slice(keys, low, high):
    """binary_search_slice (database.rs:549-561) over total-order keys: left = partition_point(< low) - 1 saturating, right = left +
    partition_point of slice[left..] (<= high)."""
    left = np.maximum(np.searchsorted(keys, low, side="left") - 1, 0)
    right = np.maximum(np.searchsorted(keys, high, side="right"), left)
    return left, right


# ---------------------------------------------------------------------------------------------------- composition and isotopes
_C = dict(A=3, R=6, N=4, D=4, C=3, E=5, Q=5, G=2, H=6, I=6, L=6, K=6, M=5, F=9, P=5, S=3, T=4, W=11, Y=9, V=5, U=3, O=12)   # mass.rs:78-104
_S = dict(C=1, M=1)
CARBON = np.zeros(256, np.int64)
SULFUR = np.zeros(256, np.int64)
for _aa, _n in _C.items():
    CARBON[ord(_aa)] = _n
for _aa, _n in _S.items():
    SULFUR[ord(_aa)] = _n


def composition(seq: np.ndarray):
    """Composition summed over a sequence (mass.rs:118-128, u16 fields)."""
    s = np.asarray(seq, np.uint8)
    return int(CARBON[s].sum()) & 0xFFFF, int(SULFUR[s].sum()) & 0xFFFF


def _powi(x, k):
    """f32::powi for k = 0..3: 1, x, x*x, x*(x*x), the square-and-multiply expansion."""
    return [np.ones_like(x), x, x * x, x * (x * x)][k]


def _convolve4(a, b):
    """isotopes.rs:2-10"""
    return [a[0] * b[0], a[0] * b[1] + a[1] * b[0], a[0] * b[2] + a[1] * b[1] + a[2] * b[0],
            a[0] * b[3] + a[1] * b[2] + a[2] * b[1] + a[3] * b[0]]


def peptide_isotopes(carbons, sulfurs):
    """peptide_isotopes (isotopes.rs:43-50) in f32, elementwise over broadcastable count arrays -> [..., 3]."""
    carbons, sulfurs = np.broadcast_arrays(np.asarray(carbons, np.int64), np.asarray(sulfurs, np.int64))
    fact = [f32(1), f32(1), f32(2), f32(6)]
    lc = carbons.astype(f32) * f32(0.011)                                           # isotopes.rs:13
    ec = expf(-lc)
    c13 = [_powi(lc, k) * ec / fact[k] for k in range(4)]                           # isotopes.rs:17-19
    l33, l35 = sulfurs.astype(f32) * f32(0.0076), sulfurs.astype(f32) * f32(0.044)  # isotopes.rs:24-25
    e33, e35 = expf(-l33), expf(-l35)
    zero = np.zeros_like(l35)
    s35 = [_powi(l35, 0) * e35, zero, _powi(l35, 1) * e35, zero]                    # isotopes.rs:27-33
    s33 = [_powi(l33, k) * e33 / fact[k] for k in range(4)]                         # isotopes.rs:36-38
    c = _convolve4(c13, _convolve4(s33, s35))                                       # isotopes.rs:40, 46
    mx = np.fmax(np.fmax(c[0], c[1]), c[2])                                         # isotopes.rs:47
    return np.stack([c[0] / mx, c[1] / mx, c[2] / mx], axis=-1)


# ---------------------------------------------------------------------------------------------------- feature map
def tol_bounds(lo, hi, center, divisor):
    """Tolerance::Ppm (divisor 1e6) / Tolerance::Pct (divisor 100) bounds (mass.rs:21-31)."""
    center = np.asarray(center, f32)
    return center + center * lo / f32(divisor), center + center * hi / f32(divisor)


def build_map(settings, precursor_charge, features):
    """build_feature_map (lfq.rs:94-193) -> (ranges as LFQ_RANGE_DTYPE, min_rts)."""
    col = lambda k, t: np.asarray(features[k], t)   # noqa: E731
    kept = np.nonzero((col("peptide_q", f32) <= f32(settings.peptide_q_value)) & (col("label", np.int32) == 1))[0]   # lfq.rs:102
    peps, first = np.unique(col("peptide_idx", np.uint32)[kept], return_index=True)                              # lfq.rs:105: first row wins
    row = kept[first]
    rt, mono, fid, ims = col("aligned_rt", f32)[row], col("calcmass", f32)[row], col("file_id", np.uint32)[row], col("ims", f32)[row]
    mt = f32(settings.mobility_pct_tolerance)
    mob_lo, mob_hi = tol_bounds(-mt, mt, ims, 100.0)                                                            # lfq.rs:111-115
    charges = np.arange(precursor_charge[0], precursor_charge[1] + 1)
    n, nc = len(peps), len(charges)
    shape = (n, nc, N_ISOTOPES, 2)                                                                               # pre-sort order
    r = np.zeros(shape, LFQ_RANGE_DTYPE)
    mass = (mono[:, None, None] + np.arange(N_ISOTOPES).astype(f32)[None, None, :] * NEUTRON) / charges.astype(f32)[None, :, None]   # lfq.rs:140
    ppm = f32(settings.ppm_tolerance)
    r["mass_lo"][..., 0], r["mass_hi"][..., 0] = tol_bounds(-ppm, ppm, mass, 1e6)                                # lfq.rs:141-143
    r["mass_lo"][..., 1], r["mass_hi"][..., 1] = tol_bounds(-ppm, ppm, mass + DECOY_SHIFT, 1e6)                  # lfq.rs:154-156
    r["rt"][..., 0] = rt[:, None, None]
    r["rt"][..., 1] = np.fmax(rt - RT_TOL * f32(2.0), f32(0.0))[:, None, None]                                  # lfq.rs:159: f32::max ignores NaN
    r["mobility_lo"] = mob_lo[:, None, None, None]
    r["mobility_hi"] = mob_hi[:, None, None, None]
    r["peptide"] = peps[:, None, None, None]
    r["file_id"] = fid[:, None, None, None]
    r["charge"] = charges[None, :, None, None]
    r["isotope"] = np.arange(N_ISOTOPES)[None, None, :, None]
    r["decoy"] = np.arange(2)[None, None, None, :]
    r = r.ravel()
    r = r[np.argsort(total_key(r["rt"]), kind="stable")]                                                         # lfq.rs:174
    min_rts = []
    for c in range(0, len(r), BIN_SIZE):                                                                         # lfq.rs:175-184
        min_rts.append(r["rt"][c])
        page = r[c:c + BIN_SIZE]
        r[c:c + BIN_SIZE] = page[np.argsort(total_key(page["mass_lo"]), kind="stable")]
    return r, np.array(min_rts, f32)


def gaussian_kernel(sigma: float, n: int):
    """lfq.rs:614-628"""
    step = 2.0 / (n - 1)
    constant = 1.0 / (sigma * math.sqrt(2.0 * math.pi))
    k = []
    for i in range(n):
        xs = (i * step - 1.0) / sigma
        k.append(constant * math.exp(-0.5 * (xs * xs)))
    s = 0.0
    for v in k:
        s = s + v
    return [v / s for v in k]


class LfqReference:
    """build_feature_map + FeatureMap::quantify. Arguments as sage_b200.FeatureMap.build; `peptides` needs seq_off and seq."""

    def __init__(self, peptides, settings, precursor_charge, features, alignments):
        self.settings = settings
        self.combine = bool(settings.combine_charge_states)
        self.ranges, self.min_rts = build_map(settings, precursor_charge, features)
        al = np.ascontiguousarray(alignments)
        self.align = al.view(f32).reshape(-1, 3) if al.dtype.names else np.asarray(al, f32).reshape(-1, 3)
        self.n_files = len(self.align)
        self.seq_off = np.asarray(peptides.seq_off, np.int64)
        self.seq = np.asarray(peptides.seq, np.uint8)
        self.grids = {}       # (PeptideIx, charge or 0, decoy) -> [n_files * 3, 100] f64 (lfq.rs:232, 250-262)
        self.grid_info = {}   # key -> (reference_file_id, distribution)
        self.matches = 0      # add_entry calls
        self._page_keys = [total_key(self.ranges["mass_lo"][c:c + BIN_SIZE]) for c in range(0, len(self.ranges), BIN_SIZE)]

    def add_ms1(self, batch):
        """The tracing loop of quantify (lfq.rs:239-287) over one batch, spectra and peaks in order."""
        off = np.asarray(batch.peak_off, np.int64)
        n = len(batch.file_id)
        if n == 0 or len(self.ranges) == 0:
            return
        fid = np.asarray(batch.file_id, np.int64)
        a = self.align[fid]
        rt = (np.asarray(batch.scan_start_time, f32) / a[:, 0]) * a[:, 1] + a[:, 2]                           # lfq.rs:241
        min_rt, max_rt = rt - RT_TOL, rt + RT_TOL                                                               # lfq.rs:209-210, 218-219
        page_lo, page_hi = search_slice(total_key(self.min_rts), total_key(min_rt), total_key(max_rt))       # lfq.rs:206-211
        peak = np.arange(off[0], off[-1])
        spec = np.repeat(np.arange(n), np.diff(off))
        masses = np.asarray(batch.masses, f32)
        mob = None if batch.mobilities is None else np.asarray(batch.mobilities, f32)
        found_peak, found_pos = [], []
        for page, keys in enumerate(self._page_keys):                                                          # lfq.rs:650
            on = (page_lo[spec] <= page) & (page < page_hi[spec])
            pk = peak[on]
            m = masses[pk]
            il, ir = search_slice(keys, total_key(m - f32(0.1)), total_key(m + f32(0.1)))                      # lfq.rs:660-665
            cnt = ir - il
            pk = np.repeat(pk, cnt)
            pos = np.repeat(il - np.cumsum(cnt) + cnt, cnt) + np.arange(int(cnt.sum())) + page * BIN_SIZE
            e = self.ranges[pos]
            m, s = masses[pk], spec[pk - off[0]]
            ok = (e["rt"] <= max_rt[s]) & (e["rt"] >= min_rt[s]) & (m >= e["mass_lo"]) & (m <= e["mass_hi"])    # lfq.rs:668-673
            if mob is not None:
                ok &= (e["mobility_hi"] >= mob[pk]) & (e["mobility_lo"] <= mob[pk])                            # lfq.rs:682-685
            found_peak.append(pk[ok])
            found_pos.append(pos[ok])
        pk, pos = np.concatenate(found_peak), np.concatenate(found_pos)
        order = np.lexsort((pos, pk))                                                                           # peaks in order, then map position
        pk, pos = pk[order], pos[order]
        self.matches += len(pk)
        if len(pk) == 0:
            return
        e = self.ranges[pos]
        s = spec[pk - off[0]]
        # the grid of each entry (lfq.rs:245-262)
        charge = np.zeros(len(e), np.int64) if self.combine else e["charge"].astype(np.int64)
        key = (e["peptide"].astype(np.int64) << 9) | (charge << 1) | e["decoy"].astype(np.int64)
        ukey, first, gi = np.unique(key, return_index=True, return_inverse=True)
        for k, j in zip(ukey.tolist(), first.tolist()):
            t = (k >> 9, (k >> 1) & 0xFF, k & 1)
            if t not in self.grids:
                pep = t[0]
                c, su = composition(self.seq[self.seq_off[pep]:self.seq_off[pep + 1]])
                self.grids[t] = np.zeros((self.n_files * N_ISOTOPES, GRID_SIZE))
                self.grid_info[t] = (int(e["file_id"][j]), peptide_isotopes(c, su))
        # Grid::add_entry (lfq.rs:538-550); rt_min = entry.rt - RT_TOL (lfq.rs:528), the same for every entry of one grid
        rt_step = (RT_TOL * f32(2.0)) / f32(GRID_SIZE)                                                          # lfq.rs:525
        rt_min = e["rt"] - RT_TOL
        srt = rt[s]
        with np.errstate(invalid="ignore"):
            x = np.floor((srt - rt_min) / rt_step)
            lo = np.where(x > 0, np.minimum(x, f32(GRID_SIZE - 1)), f32(0)).astype(np.int64)                    # `as usize` saturates, NaN -> 0
        hi = np.minimum(lo + 1, GRID_SIZE - 1)
        interp = (srt - (lo.astype(f32) * rt_step + rt_min)) / rt_step
        inten = np.asarray(batch.intensities, f32)[pk]
        row = fid[s] * N_ISOTOPES + e["isotope"].astype(np.int64)
        cells = GRID_SIZE * N_ISOTOPES * self.n_files
        cell = np.stack([gi * cells + row * GRID_SIZE + lo, gi * cells + row * GRID_SIZE + hi], axis=1).ravel()
        val = np.stack([((f32(1.0) - interp) * inten).astype(np.float64), (interp * inten).astype(np.float64)], axis=1).ravel()
        stack = np.stack([self.grids[(k >> 9, (k >> 1) & 0xFF, k & 1)] for k in ukey.tolist()]).ravel()
        # each cell adds its contributions in sequence: the r-th contribution of every cell in round r
        order = np.argsort(cell, kind="stable")
        cs = cell[order]
        start = np.r_[0, np.nonzero(np.diff(cs))[0] + 1]
        rank = np.arange(len(cs)) - np.repeat(start, np.diff(np.r_[start, len(cs)]))
        by_rank = np.argsort(rank, kind="stable")
        bounds = np.searchsorted(rank[by_rank], np.arange(rank.max() + 2))
        for r_ in range(rank.max() + 1):
            j = order[by_rank[bounds[r_]:bounds[r_ + 1]]]
            stack[cell[j]] = stack[cell[j]] + val[j]
        stack = stack.reshape(len(ukey), self.n_files * N_ISOTOPES, GRID_SIZE)
        for i, k in enumerate(ukey.tolist()):
            self.grids[(k >> 9, (k >> 1) & 0xFF, k & 1)] = stack[i]

    def export_grids(self):
        """keys [n, 3] in (id, decoy) order and the matrices [n, n_files * 3, 100]."""
        keys = sorted(self.grids)
        mats = np.stack([self.grids[k] for k in keys]) if keys else np.zeros((0, self.n_files * 3, GRID_SIZE))
        return np.array(keys, np.uint32).reshape(-1, 3), mats

    def quantify(self):
        """summarize_traces + integrate (lfq.rs:290-304) for every grid, in (id, decoy) order. Returns present, rt, spectral_angle, score,
        areas [n, n_files] and warps [n, n_files], the time warps find_time_warps chose."""
        keys, mats = self.export_grids()
        F = self.n_files
        out = dict(id=keys[:, 0].copy(), charge=keys[:, 1].astype(np.uint8), decoy=keys[:, 2].astype(bool))
        res = [self._integrate(mats[a:a + 64], [self.grid_info[tuple(k)] for k in keys[a:a + 64].tolist()]) for a in range(0, len(keys), 64)]
        for f, dt, shape in (("present", bool, ()), ("rt", np.uint32, ()), ("spectral_angle", np.float64, ()), ("score", np.float64, ()),
                             ("areas", np.float64, (F,)), ("warps", np.int64, (F,))):
            out[f] = np.concatenate([r[f] for r in res]) if res else np.zeros((0,) + shape, dt)
        return out

    def _integrate(self, mats, info):
        s = self.settings
        G, F, C = len(mats), self.n_files, GRID_SIZE
        m = mats.reshape(G, F, N_ISOTOPES, C)
        ref = np.array([i[0] for i in info])
        dist = np.stack([i[1] for i in info]).astype(f32)
        k = gaussian_kernel(0.5, K_WIDTH)                                                                       # lfq.rs:559
        # convolve (lfq.rs:632-646), every row at once
        n = K_WIDTH - K_WIDTH // 2
        conv = np.zeros_like(m)
        for idx in range(C):
            ks, ws = max(K_WIDTH - (n + idx), 0), max(idx - (n - 1), 0)
            acc = np.zeros(m.shape[:3])
            for t in range(min(C - ws, K_WIDTH - ks)):
                acc = acc + m[..., ws + t] * k[ks + t]
            conv[..., idx] = acc
        # summarize_traces (lfq.rs:558-610)
        ss_dist = np.sqrt(dist[:, 0] * dist[:, 0] + dist[:, 1] * dist[:, 1] + dist[:, 2] * dist[:, 2]).astype(np.float64)   # lfq.rs:571-576
        dot = np.zeros((G, F, C))
        ssq = np.zeros((G, F, C))
        for iso in range(N_ISOTOPES):
            dot = dot + conv[:, :, iso, :] * dist[:, iso].astype(np.float64)[:, None, None]
            ssq = ssq + conv[:, :, iso, :] * conv[:, :, iso, :]
        with np.errstate(divide="ignore", invalid="ignore"):
            sim = np.where(ssq > 0.0, dot / (np.sqrt(ssq) * ss_dist[:, None, None]), 0.0)
        sa = 1.0 - 2.0 * acos(sim) / math.pi                                                                    # lfq.rs:600
        # find_time_warps (lfq.rs:361-385): dot products of every shift, each summed over i in order
        refrow = dot[np.arange(G), ref]
        wd = np.zeros((G, F, 2 * SLACK + 1))
        for i in range(C):
            o_lo, o_hi = max(-SLACK, -i), min(SLACK, C - 1 - i)
            wd[:, :, o_lo + SLACK:o_hi + SLACK + 1] += refrow[:, None, i, None] * dot[:, :, i + o_lo:i + o_hi + 1]
        warps = np.zeros((G, F), np.int64)
        best = np.zeros((G, F))
        for o in range(2 * SLACK + 1):
            up = wd[:, :, o] >= best
            warps[up] = o - SLACK
            best[up] = wd[:, :, o][up]
        # apply_time_warps (lfq.rs:388-400)
        j = np.arange(C)[None, None, :] + warps[:, :, None]
        ok = (j >= 0) & (j < C)
        jc = np.clip(j, 0, C - 1)
        sa = np.where(ok, np.take_along_axis(sa, jc, axis=2), 0.0)
        dot = np.where(ok, np.take_along_axis(dot, jc, axis=2), 0.0)
        # scores (lfq.rs:402-437)
        summed = np.ones((G, C))
        weighted = np.zeros((G, C))
        for f in range(F):
            weighted = weighted + sa[:, f, :] * dot[:, f, :]
            summed = summed + dot[:, f, :]
        with np.errstate(divide="ignore", invalid="ignore"):
            spectral = weighted / summed
            mx = np.zeros(G)
            for col in range(C):
                mx = np.fmax(mx, summed[:, col])
            center = C // 2
            rtf = np.array([math.pow(1.0 - (abs(col - center) / center), 0.33) for col in range(C)])
            if s.peak_scoring == "RetentionTime":
                scores = np.broadcast_to(rtf, (G, C)).copy()
            elif s.peak_scoring == "SpectralAngle":
                scores = spectral.copy()
            elif s.peak_scoring == "Intensity":
                scores = np.sqrt(summed / mx[:, None])
            else:
                scores = spectral * (spectral * spectral) * rtf[None, :] * np.sqrt(summed / mx[:, None])
        # integrate (lfq.rs:447-509)
        thr_sa = float(s.spectral_angle)
        best = np.zeros(G)
        brt = np.zeros(G, np.int64)
        for col in range(C):
            up = (scores[:, col] > best) & (spectral[:, col] >= thr_sa)
            best[up] = scores[:, col][up]
            brt[up] = col
        g = np.arange(G)
        left, right = np.maximum(brt - 1, 0), brt + 1
        threshold = best * 0.50
        llim, rlim = np.maximum(brt - C // 5, 0), np.minimum(C - 1, brt + 20)
        go = np.ones(G, bool)
        while go.any():
            go &= (left > llim) & (scores[g, left] >= threshold) & (spectral[g, left] >= thr_sa)
            left -= go
        go = np.ones(G, bool)
        while go.any():
            go &= (right < rlim) & (scores[g, np.minimum(right, C - 1)] >= threshold) & (spectral[g, np.minimum(right, C - 1)] >= thr_sa)
            right += go
        if s.integration == "Sum":
            areas = np.zeros((G, F))
            for i in range(C):
                inside = ((i >= left) & (i < right))[:, None]
                areas = np.where(inside, areas + dot[:, :, i], areas)
        else:
            areas = dot[g, :, brt]
        present = best != 0.0
        return dict(present=present, rt=np.where(present, brt, 0).astype(np.uint32), spectral_angle=np.where(present, spectral[g, brt], 0.0),
                    score=np.where(present, best, 0.0), areas=np.where(present[:, None], areas, 0.0), warps=warps)

    def touched(self):
        return sorted(self.grids)
