"""CPU checks of label-free quantification: the CPU oracle (oracle_lfq/) against the reference's known answer and against an independent
numpy restatement of lfq.rs on a hand-sized case, and the C header's LFQ structs against their ctypes mirrors."""
import math
import os
import subprocess

import numpy as np
import pytest

from oracle_lfq import lfq_oracle as LO
from sage_b200 import api
from sage_b200.api import ALIGNMENT_DTYPE, LfqSettings, Ms1Batch, Peptides

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
RT_TOL = f32(0.005)
STEP = f32(RT_TOL * f32(2.0)) / f32(100.0)


def test_peptide_isotopes_known_answer():
    # isotopes.rs:56-65
    iso = LO.peptide_isotopes(60, 5)
    expected = np.array([0.3972, 0.2824, 0.1869]) / 0.3972
    assert np.all(np.abs(iso - expected) <= 0.02), iso


def test_lfq_struct_layouts_match_header(tmp_path):
    import ctypes as C
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "%s"\nint main(){printf("%%zu %%zu %%zu %%zu %%zu %%zu %%zu\\n", sizeof(sage_b200_lfq_params),'
                   'sizeof(sage_b200_lfq_features), sizeof(sage_b200_alignment), sizeof(sage_b200_ms1), sizeof(sage_b200_lfq_range),'
                   'sizeof(sage_b200_lfq_row), sizeof(sage_b200_lfq_info));return 0;}\n' % os.path.join(ROOT, "include", "sage_b200.h"))
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", str(src), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(api.CLfqParams), C.sizeof(api.CLfqFeatures), ALIGNMENT_DTYPE.itemsize, C.sizeof(api.CMs1), api.LFQ_RANGE_DTYPE.itemsize,
                     api.LFQ_ROW_DTYPE.itemsize, C.sizeof(api.CLfqInfo)]


# ---------------------------------------------------------------------------------------------------- independent numpy restatement
def np_isotopes(c, s):
    fact = [f32(1), f32(1), f32(2), f32(6)]
    powi = lambda x, k: [f32(1), x, x * x, x * (x * x)][k]  # noqa: E731
    lc, l33, l35 = f32(c) * f32(0.011), f32(s) * f32(0.0076), f32(s) * f32(0.044)
    c13 = [powi(lc, k) * np.exp(-lc) / fact[k] for k in range(4)]
    s33 = [powi(l33, k) * np.exp(-l33) / fact[k] for k in range(4)]
    s35 = [f32(1) * np.exp(-l35), f32(0), l35 * np.exp(-l35), f32(0)]

    def conv(a, b):
        return [a[0] * b[0], a[0] * b[1] + a[1] * b[0], a[0] * b[2] + a[1] * b[1] + a[2] * b[0]]
    sc = conv(s33, s35) + [s33[0] * s35[3] + s33[1] * s35[2] + s33[2] * s35[1] + s33[3] * s35[0]]
    cc = conv(c13, sc)
    mx = max(cc[0], cc[1], cc[2])
    return [x / mx for x in cc]


def np_add_entry(mat, rt_min, rt, iso, file, inten):
    x = np.floor((rt - rt_min) / STEP)
    lo = 0 if not x > 0 else int(x)
    lo = min(lo, 99)
    hi = min(lo + 1, 99)
    interp = (rt - (f32(lo) * STEP + rt_min)) / STEP
    mat[file * 3 + iso, lo] += float(f32((f32(1) - interp) * inten))
    mat[file * 3 + iso, hi] += float(f32(interp * inten))
    return lo


def np_integrate(mat, dist, ref, n_files, scoring, integration, sa_thr):
    sig = 0.5
    step = 2.0 / 9.0
    const = 1.0 / (sig * math.sqrt(2.0 * math.pi))
    k = [const * math.exp(-0.5 * ((i * step - 1.0) / sig) ** 2) for i in range(10)]
    tot = 0.0
    for v in k:
        tot += v
    k = [v / tot for v in k]

    def convolve(row):
        out = []
        for idx in range(100):
            ks, ws = max(10 - (5 + idx), 0), max(idx - 4, 0)
            acc = 0.0
            for x, y in zip(row[ws:], k[ks:]):
                acc = acc + x * y
            out.append(acc)
        return out
    ss_dist = float(np.sqrt(dist[0] * dist[0] + dist[1] * dist[1] + dist[2] * dist[2]))
    sa = np.zeros((n_files, 100))
    dot = np.zeros((n_files, 100))
    for f in range(n_files):
        ssq = [0.0] * 100
        acc = [0.0] * 100
        for iso in range(3):
            cv = convolve(list(mat[f * 3 + iso]))
            for c in range(100):
                acc[c] += cv[c] * float(dist[iso])
                ssq[c] += cv[c] * cv[c]
        for c in range(100):
            sim = acc[c] / (math.sqrt(ssq[c]) * ss_dist) if ssq[c] > 0 else 0.0
            sa[f, c] = 1.0 - 2.0 * math.acos(sim) / math.pi
            dot[f, c] = acc[c]
    warps = []
    for f in range(n_files):
        best = (0, 0.0)
        for off in range(-75, 76):
            d = 0.0
            for i in range(100):
                j = i + off
                if 0 <= j < 100:
                    d += dot[ref, i] * dot[f, j]
            if d >= best[1]:
                best = (off, d)
        warps.append(best[0])
    for m in (sa, dot):
        for f in range(n_files):
            row = m[f].copy()
            m[f] = [row[i + warps[f]] if 0 <= i + warps[f] < 100 else 0.0 for i in range(100)]
    spectral, inten = [], []
    for c in range(100):
        s, w = 1.0, 0.0
        for f in range(n_files):
            w += sa[f, c] * dot[f, c]
            s += dot[f, c]
        spectral.append(w / s)
        inten.append(s)
    mx = 0.0
    for v in inten:
        mx = max(mx, v)
    scores = []
    for c in range(100):
        rtf = (1.0 - abs(c - 50) / 50.0) ** 0.33
        s = spectral[c]
        scores.append({"RetentionTime": rtf, "SpectralAngle": s, "Intensity": math.sqrt(inten[c] / mx),
                       "Hybrid": s * (s * s) * rtf * math.sqrt(inten[c] / mx)}[scoring])
    best, brt = 0.0, 0
    for c in range(100):
        if scores[c] > best and spectral[c] >= sa_thr:
            best, brt = scores[c], c
    if best == 0.0:
        return None, warps
    left, right = max(brt - 1, 0), brt + 1
    while left > max(brt - 20, 0) and scores[left] >= best * 0.5 and spectral[left] >= sa_thr:
        left -= 1
    while right < min(99, brt + 20) and scores[right] >= best * 0.5 and spectral[right] >= sa_thr:
        right += 1
    areas = []
    for f in range(n_files):
        if integration == "Sum":
            a = 0.0
            for i in range(left, right):
                a += dot[f, i]
            areas.append(a)
        else:
            areas.append(dot[f, brt])
    return dict(rt=brt, score=best, spectral_angle=spectral[brt], areas=areas), warps


def _rt_below_bin_zero(r_rt):
    """An f32 spectrum RT that passes the filter (r_rt <= rt + RT_TOL) yet lies before the grid's first bin (rt < r_rt - RT_TOL)."""
    rt_min = f32(r_rt - RT_TOL)
    x = rt_min
    for _ in range(64):
        x = np.nextafter(x, f32(0))
        if r_rt <= f32(x + RT_TOL):
            return x
    return None


def hand_case():
    seq = b"PEPTCIDEMK"
    pep = Peptides(seq_off=np.array([0, len(seq)], np.uint32), seq=np.frombuffer(seq, np.uint8).copy(), mods=np.zeros(len(seq), f32),
                   nterm=np.full(1, np.nan, f32), mono=np.array([1176.5], f32), decoy=np.zeros(1, np.uint8), missed=np.zeros(1, np.uint8))
    r_rt = None
    for cand in np.arange(0.3, 0.7, 0.001, dtype=f32):
        x = _rt_below_bin_zero(cand)
        if x is not None:
            r_rt, neg_rt = cand, x
            break
    assert r_rt is not None
    feats = dict(peptide_idx=np.array([0, 0], np.uint32), peptide_q=np.array([0.001, 0.0], f32), label=np.array([1, 1], np.int32),
                 aligned_rt=np.array([r_rt, 0.1], f32), calcmass=pep.mono[[0, 0]], file_id=np.array([0, 1], np.uint32), ims=np.zeros(2, f32))
    align = np.zeros(2, ALIGNMENT_DTYPE)
    align["max_rt"], align["slope"], align["intercept"] = 1.0, 1.0, 0.0
    clamp_rt = f32(r_rt + f32(0.00499))       # bin_lo 99: both contributions land in bin 99
    rts = [neg_rt, f32(r_rt - f32(0.0021)), f32(r_rt - f32(0.0003)), r_rt, f32(r_rt + f32(0.0012)), clamp_rt]
    mz = [f32((pep.mono[0] + f32(k) * f32(1.00335)) / f32(2)) for k in range(3)]
    masses, intens, off = [], [], [0]
    for i, _ in enumerate(rts):
        m = np.array(sorted([f32(200.0)] + mz + [f32(mz[1] + f32(0.05))]), f32)   # a noise peak and one outside the ppm window
        masses.append(m)
        intens.append(np.array([1000.0 * (i + 1) + 7 * j for j in range(len(m))], f32))
        off.append(off[-1] + len(m))
    batch = Ms1Batch(np.array(off, np.uint64), np.concatenate(masses), np.concatenate(intens), np.zeros(len(rts), np.uint32), np.array(rts, f32))
    return pep, feats, align, batch, r_rt


@pytest.mark.parametrize("scoring", ["RetentionTime", "SpectralAngle", "Intensity", "Hybrid"])
@pytest.mark.parametrize("integration", ["Apex", "Sum"])
def test_hand_sized_case_against_numpy(scoring, integration):
    pep, feats, align, batch, r_rt = hand_case()
    settings = LfqSettings(peak_scoring=scoring, integration=integration, spectral_angle=0.0)
    o = LO.LfqOracle(pep, settings, (2, 2), feats, align)
    ranges, min_rts = o.export_map()
    assert len(ranges) == 6 and np.all(np.diff(ranges["mass_lo"]) >= 0)   # one page: sorted by mass_lo
    assert min_rts.tolist() == [f32(max(f32(r_rt - f32(0.01)), f32(0)))]    # its first entry in RT order is a decoy
    o.add_ms1(batch)
    keys, mats = o.export_grids()
    assert keys.tolist() == [[0, 0, 0]]                    # the decoy ranges sit 11.06 Da higher: no peak reaches them

    # grid, recomputed here
    mat = np.zeros((6, 100))
    dist = np_isotopes(5 + 5 + 5 + 4 + 3 + 6 + 4 + 5 + 5 + 6, 2)   # carbons of P E P T C I D E M K, sulfurs of C and M (mass.rs:78-104)
    lows = []
    for s in range(len(batch)):
        for p in range(int(batch.peak_off[s]), int(batch.peak_off[s + 1])):
            m, inten = batch.masses[p], batch.intensities[p]
            for r in ranges:
                if r["rt"] <= f32(batch.scan_start_time[s] + RT_TOL) and r["rt"] >= f32(batch.scan_start_time[s] - RT_TOL) and r["mass_lo"] <= m <= r["mass_hi"] \
                        and not r["decoy"]:
                    lows.append(np_add_entry(mat, f32(r["rt"] - RT_TOL), batch.scan_start_time[s], int(r["isotope"]), 0, inten))
    assert 0 in lows and 99 in lows                        # the below-the-grid spectrum saturates to bin 0; the last one is clamped to 99
    assert mats[0].tobytes() == mat.tobytes()

    q = o.quantify()
    want, warps = np_integrate(mat, dist, 0, 2, scoring, integration, 0.0)
    assert warps[1] == 75                                  # file 1 has no signal: the last of the equal (zero) dot products wins
    assert q["present"][0] == (want is not None)
    if want is not None:
        assert q["rt"][0] == want["rt"]
        assert q["score"][0] == want["score"] and q["spectral_angle"][0] == want["spectral_angle"]
        assert q["areas"][0].tolist() == want["areas"]
