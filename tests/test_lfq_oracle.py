"""CPU checks of label-free quantification: the CPU oracle (oracle_lfq/) against the reference's known answer and against an independent
numpy restatement of lfq.rs (tests/lfq_reference.py) on a hand-sized case, and the C header's LFQ structs against their ctypes mirrors."""
import os
import subprocess

import numpy as np
import pytest

from lfq_reference import LfqReference, peptide_isotopes
from oracle_lfq import lfq_oracle as LO
from sage_b200 import api
from sage_b200.api import ALIGNMENT_DTYPE, LfqSettings, Ms1Batch, Peptides

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
RT_TOL = f32(0.005)


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


# ---------------------------------------------------------------------------------------------------- a hand-sized case
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

    # the same case through the independent restatement (tests/lfq_reference.py)
    ref = LfqReference(pep, settings, (2, 2), feats, align)
    ref.add_ms1(batch)
    rk, rm = ref.export_grids()
    assert rk.tolist() == keys.tolist()
    assert rm[0][:, 0].any() and rm[0][:, 99].any()      # the below-the-grid spectrum saturates to bin 0; the last one is clamped to 99
    assert mats[0].tobytes() == rm[0].tobytes()
    assert ref.grid_info[(0, 0, 0)][1].tolist() == peptide_isotopes(5 + 5 + 5 + 4 + 3 + 6 + 4 + 5 + 5 + 6, 2).tolist()   # P E P T C I D E M K

    q = o.quantify()
    want = ref.quantify()
    assert want["warps"][0, 1] == 75                     # file 1 has no signal: the last of the equal (zero) dot products wins
    assert q["present"][0] == want["present"][0]
    if want["present"][0]:
        assert q["rt"][0] == want["rt"][0]
        assert q["score"][0] == want["score"][0] and q["spectral_angle"][0] == want["spectral_angle"][0]
        assert q["areas"][0].tolist() == want["areas"][0].tolist()
