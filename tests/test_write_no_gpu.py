"""Result-file text without a GPU: the Python restatement (tests/write_reference.py, digits from repr / numpy) and the C++ oracle
(oracle_ml/ml_oracle.cpp, digits from std::to_chars) agree on values, fields and whole files, and sage_b200_write_tsv rejects bad arguments
before it looks for a device."""
import ctypes as C
import os
import struct
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import write_reference as W  # noqa: E402
from oracle_ml import ml_oracle as M  # noqa: E402
from sage_b200 import api  # noqa: E402

FMT = {"f32": 0, "plus": 1, "f64": 2}


def edge_f64():
    xs = [0.0, -0.0, float("nan"), float("inf"), float("-inf"), 5e-324, -5e-324, 2.2250738585072014e-308, 2.225073858507201e-308, 1.7976931348623157e308]
    xs += [float("1e%d" % e) for e in range(-323, 309)]
    for kk in (16, 17, -4, -5):   # values whose kk = len + k is the threshold, one past it, and the ends of the 0.000d form
        xs += [1.2345 * 10.0 ** (kk - 1), 10.0 ** (kk - 1), 9.5 * 10.0 ** (kk - 1)]
    return np.array(xs)


def edge_f32():
    xs = [struct.unpack("<f", struct.pack("<I", u))[0] for u in (0, 0x80000000, 0x7fc00000, 0x7f800000, 0xff800000, 1, 0x80000001, 0x007fffff,
                                                                  0x00800000, 0x7f7fffff)]
    xs += [float(np.float32("1e%d" % e)) for e in range(-45, 39)]
    for kk in (13, 14, -4, -5):
        xs += [1.2345 * 10.0 ** (kk - 1), 10.0 ** (kk - 1), 9.5 * 10.0 ** (kk - 1)]
    return np.array(xs)


@pytest.mark.parametrize("kind,value,text", W.KNOWN_ANSWERS)
def test_known_answers(kind, value, text):
    assert (W.plus(value) if kind == "plus" else W.ryu(value, 64 if kind == "f64" else 32)) == text
    assert M.format_one(FMT[kind], value) == text


def test_f64_restatement_equals_oracle():
    rng = np.random.default_rng(17)
    x = np.concatenate([rng.integers(0, 1 << 64, 1_000_000, dtype=np.uint64).view(np.float64), edge_f64()])
    want = b"".join(W.ryu(float(v), 64).encode() + b"\n" for v in x)
    block = len(x)
    assert M.format_hashes(2, values=x, block=block)[0] == fnv(want)


def test_f32_restatement_equals_oracle():
    rng = np.random.default_rng(18)
    bits = rng.integers(0, 1 << 32, 1_000_000, dtype=np.uint64).astype(np.uint32)
    x = np.concatenate([bits.view(np.float32).astype(np.float64), edge_f32()])
    for fmt, f in ((0, lambda v: W.ryu(v, 32)), (1, W.plus)):
        got = [M.format_one(fmt, v) for v in x]
        want = [f(float(v)) for v in x]
        bad = [(v, g, w) for v, g, w in zip(x, got, want) if g != w]
        assert not bad, bad[:5]


def fnv(b: bytes) -> int:
    h = 0xcbf29ce484222325
    for c in b:
        h = ((h ^ c) * 0x100000001b3) & 0xffffffffffffffff
    return h


def test_format_hashes_fold_in_value_order():
    x = np.array([1.5, -0.0, 1e300])
    assert M.format_hashes(2, values=x, block=3)[0] == fnv(b"1.5\n-0.0\n1e300\n")


QUOTED = [b"plain.mzML", b"tab\there", b'say "hi"', b"cr\rlf\n", b"", b'"', b"scan=12 controllerType=0"]


@pytest.mark.parametrize("s", QUOTED)
def test_field_quoting(s):
    assert M.format_one(3, s=s).encode("latin-1") == W.field(s)


def test_tmt_file_oracle_equals_restatement():
    rng = np.random.default_rng(3)
    files = [b"a.mzML", b'we"ird\tname.mzML']
    ids = [b"controllerType=0 scan=%d" % i for i in range(20)] + [b"id\nwith newline"]
    n = 40
    fi, si = rng.integers(0, 2, n), rng.integers(0, len(ids), n)
    inj = rng.random(n).astype(np.float32) * 50
    peaks = (rng.random((n, 6)) * 1e6).astype(np.float32)
    peaks[0, :] = [0.0, -0.0, np.nan, np.inf, 1e-45, 3.4e38]
    for user in (False, True):
        assert M.write_tmt(files, ids, fi, si, inj, peaks, user, threads=3) == W.write_tmt(files, ids, fi, si, inj, peaks, user)


def test_fragment_file_oracle_equals_restatement():
    rng = np.random.default_rng(4)
    rows = np.zeros(30, api.FEATURE_DTYPE)
    counts = rng.integers(0, 5, 30)
    counts[3] = 0
    rows["fragment_count"] = counts
    rows["fragment_offset"] = np.concatenate([[0], np.cumsum(counts)[:-1]])
    fr = np.zeros(int(counts.sum()), api.FRAGMENT_DTYPE)
    fr["kind"] = rng.integers(0, 6, len(fr))
    fr["charge"] = rng.integers(1, 4, len(fr))
    fr["ordinal"] = rng.integers(1, 30, len(fr))
    for f in ("intensity", "mz_calculated", "mz_experimental"):
        fr[f] = rng.integers(0, 1 << 32, len(fr), dtype=np.uint64).astype(np.uint32).view(np.float32)
    pid = rng.integers(0, 1 << 40, 30).astype(np.uint64)
    got = M.write_fragments(pid, rows["fragment_offset"], rows["fragment_count"], fr, threads=4)
    assert got == W.write_fragments(pid, rows, fr)


# ------------------------------------------------------------------------------------------------ C ABI: arguments checked before the device
def call(file, ci, out=None, cap=0):
    size = C.c_uint64(12345)
    rc = api.load_library().sage_b200_write_tsv(C.c_int(0), C.c_int(file), C.byref(ci) if ci is not None else None, out, C.c_uint64(cap), C.byref(size))
    return rc, size.value


def test_write_tsv_rejects_bad_arguments():
    EINVAL = -1
    assert call(api.FILE_FRAGMENTS, None)[0] == EINVAL
    assert call(99, api.CWriteInputs())[0] == EINVAL
    rows = np.zeros(2, api.FEATURE_DTYPE)
    rows["fragment_offset"], rows["fragment_count"] = [0, 2], [2, 2]
    fr = np.zeros(3, api.FRAGMENT_DTYPE)
    pid = np.zeros(2, np.uint64)
    ci = api.CWriteInputs(rows=api._ptr(rows), psm_id=api._ptr(pid), n_rows=2, fragments=api._ptr(fr), n_fragments=3)
    assert call(api.FILE_FRAGMENTS, ci)[0] == EINVAL   # row 1's range ends past the array
    assert "outside" in api._last_error()
    fr2 = np.zeros(4, api.FRAGMENT_DTYPE)
    fr2["kind"][3] = 6
    ci.fragments, ci.n_fragments = api._ptr(fr2), 4
    assert call(api.FILE_FRAGMENTS, ci)[0] == EINVAL   # kind outside 0..5
    ci.psm_id = None
    assert call(api.FILE_FRAGMENTS, ci)[0] == EINVAL

    keep = []
    fo, fb, nf = api._strings(["a.mzML"], keep)
    so, sb, ns = api._strings(["s1", "s2"], keep)
    fi, si = np.array([0, 1], np.uint32), np.array([0, 1], np.uint32)
    inj, pk = np.zeros(2, np.float32), np.zeros((2, 6), np.float32)
    t = api.CWriteInputs(filename_offsets=fo, filename_bytes=fb, n_files=nf, spec_id_offsets=so, spec_id_bytes=sb, n_spec_ids=ns, n_quant=2,
                         quant_file_id=api._ptr(fi), quant_spec_id=api._ptr(si), ion_injection_time=api._ptr(inj), peaks=api._ptr(pk), n_channels=6)
    assert call(api.FILE_TMT, t)[0] == EINVAL          # file id 1 of 1 file
    fi[1] = 0
    si[1] = 2
    assert call(api.FILE_TMT, t)[0] == EINVAL          # spectrum index 2 of 2 ids
    t.filename_offsets = None
    assert call(api.FILE_TMT, t)[0] == EINVAL


def test_write_tsv_header_only_needs_no_device():
    pk = np.zeros((0, 10), np.float32)
    for user, head in ((False, "tmt_"), (True, "user_")):
        want = W.write_tmt([b"a"], [b"s"], [], [], [], pk, user)
        keep = []
        fo, fb, nf = api._strings(["a"], keep)
        so, sb, ns = api._strings(["s"], keep)
        t = api.CWriteInputs(filename_offsets=fo, filename_bytes=fb, n_files=nf, spec_id_offsets=so, spec_id_bytes=sb, n_spec_ids=ns, n_channels=10,
                             user_labels=int(user))
        rc, size = call(api.FILE_TMT, t)
        assert rc == 0 and size == len(want)
        assert call(api.FILE_TMT, t, C.create_string_buffer(4), 4) == (-5, len(want))   # ELIMIT, size reported
        buf = C.create_string_buffer(size)
        assert call(api.FILE_TMT, t, buf, size) == (0, size)
        assert buf.raw == want and head.encode() + b"10\n" in want
    assert api.write_fragments(np.zeros(0, api.FEATURE_DTYPE), np.zeros(0, api.FRAGMENT_DTYPE), []) == W.write_fragments([], [], [])


# ------------------------------------------------------------------------------------------------ results / pin / lfq inputs
def tiny_digest():
    pep = api.Peptides(seq_off=np.array([0, 3, 7], np.uint32), seq=np.frombuffer(b"PEKMAGR", np.uint8).copy(),
                       mods=np.array([0, 0, 0, 15.9949, 0, 0, 0], np.float32), nterm=np.array([np.nan, 42.010565], np.float32),
                       mono=np.array([300.0, 700.0], np.float32), decoy=np.array([0, 1], np.uint8), missed=np.zeros(2, np.uint8))
    return api.DigestResult(peptides=pep, cterm=np.array([np.nan, 0.0], np.float32), semi_enzymatic=np.array([0, 1], np.uint8),
                            protein_offsets=np.array([0, 1, 3], np.uint32), protein_ids=np.array([0, 0, 1], np.uint32), names=["A", 'B"x'], info={})


def test_pin_scan_nr_matches_python_re():
    import re
    ids = ["controllerType=0 controllerNumber=1 scan=17", "index=4", "scan=1 scan=22", "scan= scan=x", "scan=007 frame=3 scan=", "scan=5scan=6",
           "sscan=9", "", "scan=12\tq", 'a"scan=3"']
    d = tiny_digest()
    rows = np.zeros(len(ids), api.FEATURE_DTYPE)
    out = M.write_results(d, rows, np.arange(len(ids)), np.zeros(len(ids)), np.arange(len(ids)), ["f"], ids, pin=True)
    got = [ln.split(b"\t")[2] for ln in out.split(b"\n")[1:-1]]
    want = []
    for s in ids:
        m = re.findall(r"scan=([0-9]+)", s)
        want.append(W.field((m[-1] if m else s).encode()))
    assert got == want


def test_results_known_record():
    d = tiny_digest()
    rows = np.zeros(1, api.FEATURE_DTYPE)
    rows["peptide_idx"], rows["label"], rows["charge"], rows["rank"] = 1, -1, 2, 1
    rows["hyperscore"], rows["poisson"], rows["expmass"], rows["rt"] = 12.5, -3.0, 700.25, 1.5
    out = M.write_results(d, rows, [7], [0], [0], ["f"], ["scan=3"]).split(b"\n")[1].split(b"\t")
    assert out[:4] == [b"7", b"[+42.010567]-M[+15.9949]AGR-[+0]", b'"rev_A;rev_B""x"', b""]
    assert out[4:10] == [b"2", b"0", b"f", b"scan=3", b"1", b"-1"] and out[19] == b"12.5" and out[22:26] == [b"1.5", b"1.5", b"0.0", b"0.999"]
    assert out[15] == b"1" and out[-1] == b"0.0"


def test_write_tsv_rejects_bad_table_arguments():
    EINVAL = -1
    d = tiny_digest()
    keep = []
    rows = np.zeros(2, api.FEATURE_DTYPE)
    pid, fid, six = np.zeros(2, np.uint64), np.zeros(2, np.uint32), np.zeros(2, np.uint32)
    ci = api.CWriteInputs(rows=api._ptr(rows), psm_id=api._ptr(pid), n_rows=2, file_id=api._ptr(fid), spec_index=api._ptr(six))
    ci.filename_offsets, ci.filename_bytes, ci.n_files = api._strings(["f"], keep)
    ci.spec_id_offsets, ci.spec_id_bytes, ci.n_spec_ids = api._strings(["s"], keep)
    api._digest_table(ci, d, "rev_", True, keep)
    for file in (api.FILE_RESULTS, api.FILE_PIN):
        rows["peptide_idx"][1] = 2
        assert call(file, ci)[0] == EINVAL and "peptide_idx" in api._last_error()
        rows["peptide_idx"][1] = 1
        six[0] = 1
        assert call(file, ci)[0] == EINVAL
        six[0] = 0
        fid[1] = 1
        assert call(file, ci)[0] == EINVAL
        fid[1] = 0
    ids = np.array([0, 0, 2], np.uint32)   # protein id 2 of 2 names
    ci.protein_ids = api._ptr(ids)
    assert call(api.FILE_RESULTS, ci)[0] == EINVAL and "protein id" in api._last_error()
    ci.protein_ids = api._ptr(np.ascontiguousarray(d.protein_ids))
    g = dict(rgo=np.array([0, 1, 1], np.uint64), rg=np.array([1], np.uint32), go=np.array([0, 1], np.uint64), gm=np.array([0], np.uint32),
             gd=np.zeros(1, np.uint8), gp=np.array([1, 0], np.uint8))
    ci.group_pass, ci.row_group_offsets, ci.row_groups = api._ptr(g["gp"]), api._ptr(g["rgo"]), api._ptr(g["rg"])
    ci.group_offsets, ci.group_members, ci.group_decoy, ci.n_groups = api._ptr(g["go"]), api._ptr(g["gm"]), api._ptr(g["gd"]), 1
    assert call(api.FILE_RESULTS, ci)[0] == EINVAL and "row group" in api._last_error()   # group 1 of 1
    lq = np.zeros(1, api.LFQ_ROW_DTYPE)
    lq["peptide"] = 5
    q, ar = np.zeros(1, np.float32), np.zeros(1, np.float64)
    li = api.CWriteInputs(lfq_rows=api._ptr(lq), lfq_q=api._ptr(q), lfq_areas=api._ptr(ar), n_lfq=1)
    li.filename_offsets, li.filename_bytes, li.n_files = api._strings(["f"], keep)
    api._digest_table(li, d, "rev_", True, keep)
    assert call(api.FILE_LFQ, li)[0] == EINVAL and "LFQ row" in api._last_error()
