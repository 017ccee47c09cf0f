"""MgfReader::parse without a GPU: the plain-Python restatement (tests/mgf_reference.py) against the C++ oracle (oracle_mgf/) bit for bit on
every case of tests/mgf_cases.py, the errors both raise, and Rust's f32 grammar and rounding at its edges: the accept / reject table,
exact midpoints between adjacent f32s and their neighbours, the subnormal, FLT_MIN and FLT_MAX edges, long digit strings and huge exponents."""
import struct
import sys
from fractions import Fraction

import numpy as np
import pytest

import mgf_cases as MC
import mgf_reference as R
from oracle_mgf import mgf_oracle as O

FIELDS = ["peak_off", "mz", "intensity", "scan_start_time", "tic", "prec_off", "prec_mz", "prec_intensity", "prec_intensity_some", "prec_charge",
          "prec_charge_some", "iso_kind", "iso_lo", "iso_hi", "id_off", "id_bytes"]


def assert_same(a: dict, b: dict, what: str):
    assert a["info"] == b["info"], what
    for k in FIELDS:
        x, y = np.ascontiguousarray(a[k]), np.ascontiguousarray(b[k])
        assert x.dtype.itemsize == y.dtype.itemsize and x.view(np.uint8).tobytes() == y.view(np.uint8).tobytes(), f"{what}: {k}"


@pytest.mark.parametrize("name", [n for n in MC.CASES if n not in MC.BIG])
def test_restatement_equals_oracle(name):
    t = MC.CASES[name]()
    assert_same(R.parse(t), O.parse(t), name)


def test_known_answers():
    d = O.parse(MC.known_answer())
    assert d["info"]["n_spectra"] == 2
    assert d["prec_charge"].tolist() == [2, 3, 2, 3] and d["prec_charge_some"].tolist() == [1, 1, 1, 1]
    assert d["iso_kind"].tolist() == [2] * 4 and d["iso_lo"].tolist() == [-10.0] * 4 and d["iso_hi"].tolist() == [10.0] * 4
    assert d["prec_intensity"][0] == np.float32(56700.5185546875) and d["intensity"][0] == 1.0
    assert d["scan_start_time"][0] == np.float32(0.8963232289) / np.float32(60.0)
    d = O.parse(MC.matrixscience())
    # the header's CHARGE reaches Spectrum 2 only (record 0 starts from None); "dodgy" is Da 3
    assert d["prec_off"].tolist() == [0, 1, 3, 4] and d["prec_charge_some"].tolist() == [0, 1, 1, 1] and d["prec_charge"].tolist() == [0, 2, 3, 3]
    assert d["iso_kind"].tolist() == [0, 0, 0, 1] and d["iso_hi"][3] == 3.0


def test_rules_show():
    d = R.parse(MC.first_record_defaults())
    assert d["iso_kind"].tolist() == [0, 1, 1] and d["prec_charge_some"].tolist() == [0, 1, 1] and d["prec_charge"].tolist() == [0, 2, 4]
    assert d["iso_lo"].tolist() == [0.0, -0.5, -3.0] and d["iso_hi"].tolist() == [0.0, 0.5, 3.0]
    d = R.parse(MC.title_between_records())
    assert d["info"]["n_records"] == 2 and d["info"]["n_spectra"] == 1 and bytes(d["id_bytes"]) == b"between"
    d = R.parse(MC.charges())
    ids = bytes(d["id_bytes"]).decode()
    assert ids == "zerotwelvearabicmixed" and d["prec_charge"].tolist() == [0, 1, 2, 2, 2, 3, 1, 0]
    d = R.parse(MC.pepmass_x_charges())
    # the last CHARGE line wins; every PEPMASS x every charge, PEPMASS outermost
    assert d["prec_mz"].tolist() == [500.0] * 2 + [600.0] * 2 + [700.0] * 2 and d["prec_charge"].tolist() == [2, 3] * 3
    assert d["prec_intensity_some"].tolist() == [1, 1, 0, 0, 1, 1] and d["prec_intensity"][-1] == 700.0
    d = R.parse(MC.tolu_kinds())
    assert d["iso_kind"].tolist() == [1, 2, 0, 0, 1, 0, 0, 0]   # "Da " loses its space to the line's trim; " Da" keeps it and d["iso_lo"][0] == -2.5 and d["iso_hi"][0] == 2.5
    d = R.parse(MC.failed_parses_keep_previous())
    assert d["iso_hi"][0] == 5.0 and d["scan_start_time"][0] == 2.0
    assert R.parse(MC.nested_begin())["info"]["n_spectra"] == 1 and R.parse(MC.trailing_without_end())["info"]["n_spectra"] == 1


@pytest.mark.parametrize("name", list(MC.ERRORS))
def test_errors(name):
    t = MC.ERRORS[name]()
    with pytest.raises(R.ReferenceError) as a:
        R.parse(t)
    with pytest.raises(O.MgfOracleError) as b:
        O.parse(t)
    assert ("UTF-8" in str(a.value)) == ("UTF-8" in str(b.value)) == name.startswith("utf8")
    if name.startswith("utf8"):
        assert str(a.value).split("offset ")[1].split()[0] == str(b.value).split("offset ")[1]


ACCEPT = ["0", "1", "1.", ".5", "01.50", "+1", "-1", "1e5", "1E5", "1e+5", "1e-5", "1.5E-05", "inf", "INF", "Infinity", "-infinity", "+inf", "nan",
          "NaN", "-nan", "+NAN", "0e0", "00000", "1e0000000000000000000000000000", "9" * 50, "0." + "0" * 60 + "1"]
REJECT = ["", ".", "+", "-", "e5", "1e", "1e+", ".e1", "0x1", "1_0", " 1", "1 ", "1.0f", "1,5", "--1", "+-1", "in", "infinit", "nana", "1..2",
          "1.2.3", "1e5.5", "١", "1\x0b", "infinityx", "1e-"]


def test_grammar_table():
    bits, ok = O.parse_f32(ACCEPT + REJECT)
    assert ok.tolist() == [True] * len(ACCEPT) + [False] * len(REJECT)
    for t, b, k in zip(ACCEPT + REJECT, bits, ok):
        r = R.parse_f32(t)
        assert (r is not None) == k, t
        if k:
            assert r == int(b), t


def _midpoints(rng, n):
    """Exact decimal midpoints between adjacent f32s (finite, both signs), and the decimals one unit in their last place either side."""
    out = []
    for u in rng.integers(0, 0x7F7FFFFF, n, dtype=np.uint64):
        a, b = (np.array([u, u + 1], np.uint32).view(np.float32)).astype(np.float64)
        m = (Fraction(float(a)) + Fraction(float(b))) / 2
        k = 0
        while (m * 10 ** k).denominator != 1:
            k += 1
        digits = str(int(m * 10 ** k))
        out += [f"{digits}e-{k}", f"{int(digits) + 1}e-{k}", f"{int(digits) - 1}e-{k}"]
    return out


def test_rounding_edges():
    rng = np.random.default_rng(7)
    toks = _midpoints(rng, 300)
    # subnormal, FLT_MIN and FLT_MAX edges, exact and as halves
    for u in [0, 1, 2, 3, 0x7FFFFF, 0x800000, 0x800001, 0x7F7FFFFE, 0x7F7FFFFF]:
        x = Fraction(struct.unpack("<f", struct.pack("<I", u))[0])
        ulp = Fraction(2) ** -149 if u < 0x1000000 else Fraction(2) ** ((u >> 23) - 150)
        for v in (x, x + ulp / 2, x - ulp / 2 if x else x, x + ulp / 2 + Fraction(1, 10 ** 80)):
            k = 0
            while (v * 10 ** k).denominator != 1 and k < 200:
                k += 1
            toks.append(f"{int(v * 10 ** k)}e-{k}")
    toks += ["3.4028235677973366e38", "3.4028235677973367e38", "3.40282356779733661637539395458142568448e38", "1e-46", "7.0064923216240854e-46",
             "7.0064923216240862e-46", "1" + "0" * 800 + "e-800", "0." + "9" * 120, "1e" + "9" * 19, "1e-" + "9" * 19]
    toks += ["-" + t for t in toks[:50]]
    bits, ok = O.parse_f32(toks)
    assert ok.all()
    for t, b in zip(toks, bits):
        assert R.parse_f32(t) == int(b), t
