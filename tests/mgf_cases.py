"""MGF inputs, one generator per rule of MgfReader::parse (mgf.rs:324-370) that shows in its output. Each returns the file's bytes.
CASES maps a name to its generator; BIG lists the ones large enough to be run on the device only. ERRORS are files the reference rejects."""
from __future__ import annotations

import numpy as np

SPEC0 = """BEGIN IONS
TITLE=spectrum 0
RTINSECONDS=0.8963232289
PEPMASS=367.069682741984 56700.5185546875
CHARGE=2+ and 3+
TOL=10
TOLU=ppm
148.2041016 
169.5001831 4608.2421875
226.0483246 5335.4907226563
228.3407898 30918.244140625
322.5945435 5311.5737304688
1144.66272 6260.8315429688
END IONS
"""


def _rec(title="t", pepmass="PEPMASS=500.5", peaks=("100 1",), extra=()):
    lines = ["BEGIN IONS", f"TITLE={title}" if title is not None else "", pepmass, *extra, *peaks, "END IONS"]
    return "\n".join(x for x in lines if x != "") + "\n"


def known_answer():   # mgf.rs parse_spectrum / parse_two_spectra
    return ("# a comment at the beginning of the file\n" + "\n".join("        " + ln for ln in SPEC0.splitlines()) + "\n\n" + SPEC0).encode()


def matrixscience():   # mgf.rs parse_mgf_matrixscience_example_1 and _2 (header CHARGE, ITOL ignored, sequence queries in the header)
    return ("COM=10 pmol digest\nITOL=1\nITOLU=Da\nCHARGE=2+ and 3+\n1024.6\n2321 seq(n-ACTL) comp(2[C])\n"
            + _rec("Spectrum 1", "PEPMASS=983.6", ("846.60 73", "846.80 44", "1640.10 291"))
            + "\n" + _rec("Spectrum 2", "PEPMASS=1084.9", ("345.10 237", "370.20 128"), ("SCANS=3", "RTINSECONDS=25"))
            + _rec("dodgy", "PEPMASS=896.05 25674.3", ("240.1 3", "242.1 12"), ("CHARGE=3+", "TOL=3", "TOLU=Da", "SEQ=n-AC[DHK]"))).encode()


def first_record_defaults():   # record 0 does not see the header's TOL / TOLU / CHARGE; records 1.. do
    return ("TOL=0.5\nTOLU=Da\nCHARGE=2+\nBEGIN IONS\nTITLE=a\nPEPMASS=400\n100 1\nEND IONS\n" + _rec("b") + _rec("c", extra=("CHARGE=4", "TOL=-3"))).encode()


def title_between_records():   # state is not reset at BEGIN IONS: a TITLE between records belongs to the next one
    return ("BEGIN IONS\nPEPMASS=1\n1 1\nEND IONS\nTITLE=between\nBEGIN IONS\nPEPMASS=2\n2 2\nEND IONS\n").encode()


def nested_begin():
    return ("BEGIN IONS\nTITLE=x\nBEGIN IONS\nPEPMASS=3\nBEGIN IONS\n3 3\nEND IONS\n").encode()


def trailing_without_end():
    return (_rec("kept") + "BEGIN IONS\nTITLE=lost\nPEPMASS=5\n5 5\n1x 2\nPEPMASS=bad\n").encode()


def whitespace():   # CRLF, NBSP, U+3000, vertical tab at line ends and inside lines, a BOM
    return ("﻿TOL=1\r\nBEGIN IONS\r\n TITLE=crlf　\r\nPEPMASS=10 20\r\n 100\x0b 2 \r\n\x0b200\t3\x0c\r\n300 5\r\n"
            " 400 \x0b5\nTOLU=Da \nTOL=2 \nEND IONS\u0085\n"
            "　BEGIN IONS\nTITLE= nb sp \nPEPMASS= 11\n1 1\n2 2 \nEND IONS \n"
            "BEGIN IONS\nTITLE=﻿bom\nPEPMASS=12\n﻿3 3\n4 4\nEND IONS\n"
            "﻿BEGIN IONS\nTITLE=py-space\x1c\nPEPMASS=13\n5 5\x1f\n6 6\nEND IONS\n").encode()


def bom_before_begin():   # a BOM is not whitespace: the first line is not a BEGIN line
    return ("﻿BEGIN IONS\nBEGIN IONS\nTITLE=a\nPEPMASS=1\n1 1\nEND IONS\n").encode()


def charges():
    return (_rec("zero", extra=("CHARGE=0",)) + _rec("twelve", extra=("CHARGE=12",)) + _rec("none", extra=("CHARGE=+",))
            + _rec("arabic", extra=("CHARGE=٣+ and 2",)) + _rec("only-arabic", extra=("CHARGE=٣٤",))
            + _rec("mixed", extra=("CHARGE=2+, 3+ or 10-",))).encode()


def pepmass_x_charges():
    return (_rec("m", "PEPMASS=500 100", extra=("PEPMASS=600", "PEPMASS=700 7e2 junk", "CHARGE=1 2 3", "CHARGE=2+ and 3+"))).encode()


def pepmass_edges():
    return (_rec("empty", "PEPMASS=") + _rec("blank", "PEPMASS=   \t") + _rec("bad-mz", "PEPMASS=abc 5") + _rec("bad-int", "PEPMASS=400 x5")
            + _rec("bad-then-good", "PEPMASS=x", extra=("PEPMASS=401.5",)) + _rec("nbsp", "PEPMASS=402 5")).encode()


def peak_edges():
    return (_rec("one-token", peaks=("100", "200 2")) + _rec("bad-int", peaks=("100 1", "200 x")) + _rec("three", peaks=("100 1 junk", "200 2 3 4"))
            + _rec("leading", peaks=("-1.0 5", ".5 5", "+1 5", "100 1", "1e2 3", "1x 2", "1,5 2", "٥ 2", "² 3"))
            + _rec("bad-int-first", peaks=("100 y", "200 2", "300"))).encode()


def failed_parses_keep_previous():
    return (_rec("t", extra=("TOL=5", "TOL=x", "TOLU=Da", "RTINSECONDS=120", "RTINSECONDS=abc", "RTINSECONDS= 60"))
            + _rec("u", extra=("TOL=nan", "TOLU=ppm", "RTINSECONDS=-nan")) + _rec("v", extra=("TOL=-inf", "TOLU=Da", "RTINSECONDS=1e40"))).encode()


def tolu_kinds():
    return ("".join(_rec(f"u{i}", extra=("TOL=-2.5", f"TOLU={u}")) for i, u in enumerate(["Da", "ppm", "da", " Da", "Da ", "PPM", "mmu", ""]))).encode()


def titles():
    return (_rec("", peaks=("1 1",)) + _rec(None) + _rec("x", extra=("TITLE=",)) + _rec("last", extra=("TITLE=wins",))
            + _rec("scan=1 file=a.raw é中\U0001f600", extra=())).encode()


def header_only():
    return b"COM=header only\nTOL=1\n"


def no_begin():
    return b"TITLE=x\nPEPMASS=1\n1 1\nEND IONS\n"


def invalid_utf8(where: str):
    good = _rec("a").encode()
    bad = b"\xff"
    return {"start": bad + good, "middle": good[:20] + b"\xe2\x82" + good[20:], "end": good + b"\xf0\x9f\x98"}[where]


def numbers():   # the f32 grammar and rounding through every number field
    toks = ["1", "1.", ".5", "1e3", "1E-3", "+2", "1.5e+2", "3.4028235e38", "3.4028236e38", "1e39", "1e-45", "7e-46", "0.0", "-0",
            "inf", "-Infinity", "NaN", "-nan", "0x10", "1_0", "e5", "1e", ".", "", "16777217", "0.1000000000000000055511151231257827",
            "1" + "0" * 60, "0." + "0" * 40 + "1", "1.00000005960464477539062500000000000000000000000000001", "1.000000059604644775390625"]
    peaks = [f"{t} {u}" for t, u in zip(toks, reversed(toks)) if t and t[0].isdigit()]
    recs = "".join(_rec(f"n{i}", f"PEPMASS={t} {t}", extra=(f"TOL={t}", "TOLU=Da", f"RTINSECONDS={t}")) for i, t in enumerate(toks))
    return (recs + _rec("peaks", peaks=peaks)).encode()


def tic_nan_rules():
    return (_rec("a", peaks=("1 1", "2 nan", "3 -nan", "4 inf")) + _rec("b", peaks=("1 inf", "2 -inf", "3 5")) + _rec("c", peaks=("1 -0", "2 -0"))
            + _rec("d", peaks=("1 -nan", "2 nan")) + _rec("e", peaks=("1 3.4e38", "2 3.4e38", "3 -3.4e38"))).encode()


def empty_lines_and_comments():
    return ("\n\n#c\nBEGIN IONS\n\n\nTITLE=e\n\n#x\nPEPMASS=5\n\n1 1\n   \n\nEND IONS\n\n\nBEGIN IONS\nEND IONS\n").encode()


def no_trailing_newline():
    return _rec("last").rstrip("\n").encode()


def big_spectrum(n: int = 20000, seed: int = 1):
    rng = np.random.default_rng(seed)
    mz = np.sort(rng.uniform(100, 2000, n).astype(np.float32))
    it = rng.lognormal(5, 2, n).astype(np.float32)
    return ("BEGIN IONS\nTITLE=big\nPEPMASS=1000.5 10\nCHARGE=2+\n" + "".join(f"{repr(float(a))} {repr(float(b))}\n" for a, b in zip(mz, it))
            + "END IONS\n").encode()


def many_spectra(n: int = 100000):
    return "".join(f"BEGIN IONS\nTITLE=s{i}\nPEPMASS={300 + i * 0.001:.3f}\nCHARGE={2 + i % 3}+\n{100 + i % 997}.25 {i}\nEND IONS\n" for i in range(n)).encode()


def long_line():
    return ("BEGIN IONS\nTITLE=" + "x" * (1 << 20) + "\nPEPMASS=1\nCHARGE=" + "2 " * 600000 + "\n1 " + "9" * (1 << 20) + "\n2 "
            + "0" * (1 << 20) + "1e-1048576\nEND IONS\n").encode()


CASES = {
    "known_answer": known_answer, "matrixscience": matrixscience, "first_record_defaults": first_record_defaults,
    "title_between_records": title_between_records, "nested_begin": nested_begin, "trailing_without_end": trailing_without_end,
    "whitespace": whitespace, "bom_before_begin": bom_before_begin, "charges": charges, "pepmass_x_charges": pepmass_x_charges,
    "pepmass_edges": pepmass_edges, "peak_edges": peak_edges, "failed_parses_keep_previous": failed_parses_keep_previous,
    "tolu_kinds": tolu_kinds, "titles": titles, "numbers": numbers, "tic_nan_rules": tic_nan_rules,
    "empty_lines_and_comments": empty_lines_and_comments, "no_trailing_newline": no_trailing_newline,
    "big_spectrum": big_spectrum, "many_spectra": many_spectra, "long_line": long_line,
}
BIG = {"many_spectra", "long_line"}
ERRORS = {"empty": lambda: b"", "header_only": header_only, "no_begin": no_begin, "utf8_start": lambda: invalid_utf8("start"),
          "utf8_middle": lambda: invalid_utf8("middle"), "utf8_end": lambda: invalid_utf8("end")}
