"""A plain-Python restatement of MgfReader::parse (sage-cloudpath mgf.rs:324-370, util.rs:107-118), written from the Rust and not from the
C++ oracle. It imports neither the oracle nor the library. Numbers follow Rust's `str::parse::<f32>` with exact rational arithmetic
(fractions.Fraction and integers; never float(), which would round twice). The f32 sum and the division by 60 follow x86-64 SSE, NaNs
included (DESIGN.md §16). parse() returns the layout of sage_b200_mgf_export, or raises ReferenceError where the reference fails or panics.
"""
from __future__ import annotations

import re
import struct
from fractions import Fraction

import numpy as np

# char::is_whitespace: Unicode White_Space (what str::trim strips). Not str.isspace, which also strips U+001C..U+001F.
WHITE_SPACE = "".join(chr(c) for c in [*range(0x09, 0x0E), 0x20, 0x85, 0xA0, 0x1680, *range(0x2000, 0x200B), 0x2028, 0x2029, 0x202F, 0x205F, 0x3000])
ASCII_WS = " \t\n\x0c\r"   # u8::is_ascii_whitespace (no vertical tab)
_DECIMAL = re.compile(r"([0-9]*)(?:\.([0-9]*))?(?:[eE]([+-]?[0-9]+))?\Z")
QNAN, NEG_QNAN, X86_DEFAULT_NAN = 0x7FC00000, 0xFFC00000, 0xFFC00000


class ReferenceError(ValueError):
    pass


def round_f32(x: Fraction) -> int:
    """The f32 bits of the nonnegative rational x, rounded half to even (inf past the largest finite)."""
    if x == 0:
        return 0
    e = x.numerator.bit_length() - x.denominator.bit_length()
    if Fraction(2) ** e > x:
        e -= 1
    e = max(e, -126)                       # 2^e <= x < 2^(e+1), or the subnormal scale
    m = x / Fraction(2) ** (e - 23)        # in [2^23, 2^24) for normals
    q, r = divmod(m.numerator, m.denominator)
    if 2 * r > m.denominator or (2 * r == m.denominator and q & 1):
        q += 1
    bits = ((e + 126) << 23) + q
    return min(bits, 0x7F800000)


def parse_f32(s: str) -> int | None:
    """Rust's f32::from_str: the f32 bits, or None for an Err."""
    if not s or not s.isascii():
        return None
    neg = s[0] == "-"
    body = s[1:] if s[0] in "+-" else s
    sign = 0x80000000 if neg else 0
    if body.lower() in ("inf", "infinity"):
        return sign | 0x7F800000
    if body.lower() == "nan":
        return NEG_QNAN if neg else QNAN
    m = _DECIMAL.match(body)
    if not m or not (m.group(1) or m.group(2)):
        return None
    intd, frac, exp = m.group(1), m.group(2) or "", int(m.group(3) or 0)
    digits = (intd + frac).lstrip("0")
    if not digits:
        return sign
    # the place of the first significant digit: past 10^40 the value is inf, below 10^-50 it is 0, whatever the digits
    lead = len(intd + frac) - len(digits)
    top = len(intd) - 1 - lead + exp
    if top > 40:
        return sign | 0x7F800000
    if top < -50:
        return sign
    x = Fraction(int(digits)) * Fraction(10) ** (top - len(digits) + 1)
    return sign | round_f32(x)


def f32(bits: int) -> np.float32:
    return np.frombuffer(struct.pack("<I", bits), np.float32)[0]


def bits_of(x) -> int:
    return int(np.float32(x).view(np.uint32))


def _isnan(b: int) -> bool:
    return (b & 0x7F800000) == 0x7F800000 and (b & 0x7FFFFF) != 0


def add_x86(t: int, x: int) -> int:
    """addss t, x on f32 bits: a NaN result is the accumulator's NaN, else x's NaN quieted, else x86's default NaN."""
    with np.errstate(all="ignore"):
        r = bits_of(f32(t) + f32(x))
    if not _isnan(r):
        return r
    if _isnan(t):
        return t | 0x00400000
    if _isnan(x):
        return x | 0x00400000
    return X86_DEFAULT_NAN


def div60_x86(b: int) -> int:
    if _isnan(b):
        return b | 0x00400000
    with np.errstate(all="ignore"):
        return bits_of(f32(b) / np.float32(60.0))


def _charges(s: str) -> list:
    # Regex (\d)\+? is Unicode; char::to_digit(10) keeps the ASCII digits only
    return [ord(c) - 48 for c in s if "0" <= c <= "9"]


def parse(text: bytes) -> dict:
    try:
        s = bytes(text).decode("utf-8")
    except UnicodeDecodeError as e:
        raise ReferenceError(f"invalid UTF-8 at byte offset {e.start}") from None
    lines = s.split("\n")
    if lines and lines[-1] == "":   # str::lines: no line after a final '\n' (and none at all for "")
        lines.pop()
    it = iter(lines)
    d_tol = d_tolu = d_charge = None
    while True:   # DefaultParser: parse_begin, parse_tol, parse_tol_unit, parse_charge
        try:
            line = next(it).strip(WHITE_SPACE)
        except StopIteration:
            raise ReferenceError("no BEGIN IONS line (lines.next().unwrap() panics)") from None
        if line.startswith("BEGIN IONS"):
            break
        if line.startswith("TOL="):
            v = parse_f32(line[4:])
            if v is not None:
                d_tol = v
        elif line.startswith("TOLU="):
            d_tolu = line[5:]
        elif line.startswith("CHARGE="):
            d_charge = _charges(line[7:])
    spectra, n_records, malformed = [], 0, 0
    # QueryData::default_with_params: precursor_tol, precursor_tol_unit, precursor_charge_array are None for the first record
    q = dict(id="", precursors=[], tol=None, tolu=None, charge=None, rt=None, mz=[], intensity=[])
    for raw in it:
        line = raw.strip(WHITE_SPACE)
        if line[:1].isdigit() and line[0].isascii():   # parse_mz: only an ASCII digit can lead to a valid f32
            tok = [t for t in re.split("[" + re.escape(ASCII_WS) + "]+", line) if t]
            v = parse_f32(tok[0])
            if v is None:
                malformed += 1
                continue
            q["mz"].append(v)
            if len(tok) >= 2:
                w = parse_f32(tok[1])
                if w is not None:
                    q["intensity"].append(w)
            else:
                q["intensity"].append(bits_of(1.0))
        elif line.startswith("END IONS"):
            n_records += 1
            iso = (0, 0, 0)
            if q["tol"] is not None and q["tolu"] in ("Da", "ppm"):
                a = q["tol"] & 0x7FFFFFFF
                iso = (1 if q["tolu"] == "Da" else 2, a | 0x80000000, a)
            precs = []
            for p in q["precursors"]:
                if q["charge"] is not None:
                    precs += [dict(p, charge=(1, c), iso=iso) for c in q["charge"]]
                else:
                    precs.append(dict(p, charge=(0, 0), iso=iso))
            tic = 0
            for x in q["intensity"]:
                tic = add_x86(tic, x)
            sp = dict(id=q["id"], precursors=precs, rt=q["rt"] if q["rt"] is not None else 0, tic=tic, mz=q["mz"], intensity=q["intensity"])
            if sp["id"] and precs and sp["mz"] and len(sp["mz"]) == len(sp["intensity"]):
                spectra.append(sp)
            q = dict(id="", precursors=[], tol=d_tol, tolu=d_tolu, charge=d_charge, rt=None, mz=[], intensity=[])   # init()
        elif line.startswith("PEPMASS="):
            tok = [t for t in re.split("[" + re.escape(ASCII_WS) + "]+", line[8:]) if t]
            p = dict(mz=0, intensity=(0, 0))
            if tok:
                v = parse_f32(tok[0])
                if v is None:
                    malformed += 1
                    continue
                p["mz"] = v
            if len(tok) >= 2:
                w = parse_f32(tok[1])
                if w is not None:
                    p["intensity"] = (1, w)
            q["precursors"].append(p)
        elif line.startswith("TITLE="):
            q["id"] = line[6:]
        elif line.startswith("CHARGE="):
            q["charge"] = _charges(line[7:])
        elif line.startswith("TOL="):
            v = parse_f32(line[4:])
            if v is not None:
                q["tol"] = v
        elif line.startswith("TOLU="):
            q["tolu"] = line[5:]
        elif line.startswith("RTINSECONDS="):
            v = parse_f32(line[12:])
            if v is not None:
                q["rt"] = div60_x86(v)
    return _layout(spectra, len(lines), n_records, malformed)


def _layout(spectra, n_lines, n_records, malformed) -> dict:
    u32 = lambda xs: np.array(xs, np.uint32).view(np.float32)  # noqa: E731
    ids = [sp["id"].encode() for sp in spectra]
    precs = [p for sp in spectra for p in sp["precursors"]]
    cum = lambda xs: np.concatenate([[0], np.cumsum(xs)]).astype(np.uint64)  # noqa: E731
    d = dict(peak_off=cum([len(sp["mz"]) for sp in spectra]), mz=u32([x for sp in spectra for x in sp["mz"]]),
             intensity=u32([x for sp in spectra for x in sp["intensity"]]), scan_start_time=u32([sp["rt"] for sp in spectra]),
             tic=u32([sp["tic"] for sp in spectra]), prec_off=cum([len(sp["precursors"]) for sp in spectra]),
             prec_mz=u32([p["mz"] for p in precs]), prec_intensity=u32([p["intensity"][1] for p in precs]),
             prec_intensity_some=np.array([p["intensity"][0] for p in precs], np.uint8), prec_charge=np.array([p["charge"][1] for p in precs], np.uint8),
             prec_charge_some=np.array([p["charge"][0] for p in precs], np.uint8), iso_kind=np.array([p["iso"][0] for p in precs], np.uint8),
             iso_lo=u32([p["iso"][1] for p in precs]), iso_hi=u32([p["iso"][2] for p in precs]), id_off=cum([len(b) for b in ids]),
             id_bytes=np.frombuffer(b"".join(ids), np.uint8).copy())
    d["info"] = dict(n_lines=n_lines, n_records=n_records, n_spectra=len(spectra), n_peaks=len(d["mz"]), n_precursors=len(precs),
                     id_bytes=len(d["id_bytes"]), malformed_lines=malformed, dropped_records=n_records - len(spectra))
    return d
