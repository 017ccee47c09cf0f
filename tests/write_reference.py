"""A small Python restatement of the text of Sage's result files (DESIGN.md §17), independent of std::to_chars and of the device code.

Digits come from Python's repr(float) (shortest round-trip of an f64) and numpy.format_float_scientific(np.float32(x), unique=True) (shortest
round-trip of an f32); the layouts restate ryu::Buffer::format (ryu 1.0.23), Rust's `{:+}` of an f32 and csv-core 0.1.13's
QuoteStyle::Necessary with delimiter '\\t'.
"""
from __future__ import annotations

import math
from decimal import Decimal

import numpy as np

# ryu's positional threshold (kk <= T) per type, as stated from the crate as pinned (Cargo.lock: ryu 1.0.23). A cross-check against the
# real crate corrects it here.
RYU_THRESHOLD = {64: 16, 32: 13}

# (kind, value, text): kind "f64" / "f32" = ryu layout, "plus" = `{:+}` of an f32. The known answers of DESIGN.md §17.
KNOWN_ANSWERS = [
    ("f32", 5339999700.0, "5339999700.0"),
    ("f64", 12.34, "12.34"),
    ("f32", 0.0010310042, "0.0010310042"),
    ("f64", 1e16, "1e16"),
    ("f64", 2.816025e14, "281602500000000.0"),
    ("f32", 2.816025e14, "2.816025e14"),
    ("f64", 5e-324, "5e-324"),
    ("f64", 1e-6, "1e-6"),
    ("f64", 1e-5, "0.00001"),
    ("f64", 1e15, "1000000000000000.0"),
    ("f32", 1e12, "1000000000000.0"),
    ("f32", 1e13, "1e13"),
    ("f64", float("nan"), "NaN"),
    ("f64", float("inf"), "inf"),
    ("f64", float("-inf"), "-inf"),
    ("f64", 0.0, "0.0"),
    ("f64", -0.0, "-0.0"),
    ("f32", -0.0, "-0.0"),
    ("plus", 57.021465, "+57.021465"),
    ("plus", 42.0, "+42"),
    ("plus", -0.0, "-0"),
    ("plus", float("inf"), "+inf"),
    ("plus", float("nan"), "NaN"),
    ("plus", 1e20, "+100000000000000000000"),
]


def shortest(x: float, bits: int):
    """Shortest round-trip digits of finite nonzero |x| as (digits, k): |x| = digits * 10^k."""
    text = repr(abs(float(x))) if bits == 64 else np.format_float_scientific(np.float32(abs(x)), unique=True)
    t = Decimal(text).as_tuple()
    d, k = "".join(map(str, t.digits)), t.exponent
    stripped = d.rstrip("0")
    return stripped, k + len(d) - len(stripped)


def ryu(x: float, bits: int) -> str:
    """ryu::Buffer::format of an f64 (bits 64) or of the f32 nearest x (bits 32)."""
    if bits == 32:
        x = float(np.float32(x))
    if math.isnan(x):
        return "NaN"
    if math.isinf(x):
        return "inf" if x > 0 else "-inf"
    sign = "-" if math.copysign(1.0, x) < 0 else ""
    if x == 0:
        return sign + "0.0"
    d, k = shortest(x, bits)
    n, kk, T = len(d), len(d) + k, RYU_THRESHOLD[bits]
    if 0 <= k and kk <= T:
        return sign + d + "0" * k + ".0"
    if 0 < kk <= T:
        return sign + d[:kk] + "." + d[kk:]
    if -5 < kk <= 0:
        return sign + "0." + "0" * (-kk) + d
    return sign + d[0] + ("." + d[1:] if n > 1 else "") + "e" + str(kk - 1)


def plus(x: float) -> str:
    """`{:+}` of an f32 (Rust Display): shortest digits, positional, signed; NaN prints NaN."""
    x = float(np.float32(x))
    if math.isnan(x):
        return "NaN"
    sign = "-" if math.copysign(1.0, x) < 0 else "+"
    if math.isinf(x):
        return sign + "inf"
    if x == 0:
        return sign + "0"
    d, k = shortest(x, 32)
    kk = len(d) + k
    if k >= 0:
        return sign + d + "0" * k
    if kk > 0:
        return sign + d[:kk] + "." + d[kk:]
    return sign + "0." + "0" * (-kk) + d


def field(b: bytes) -> bytes:
    """One csv-core field: quoted when it holds '\\t', '"', '\\r' or '\\n', with '"' doubled inside."""
    if any(c in b for c in b'\t"\r\n'):
        return b'"' + b.replace(b'"', b'""') + b'"'
    return b


def record(fields) -> bytes:
    return b"\t".join(field(f if isinstance(f, bytes) else f.encode()) for f in fields) + b"\n"


def write_fragments(psm_id, rows, fragments) -> bytes:
    out = [record(["psm_id", "fragment_type", "fragment_ordinals", "fragment_charge", "fragment_mz_calculated", "fragment_mz_experimental",
                   "fragment_intensity"])]
    for pid, r in zip(psm_id, rows):
        for f in fragments[int(r["fragment_offset"]):int(r["fragment_offset"]) + int(r["fragment_count"])]:
            out.append(record([str(int(pid)), "abcxyz"[int(f["kind"])], str(int(f["ordinal"])), str(int(f["charge"])), ryu(f["mz_calculated"], 32),
                               ryu(f["mz_experimental"], 32), ryu(f["intensity"], 32)]))
    return b"".join(out)


def write_tmt(filenames, spec_ids, file_id, spec, injection, peaks, user_labels=False) -> bytes:
    peaks = np.asarray(peaks, np.float32)
    head = ["filename", "scannr", "ion_injection_time"] + [("user_%d" if user_labels else "tmt_%d") % (c + 1) for c in range(peaks.shape[1])]
    out = [record(head)]
    for i in range(len(file_id)):
        out.append(record([filenames[int(file_id[i])], spec_ids[int(spec[i])], ryu(injection[i], 32)] + [ryu(p, 32) for p in peaks[i]]))
    return b"".join(out)
