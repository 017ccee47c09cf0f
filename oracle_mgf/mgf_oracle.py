"""ctypes binding of the CPU oracle of MgfReader::parse (oracle_mgf/mgf_oracle.cpp).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__ and tools/bench_mgf.py. Never imported by the sage_b200 package.
parse() returns the arrays of sage_b200_mgf_export (the layout of sage_b200.read_mgf), or raises MgfOracleError where the reference
fails (invalid UTF-8) or panics (no BEGIN IONS line).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "mgf_oracle.cpp")
_SO = os.path.join(_HERE, "_build", "libmgf_oracle.so")
# no FMA contraction, no fast-math: every f32 operation stays one separately rounded SSE instruction, as rustc emits it
CXXFLAGS = ["-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall"]

_lib = None


class MgfOracleError(ValueError):
    pass


def build(force: bool = False) -> str:
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        env = dict(os.environ)
        env.pop("CXX", None)
        subprocess.check_call(["/usr/bin/g++"] + CXXFLAGS + ["-o", _SO, _SRC], env=env)
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        _lib.mo_create.restype = C.c_void_p
        _lib.mo_create.argtypes = [C.c_char_p, C.c_uint64]
        _lib.mo_destroy.argtypes = [C.c_void_p]
        _lib.mo_info.argtypes = [C.c_void_p, C.c_void_p, C.c_char_p, C.c_uint64]
        _lib.mo_export.argtypes = [C.c_void_p] + [C.c_void_p] * 16
        _lib.mo_parse_f32.argtypes = [C.c_char_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def parse(text: bytes) -> dict:
    """MgfReader::parse of the file's bytes -> dict: info (n_lines, n_records, n_spectra, n_peaks, n_precursors, id_bytes, malformed_lines,
    dropped_records) and the arrays of sage_b200_mgf_export."""
    L = lib()
    h = L.mo_create(bytes(text), len(text))
    try:
        v = np.zeros(7, np.uint64)
        err = C.create_string_buffer(512)
        rc = L.mo_info(h, _p(v), err, 512)
        if rc != 0:
            raise MgfOracleError(err.value.decode())
        n_lines, n_rec, n, npk, npr, nid, bad = (int(x) for x in v)
        d = dict(peak_off=np.zeros(n + 1, np.uint64), mz=np.zeros(npk, np.float32), intensity=np.zeros(npk, np.float32),
                 scan_start_time=np.zeros(n, np.float32), tic=np.zeros(n, np.float32), prec_off=np.zeros(n + 1, np.uint64),
                 prec_mz=np.zeros(npr, np.float32), prec_intensity=np.zeros(npr, np.float32), prec_intensity_some=np.zeros(npr, np.uint8),
                 prec_charge=np.zeros(npr, np.uint8), prec_charge_some=np.zeros(npr, np.uint8), iso_kind=np.zeros(npr, np.uint8),
                 iso_lo=np.zeros(npr, np.float32), iso_hi=np.zeros(npr, np.float32), id_off=np.zeros(n + 1, np.uint64),
                 id_bytes=np.zeros(max(nid, 1), np.uint8))
        L.mo_export(h, *[_p(d[k]) for k in ("peak_off", "mz", "intensity", "scan_start_time", "tic", "prec_off", "prec_mz", "prec_intensity",
                                             "prec_intensity_some", "prec_charge", "prec_charge_some", "iso_kind", "iso_lo", "iso_hi", "id_off",
                                             "id_bytes")])
        d["id_bytes"] = d["id_bytes"][:nid]
        d["info"] = dict(n_lines=n_lines, n_records=n_rec, n_spectra=n, n_peaks=npk, n_precursors=npr, id_bytes=nid, malformed_lines=bad,
                         dropped_records=n_rec - n)
        return d
    finally:
        L.mo_destroy(h)


def parse_f32(tokens) -> tuple[np.ndarray, np.ndarray]:
    """str::parse::<f32> of each token (str or bytes) -> (values as u32 bits, ok as bool); a failed parse gives bits 0."""
    bs = [t.encode() if isinstance(t, str) else bytes(t) for t in tokens]
    off = np.zeros(len(bs) + 1, np.uint64)
    off[1:] = np.cumsum([len(b) for b in bs])
    out, ok = np.zeros(len(bs), np.float32), np.zeros(len(bs), np.uint8)
    lib().mo_parse_f32(b"".join(bs), _p(off), len(bs), _p(out), _p(ok))
    return out.view(np.uint32), ok.astype(bool)
