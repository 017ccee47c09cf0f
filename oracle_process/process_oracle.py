"""ctypes binding of the CPU oracle of SpectrumProcessor::process for every MS level (oracle_process/process_oracle.cpp).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__ and tools/bench_process.py. Never imported by the sage_b200 package.
so_process composes the two oracles as spectrum.rs:338-412 does: level 2 is oracle.process_ms2 (oracle/sage_oracle.cpp), every other
level is po_process_other, which keeps every peak.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "process_oracle.cpp")
_SO = os.path.join(_HERE, "_build", "libprocess_oracle.so")
# no FMA contraction, no fast-math: every f32 operation stays one separately rounded SSE instruction, as rustc emits it
CXXFLAGS = ["-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall"]

_lib = None


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
        _lib.po_process_other.restype = C.c_float
        _lib.po_process_other.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def process_one(mz, intensity, level: int, mobility=None, precursor_charge=None, take_top_n=150, deisotope=False, min_deisotope_mz=0.0):
    """SpectrumProcessor::new(take_top_n, deisotope, min_deisotope_mz).process(one RawSpectrum) -> (masses, intensities, mobilities, tic);
    mobilities is an empty array where ProcessedSpectrum::mobilities is empty."""
    mz, intensity = np.ascontiguousarray(mz, np.float32), np.ascontiguousarray(intensity, np.float32)
    if level == 2:
        from oracle import oracle as O
        m, i, tic = O.process_ms2(mz, intensity, precursor_charge, take_top_n, deisotope, min_deisotope_mz)
        return np.asarray(m, np.float32), np.asarray(i, np.float32), np.zeros(0, np.float32), np.float32(tic)
    mob = None if mobility is None else np.ascontiguousarray(mobility, np.float32)
    n = len(mz)
    om, oi = np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.float32)
    with_mob = level == 1 and mob is not None
    ob = np.zeros(max(n, 1), np.float32) if with_mob else None
    tic = lib().po_process_other(_p(mz), _p(intensity), _p(mob), n, level, _p(om), _p(oi), _p(ob))
    return om[:n].copy(), oi[:n].copy(), ob[:n].copy() if with_mob else np.zeros(0, np.float32), np.float32(tic)


def so_process(raw, take_top_n=150, deisotope=False, min_deisotope_mz=0.0) -> dict:
    """process() of every spectrum of a sage_b200.RawSpectra batch, flattened as SpectrumProcessor.process_raw returns it: peak_off,
    masses, intensities, mobilities (NaN where a spectrum has none), has_mobilities, tic, level."""
    off = np.asarray(raw.peak_off, np.int64)
    n = len(off) - 1
    chg = np.zeros(n, np.uint8) if raw.precursor_charge is None else np.asarray(raw.precursor_charge, np.uint8)
    ms, its, mbs, tic, has = [], [], [], np.zeros(n, np.float32), np.zeros(n, bool)
    out_off = np.zeros(n + 1, np.uint64)
    for s in range(n):
        a, b = off[s] - off[0], off[s + 1] - off[0]
        mob = None if raw.mobility is None else raw.mobility[a:b]
        m, i, mb, t = process_one(raw.mz[a:b], raw.intensity[a:b], int(raw.level[s]), mob, int(chg[s]) or None, take_top_n, deisotope, min_deisotope_mz)
        has[s] = int(raw.level[s]) == 1 and raw.mobility is not None
        ms.append(m)
        its.append(i)
        mbs.append(mb if has[s] else np.full(len(m), np.nan, np.float32))
        tic[s] = t
        out_off[s + 1] = out_off[s] + len(m)
    cat = (lambda x: np.concatenate(x).astype(np.float32) if x else np.zeros(0, np.float32))
    return dict(peak_off=out_off, masses=cat(ms), intensities=cat(its), mobilities=cat(mbs), has_mobilities=has, tic=tic,
                level=np.asarray(raw.level, np.uint8).copy())
