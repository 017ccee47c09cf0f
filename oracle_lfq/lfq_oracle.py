"""ctypes binding of the CPU oracle of label-free quantification (oracle_lfq/lfq_oracle.cpp).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__ and tools/bench_lfq.py. Never imported by the sage_b200 package.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "lfq_oracle.cpp")
_SO = os.path.join(_HERE, "_build", "liblfq_oracle.so")
# no FMA contraction, no fast-math: every f32/f64 operation stays separately rounded, as rustc emits it
CXXFLAGS = ["-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-pthread", "-Wall"]

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
        _lib.lo_create.restype = C.c_void_p
        _lib.lo_destroy.argtypes = [C.c_void_p]
        for f in ("lo_n_ranges", "lo_n_pages", "lo_n_grids", "lo_integrate"):
            getattr(_lib, f).restype = C.c_uint64
            getattr(_lib, f).argtypes = [C.c_void_p] + ([C.c_int] + [C.c_void_p] * 7 if f == "lo_integrate" else [])
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def peptide_isotopes(carbons: int, sulfurs: int) -> np.ndarray:
    """isotopes.rs:43-50"""
    out = np.zeros(3, np.float32)
    lib().lo_peptide_isotopes(C.c_uint16(carbons), C.c_uint16(sulfurs), _p(out))
    return out


class LfqOracle:
    """build_feature_map + quantify on the CPU. Arguments as sage_b200.FeatureMap.build; `peptides` needs seq_off and seq."""

    def __init__(self, peptides, settings, precursor_charge, features, alignments):
        from sage_b200.api import LFQ_FEATURE_FIELDS, _LFQ_FEATURE_TYPES
        self._keep = []
        cols = [np.ascontiguousarray(features[f], dtype=t) for f, t in zip(LFQ_FEATURE_FIELDS, _LFQ_FEATURE_TYPES)]
        al = np.ascontiguousarray(alignments)
        al = np.ascontiguousarray(al.view(np.float32).reshape(-1, 3) if al.dtype.names else np.asarray(al, np.float32).reshape(-1, 3))
        self.n_files = len(al)
        self.params = settings._c(precursor_charge)
        seq_off = np.ascontiguousarray(peptides.seq_off, np.uint32)
        seq = np.ascontiguousarray(peptides.seq, np.uint8)
        self._h = C.c_void_p(lib().lo_create(C.byref(self.params), C.c_uint64(len(cols[0])), *[_p(c) for c in cols], C.c_uint64(self.n_files), _p(al),
                                             C.c_uint64(len(seq_off) - 1), _p(seq_off), _p(seq)))

    def __del__(self):
        if getattr(self, "_h", None):
            lib().lo_destroy(self._h)
            self._h = None

    def export_map(self):
        from sage_b200.api import LFQ_RANGE_DTYPE
        ranges = np.zeros(lib().lo_n_ranges(self._h), LFQ_RANGE_DTYPE)
        min_rts = np.zeros(lib().lo_n_pages(self._h), np.float32)
        lib().lo_export_map(self._h, _p(ranges), _p(min_rts))
        return ranges, min_rts

    def add_ms1(self, batch):
        off = np.ascontiguousarray(batch.peak_off, np.uint64)
        arrs = [np.ascontiguousarray(x, t) for x, t in ((batch.masses, np.float32), (batch.intensities, np.float32), (batch.file_id, np.uint32),
                                                         (batch.scan_start_time, np.float32))]
        mob = None if batch.mobilities is None else np.ascontiguousarray(batch.mobilities, np.float32)
        lib().lo_add_ms1(self._h, C.c_uint64(len(batch)), _p(off), *[_p(a) for a in arrs], _p(mob))

    def export_grids(self):
        """keys [n, 3] (peptide, charge or 0, decoy) in (id, decoy) order and the matrices [n, n_files * 3, 100]."""
        n = lib().lo_n_grids(self._h)
        keys = np.zeros((n, 3), np.uint32)
        mats = np.zeros((n, self.n_files * 3, 100), np.float64)
        lib().lo_export_grids(self._h, _p(keys), _p(mats))
        return keys, mats

    def quantify(self, threads: int = 1) -> dict:
        """Every grid in (id, decoy) order: present (False where integrate returned None), rt, spectral_angle, score, areas, and margin, the smallest
        relative gap of a decision whose outcome depends on acos (inf when there is none)."""
        n = lib().lo_n_grids(self._h)
        keys = np.zeros((n, 3), np.uint32)
        present = np.zeros(n, np.uint8)
        rt = np.zeros(n, np.uint32)
        sa, score, margin = np.zeros(n), np.zeros(n), np.zeros(n)
        areas = np.zeros((n, self.n_files))
        lib().lo_integrate(self._h, int(threads), _p(keys), _p(present), _p(rt), _p(sa), _p(score), _p(areas), _p(margin))
        return dict(id=keys[:, 0].copy(), charge=keys[:, 1].astype(np.uint8), decoy=keys[:, 2].astype(bool), present=present.astype(bool), rt=rt, spectral_angle=sa,
                    score=score, areas=areas, margin=margin)
