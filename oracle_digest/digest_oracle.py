"""ctypes binding of the CPU oracle's digest with bulk accessors (oracle_digest/digest_oracle.cpp, which compiles oracle/sage_oracle.cpp).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__ and tools/bench_digest.py. Never imported by the sage_b200 package.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "digest_oracle.cpp")
_DEP = os.path.join(os.path.dirname(_HERE), "oracle", "sage_oracle.cpp")
_SO = os.path.join(_HERE, "_build", "libdigest_oracle.so")
# the oracle's own flags (oracle/Makefile): no FMA contraction, no fast-math
CXXFLAGS = ["-O3", "-march=x86-64-v3", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-fPIC", "-shared", "-Wall",
            "-Wno-unused-function"]

_lib = None


def build(force: bool = False) -> str:
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(_SRC), os.path.getmtime(_DEP)):
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
        _lib.sod_digest.restype = C.c_void_p
        _lib.sod_prefilter.restype = C.c_void_p
        _lib.sod_auto_chunk_size.restype = C.c_uint64
        for f in ("sod_free", "sod_sizes", "sod_export", "sod_db_sizes", "sod_db_export", "sod_pf_free", "sod_pf_info", "sod_pf_sizes", "sod_pf_export"):
            getattr(_lib, f).restype = None
    return _lib


def _build_params(kw: dict, keep: list):
    from oracle.oracle import KIND, BuildParams
    bp = BuildParams()
    bp.bucket_size = kw.get("bucket_size", 8192)
    bp.missed_cleavages = kw.get("missed_cleavages", 0)
    bp.min_len, bp.max_len = kw.get("min_len", 5), kw.get("max_len", 50)
    bp.cleave_at, bp.restrict_ = kw.get("cleave_at", "KR").encode(), kw.get("restrict", "P").encode()
    bp.c_terminal, bp.semi_enzymatic = int(kw.get("c_terminal", True)), int(kw.get("semi_enzymatic", False))
    bp.peptide_min_mass, bp.peptide_max_mass = kw.get("peptide_min_mass", 500.0), kw.get("peptide_max_mass", 5000.0)
    kinds = (C.c_uint8 * 2)(KIND["b"], KIND["y"])
    bp.ion_kinds, bp.n_kinds, bp.min_ion_index = kinds, 2, 2
    sm = list((kw.get("static_mods") or {}).items())
    sspec = (C.c_char_p * max(1, len(sm)))(*[k.encode() for k, _ in sm])
    smass = (C.c_float * max(1, len(sm)))(*[v for _, v in sm])
    bp.static_mod_specs, bp.static_mod_masses, bp.n_static = sspec, smass, len(sm)
    vm = [(k, m) for k, ms in (kw.get("variable_mods") or {}).items() for m in ms]
    vspec = (C.c_char_p * max(1, len(vm)))(*[k.encode() for k, _ in vm])
    vmass = (C.c_float * max(1, len(vm)))(*[v for _, v in vm])
    bp.var_mod_specs, bp.var_mod_masses, bp.n_var = vspec, vmass, len(vm)
    bp.max_variable_mods = kw.get("max_variable_mods", 2)
    bp.decoy_tag = kw.get("decoy_tag", "rev_").encode()
    bp.generate_decoys = int(kw.get("generate_decoys", True))
    keep += [kinds, sspec, smass, vspec, vmass]
    return bp


def _table(sizes_fn, export_fn, h) -> dict:
    sz = np.zeros(4, np.uint64)
    sizes_fn(h, sz.ctypes.data_as(C.c_void_p))
    n, nres, nref, nb = (int(x) for x in sz)
    t = dict(seq_off=np.empty(n + 1, np.uint32), seq=np.empty(nres, np.uint8), mods=np.empty(nres, np.float32), nterm=np.empty(n, np.float32),
             cterm=np.empty(n, np.float32), mono=np.empty(n, np.float32), decoy=np.empty(n, np.uint8), missed=np.empty(n, np.uint8),
             semi=np.empty(n, np.uint8), prot_off=np.empty(n + 1, np.uint64), name_off=np.empty(nref + 1, np.uint64), names=np.empty(max(nb, 1), np.uint8))
    export_fn(h, *[t[k].ctypes.data_as(C.c_void_p) for k in ("seq_off", "seq", "mods", "nterm", "cterm", "mono", "decoy", "missed", "semi", "prot_off",
                                                             "name_off", "names")])
    return t


def digest(fasta, **kw) -> dict:
    """The oracle's digest() of FASTA text (str or bytes) with OracleDB.from_fasta's keywords: the peptide table in PeptideIx order with
    semi_enzymatic, and every peptide's proteins as a CSR of name strings (prot_off into name_off into names)."""
    text = fasta.encode() if isinstance(fasta, str) else bytes(fasta)
    keep: list = []
    bp = _build_params(kw, keep)
    L = lib()
    h = C.c_void_p(L.sod_digest(C.c_char_p(text), C.byref(bp)))
    try:
        return _table(L.sod_sizes, L.sod_export, h)
    finally:
        L.sod_free(h)


def db_table(db) -> dict:
    """The same table of a database the oracle built from FASTA (OracleDB.from_fasta)."""
    L = lib()
    return _table(L.sod_db_sizes, L.sod_db_export, db.h)


def protein_lists(t: dict) -> list:
    """Each peptide's proteins as a list of bytes, in stored order."""
    raw = t["names"].tobytes()
    no, po = t["name_off"], t["prot_off"]
    return [[raw[no[j]:no[j + 1]] for j in range(po[i], po[i + 1])] for i in range(len(po) - 1)]


def auto_chunk_size(fasta, **kw) -> int:
    """Parameters::auto_calculate_prefilter_chunk_size (database.rs:142-160) of FASTA text with OracleDB.from_fasta's keywords (0 where the
    reference's chunks(0) would panic)."""
    text = fasta.encode() if isinstance(fasta, str) else bytes(fasta)
    keep: list = []
    bp = _build_params(kw, keep)
    return int(lib().sod_auto_chunk_size(C.c_char_p(text), C.byref(bp)))


def prefilter(fasta, spectra: dict, cfg, chunk_size: int = 0, low_memory: bool = True, min_peaks: int = 15, **kw):
    """The oracle's prefilter (runner.rs:104-128, 161-278) of FASTA text: spectra as OracleDB.score_batch takes them, cfg an oracle
    ScorerConfig (report_psms as the search's: the chunk scorers add 1), kw OracleDB.from_fasta's keywords. Returns (table, info) with the
    table of digest() and info = dict(chunk_size, n_chunks, plain_build, rows, kept); None when the chunk size is 0."""
    text = fasta.encode() if isinstance(fasta, str) else bytes(fasta)
    keep: list = []
    bp = _build_params(kw, keep)
    f32 = lambda x: np.ascontiguousarray(x, np.float32)  # noqa: E731
    arrs = [np.ascontiguousarray(spectra["peak_off"], np.uint64), f32(spectra["masses"]), f32(spectra["intensities"]), f32(spectra["prec_mz"]),
            np.ascontiguousarray(spectra["prec_charge"], np.uint8), f32(spectra["iso_lo"]), f32(spectra["iso_hi"]), f32(spectra["tic"])]
    level = None if spectra.get("level") is None else np.ascontiguousarray(spectra["level"], np.uint8)
    sp = cfg.to_c()
    L = lib()
    h = L.sod_prefilter(C.c_char_p(text), C.byref(bp), C.byref(sp), C.c_uint64(int(chunk_size)), C.c_int(int(bool(low_memory))), C.c_uint64(int(min_peaks)),
                        C.c_uint64(len(arrs[3])), *[a.ctypes.data_as(C.c_void_p) for a in arrs], None if level is None else level.ctypes.data_as(C.c_void_p))
    if not h:
        return None
    h = C.c_void_p(h)
    try:
        head = np.zeros(3, np.uint64)
        L.sod_pf_info(h, head.ctypes.data_as(C.c_void_p), None, None)
        rows, kept = np.zeros(int(head[1]), np.uint64), np.zeros(int(head[1]), np.uint64)
        L.sod_pf_info(h, head.ctypes.data_as(C.c_void_p), rows.ctypes.data_as(C.c_void_p), kept.ctypes.data_as(C.c_void_p))
        info = dict(chunk_size=int(head[0]), n_chunks=int(head[1]), plain_build=int(head[2]), rows=rows, kept=kept)
        return _table(L.sod_pf_sizes, L.sod_pf_export, h), info
    finally:
        L.sod_pf_free(h)
