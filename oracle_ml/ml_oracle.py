"""ctypes binding of the CPU oracle of PSM rescoring (oracle_ml/ml_oracle.cpp).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__ and tools/bench_rescore.py. Never imported by the sage_b200 package.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "ml_oracle.cpp")
_SO = os.path.join(_HERE, "_build", "libml_oracle.so")
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
        _lib.mo_spectrum_fdr.restype = C.c_double
        _lib.mo_spectrum_fdr.argtypes = [C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_uint64] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 9
        _lib.mo_kde_build.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_int, C.c_double, C.c_int] + [C.c_void_p] * 3
        _lib.mo_lda_train.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_void_p]
        _lib.mo_rt_embed.argtypes = [C.c_int, C.c_void_p, C.c_uint64, C.c_float, C.c_uint32, C.c_void_p]
        _lib.mo_linreg_fit.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.mo_predict_rt.restype = C.c_double
        _lib.mo_predict_rt.argtypes = [C.c_void_p] * 5 + [C.c_uint64, C.c_uint64, C.c_int] + [C.c_void_p] * 13
        _lib.mo_picked_fdr.argtypes = [C.c_void_p] * 9 + [C.c_char_p, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int] + [C.c_void_p] * 5
        _lib.mo_picked_precursor.restype = C.c_uint64
        _lib.mo_picked_precursor.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        _lib.mo_protein_groups.restype = C.c_uint64
        _lib.mo_protein_groups.argtypes = [C.c_void_p] * 8 + [C.c_uint64, C.c_int, C.c_int, C.c_float, C.c_int, C.c_char_p, C.c_int] + [C.c_void_p] * 4
        _lib.mo_grouping_text.argtypes = [C.c_void_p]
        _lib.mo_bipartite_cover.restype = C.c_uint64
        _lib.mo_bipartite_cover.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p]
        _lib.mo_format_hashes.argtypes = [C.c_int, C.c_uint64, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_int]
        _lib.mo_format_one.restype = C.c_uint64
        _lib.mo_format_one.argtypes = [C.c_int, C.c_double, C.c_char_p, C.c_uint64, C.c_void_p]
        _lib.mo_write_fragments.restype = C.c_uint64
        _lib.mo_write_fragments.argtypes = [C.c_void_p] * 3 + [C.c_uint64, C.c_void_p, C.c_int]
        _lib.mo_write_tmt.restype = C.c_uint64
        _lib.mo_write_tmt.argtypes = [C.c_void_p] * 8 + [C.c_uint64, C.c_uint64, C.c_int, C.c_int]
        _lib.mo_take_text.argtypes = [C.c_void_p]
        _lib.mo_write_results.restype = C.c_uint64
        _lib.mo_write_results.argtypes = [C.c_int] + [C.c_void_p] * 4 + [C.c_uint64] + [C.c_void_p] * 6 + [C.c_int]
        _lib.mo_write_lfq.restype = C.c_uint64
        _lib.mo_write_lfq.argtypes = [C.c_void_p] * 3 + [C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int]
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def default_threads() -> int:
    return max(1, len(os.sched_getaffinity(0)))


def kde_build(scores, decoy, bins=1000, monotonic=True, bw_factor=1.0, threads=None):
    """kde::Builder::build: (PEP per bin, min_score, score_step)."""
    s = np.ascontiguousarray(scores, np.float64)
    d = np.ascontiguousarray(decoy, np.uint8)
    out = np.zeros(int(bins))
    lo, step = C.c_double(), C.c_double()
    lib().mo_kde_build(_p(s), _p(d), len(s), int(bins), int(monotonic), float(bw_factor), int(threads or default_threads()), _p(out), C.byref(lo), C.byref(step))
    return out, lo.value, step.value


def lda_train(X, decoy):
    """LinearDiscriminantAnalysis::train on any [n, D] matrix: (coef, eps), or None when the reference returns None."""
    X = np.ascontiguousarray(X, np.float64)
    d = np.ascontiguousarray(decoy, np.uint8)
    coef = np.zeros(X.shape[1])
    eps = C.c_double()
    if not lib().mo_lda_train(_p(X), _p(d), X.shape[0], X.shape[1], _p(coef), C.byref(eps)):
        return None
    return coef, eps.value


def spectrum_fdr(features, precursor_tol, aligned_rt=None, delta_rt_model=None, delta_ims_model=None, threads=None, with_features=False) -> dict:
    """runner.rs spectrum_fdr on the CPU; the same keys as sage_b200.spectrum_fdr, plus `seconds` (wall time) and `threads`."""
    rows = np.ascontiguousarray(features)
    assert rows.dtype.itemsize == 128
    n = len(rows)
    cols = [None if c is None else np.ascontiguousarray(c, np.float32) for c in (aligned_rt, delta_rt_model, delta_ims_model)]
    disc, pep, q = np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)
    order = np.zeros(n, np.uint32)
    passing, fitted = C.c_uint64(), C.c_int32()
    coef, eps = np.zeros(20), C.c_double()
    feats = np.zeros((n, 20)) if with_features else None
    threads = int(threads or default_threads())
    secs = lib().mo_spectrum_fdr(precursor_tol.kind, precursor_tol.lo, precursor_tol.hi, _p(rows), n, *[_p(c) for c in cols], threads, _p(disc), _p(pep),
                                 _p(q), _p(order), C.byref(passing), C.byref(fitted), _p(coef), C.byref(eps), _p(feats))
    res = dict(discriminant_score=disc, posterior_error=pep, spectrum_q=q, order=order, passing=passing.value, lda_fitted=bool(fitted.value), coef=coef,
               eps=eps.value, seconds=secs, threads=threads)
    if with_features:
        res["features"] = feats
    return res


def rt_embed(model: int, sequence, monoisotopic: float, charge: int = 2) -> np.ndarray:
    """RetentionModel::embed (model 0, 69 features) or MobilityModel::embed (model 1, 100 features) of one peptide."""
    seq = np.frombuffer(sequence.encode() if isinstance(sequence, str) else bytes(sequence), np.uint8).copy()
    out = np.zeros(69 if model == 0 else 100)
    lib().mo_rt_embed(int(model), _p(seq), len(seq), float(monoisotopic), int(charge), _p(out))
    return out


def linreg_fit(X, y, threads=None):
    """LinearRegression::fit over a given [n, d] matrix (every row passes the filter): (beta, r2, eps), or None when the reference returns None."""
    X = np.ascontiguousarray(X, np.float64)
    y = np.ascontiguousarray(y, np.float64)
    beta, r2, eps = np.zeros(X.shape[1]), C.c_double(), C.c_double()
    if not lib().mo_linreg_fit(_p(X), _p(y), len(y), X.shape[1], int(threads or default_threads()), _p(beta), C.byref(r2), C.byref(eps)):
        return None
    return beta, r2.value, eps.value


def predict_rt(peptides, features, file_id, n_files, threads=None) -> dict:
    """runner.rs:513-531 on the CPU; the same keys as sage_b200.predict_rt (stage times aside), plus `seconds` (wall time) and `threads`."""
    rows = np.ascontiguousarray(features)
    assert rows.dtype.itemsize == 128
    n = len(rows)
    fid = np.ascontiguousarray(file_id, np.uint32)
    off, seq, mono = (np.ascontiguousarray(a, t) for a, t in ((peptides.seq_off, np.uint32), (peptides.seq, np.uint8), (peptides.mono, np.float32)))
    cols = {c: np.zeros(n, np.float32) for c in ("aligned_rt", "predicted_rt", "delta_rt_model", "predicted_ims", "delta_ims_model", "spectrum_q")}
    align = np.zeros((int(n_files), 3), np.float32)
    stats, fitted = np.zeros(2, np.uint64), np.zeros(2, np.int32)
    r2, eps, rt_beta, ims_beta = np.zeros(2), np.zeros(2), np.zeros(69), np.zeros(100)
    threads = int(threads or default_threads())
    secs = lib().mo_predict_rt(_p(off), _p(seq), _p(mono), _p(rows), _p(fid), n, int(n_files), threads, *[_p(cols[c]) for c in cols], _p(align), _p(stats),
                               _p(fitted), _p(r2), _p(eps), _p(rt_beta), _p(ims_beta))
    from sage_b200.api import ALIGNMENT_DTYPE
    res = dict(cols, alignments=align.view(ALIGNMENT_DTYPE).reshape(-1), training_rows=int(stats[0]), aligned_peptides=int(stats[1]),
               rt_fitted=bool(fitted[0]), rt_r2=float(r2[0]), rt_eps=float(eps[0]), rt_beta=rt_beta, ims_fitted=bool(fitted[1]), ims_r2=float(r2[1]),
               ims_eps=float(eps[1]), ims_beta=ims_beta, seconds=secs, threads=threads)
    return res


class PickedClash(ValueError):
    """Two distinct peptides on one side with one key: the reference panics at fdr.rs:149."""


def _name_table(proteins):
    names = [nm.encode() for lst in proteins for nm in lst]
    prot_off = np.zeros(len(proteins) + 1, np.uint32)
    prot_off[1:] = np.cumsum([len(lst) for lst in proteins])
    name_off = np.zeros(len(names) + 1, np.uint64)
    name_off[1:] = np.cumsum([len(b) for b in names])
    chars = np.frombuffer(b"".join(names) + b"\0", np.uint8).copy()
    return prot_off, name_off, chars


def picked_fdr(peptides, pep_idx, score, proteins, cterm=None, generate_decoys=True, decoy_tag="rev_", threads=None) -> dict:
    """picked_peptide then picked_protein (fdr.rs) on the CPU with real key strings. `peptides` has seq_off, seq, mods, nterm and decoy;
    proteins[p] is Peptide::proteins of peptide p (a list of names). The same keys as sage_b200.picked_fdr (stage times aside), plus `seconds`."""
    import time
    off, seq, mods, nterm, dec = (np.ascontiguousarray(a, t) for a, t in ((peptides.seq_off, np.uint32), (peptides.seq, np.uint8), (peptides.mods, np.float32),
                                                                             (peptides.nterm, np.float32), (peptides.decoy, np.uint8)))
    ct = None if cterm is None else np.ascontiguousarray(cterm, np.float32)
    names = [nm.encode() for lst in proteins for nm in lst]
    prot_off = np.zeros(len(proteins) + 1, np.uint32)
    prot_off[1:] = np.cumsum([len(lst) for lst in proteins])
    name_off = np.zeros(len(names) + 1, np.uint64)
    name_off[1:] = np.cumsum([len(b) for b in names])
    chars = np.frombuffer(b"".join(names) + b"\0", np.uint8).copy()
    idx = np.ascontiguousarray(pep_idx, np.uint32)
    disc = np.ascontiguousarray(score, np.float32)
    n = len(idx)
    pq, rq = np.zeros(n, np.float32), np.zeros(n, np.float32)
    passing, entries, clash = np.zeros(2, np.uint64), np.zeros(2, np.uint64), np.zeros(2, np.uint32)
    t0 = time.perf_counter()
    rc = lib().mo_picked_fdr(_p(off), _p(seq), _p(mods), _p(nterm), _p(ct), _p(dec), _p(prot_off), _p(name_off), _p(chars), decoy_tag.encode(),
                             int(bool(generate_decoys)), _p(idx), _p(disc), n, int(threads or default_threads()), _p(pq), _p(rq), _p(passing), _p(entries),
                             _p(clash))
    if rc != 0:
        raise PickedClash(f"peptides {clash[0]} and {clash[1]} share a key on one side")
    return dict(peptide_q=pq, protein_q=rq, peptide_passing=int(passing[0]), protein_passing=int(passing[1]), peptide_entries=int(entries[0]),
                protein_entries=int(entries[1]), seconds=time.perf_counter() - t0)


def picked_precursor(score, decoy):
    """picked_precursor (fdr.rs:228-287) on the CPU over the rows in the given order: (q per row, passing)."""
    s = np.ascontiguousarray(score, np.float64)
    d = np.ascontiguousarray(decoy, np.uint8)
    q = np.zeros(len(s), np.float32)
    passing = lib().mo_picked_precursor(_p(s), _p(d), len(s), _p(q))
    return q, int(passing)


GROUPING_STATS = ("peptides", "meta_peptides", "groups", "covered", "greedy_picks", "annotated")


def protein_groups(decoy, proteins, pep_idx, label, peptide_q, score, protein_grouping=True, threshold=0.01, generate_decoys=True, decoy_tag="rev_",
                   threads=None) -> dict:
    """generate_protein_groups then picked_protein_group (protein_grouping.rs, fdr.rs:192-226) on the CPU with real name strings. decoy[p] is
    Peptide::decoy and proteins[p] Peptide::proteins (a list of names) of peptide p; threshold None is the reference's None. Returns
    protein_groups (the strings), num_protein_groups, pass, protein_group_q per row; tables (per pass, a list of (covered, decoy, raw names
    sorted and joined with '/') in group order); per-pass counts as 2-element lists (GROUPING_STATS); passing, entries, seconds, threads."""
    import time
    prot_off, name_off, chars = _name_table(proteins)
    dec = np.ascontiguousarray(decoy, np.uint8)
    idx = np.ascontiguousarray(pep_idx, np.uint32)
    lab = np.ascontiguousarray(label, np.int32)
    pq = np.ascontiguousarray(peptide_q, np.float32)
    disc = np.ascontiguousarray(score, np.float32)
    n = len(idx)
    num, passes, q, stats = np.zeros(n, np.uint32), np.zeros(n, np.uint8), np.zeros(n, np.float32), np.zeros(14, np.uint64)
    threads = int(threads or default_threads())
    t0 = time.perf_counter()
    size = lib().mo_protein_groups(_p(prot_off), _p(name_off), _p(chars), _p(dec), _p(idx), _p(lab), _p(pq), _p(disc), n, int(bool(protein_grouping)),
                                   int(threshold is not None), float("nan") if threshold is None else float(threshold), int(bool(generate_decoys)),
                                   decoy_tag.encode(), threads, _p(num), _p(passes), _p(q), _p(stats))
    secs = time.perf_counter() - t0
    buf = np.zeros(size, np.uint8)
    lib().mo_grouping_text(_p(buf))
    lines = buf.tobytes().decode().split("\n")[:-1] if size else []
    st = stats.reshape(-1)
    res = dict(protein_groups=lines[:n], num_protein_groups=num, **{"pass": passes}, protein_group_q=q, passing=int(st[12]), entries=int(st[13]),
               seconds=secs, threads=threads)
    res.update({k: [int(st[j]), int(st[6 + j])] for j, k in enumerate(GROUPING_STATS)})
    tables, at = [], n
    for k in range(2):
        g = res["groups"][k]
        tables.append([(int(c), int(d), names) for c, d, names in (ln.split(" ", 2) for ln in lines[at:at + g])])
        at += g
    res["tables"] = tables
    return res


def bipartite_cover(left, right, n_left, n_right):
    """BipartiteGraph::new(edges, n_left, n_right).into_cover(), the literal loop: (cover as bools, add_largest picks)."""
    lft = np.ascontiguousarray(left, np.uint32)
    rgt = np.ascontiguousarray(right, np.uint32)
    cover = np.zeros(int(n_left), np.uint8)
    picks = lib().mo_bipartite_cover(_p(lft), _p(rgt), len(lft), int(n_left), int(n_right), _p(cover))
    return cover.astype(bool), int(picks)


# ------------------------------------------------------------------------------------------------ result files (runner.rs writers)
def format_hashes(fmt: int, first: int = 0, values=None, n: int = 0, block: int = 1 << 16, threads=None) -> np.ndarray:
    """Per-block FNV-1a 64 of formatted values (each followed by '\n'): fmt 0 ryu f32 of bits first + i, 1 `{:+}` of that f32, 2 ryu f64."""
    v = None if values is None else np.ascontiguousarray(values, np.float64)
    n = len(v) if v is not None else n
    out = np.zeros(n // block, np.uint64)
    lib().mo_format_hashes(fmt, first, _p(v), n, block, _p(out), int(threads or default_threads()))
    return out


def format_one(fmt: int, x: float = 0.0, s: bytes = b"") -> str:
    """One value: fmt 0 ryu f32, 1 `{:+}` f32, 2 ryu f64, 3 the csv field of bytes s."""
    buf = C.create_string_buffer(2 * len(s) + 128)
    n = lib().mo_format_one(fmt, float(x), s, len(s), buf)
    return buf.raw[:n].decode("latin-1")


def _take(n: int) -> bytes:
    buf = C.create_string_buffer(max(n, 1))
    lib().mo_take_text(buf)
    return buf.raw[:n]


def write_fragments(psm_id, frag_offset, frag_count, fragments, threads=None) -> bytes:
    """matched_fragments.sage.tsv; fragments: a structured array in sage_b200_fragment's layout."""
    a = [np.ascontiguousarray(psm_id, np.uint64), np.ascontiguousarray(frag_offset, np.uint32), np.ascontiguousarray(frag_count, np.uint32)]
    fr = np.ascontiguousarray(fragments)
    n = lib().mo_write_fragments(_p(a[0]), _p(a[1]), _p(a[2]), len(a[0]), _p(fr), int(threads or default_threads()))
    return _take(n)


def write_tmt(filenames, spec_ids, file_id, spec, injection, peaks, user_labels=False, threads=None) -> bytes:
    """tmt.tsv; filenames / spec_ids: lists of bytes."""
    def csr(strs):
        off = np.concatenate([[0], np.cumsum([len(s) for s in strs])]).astype(np.uint64)
        return off, np.frombuffer(b"".join(strs) + b"\0", np.uint8)
    fo, fb = csr(filenames)
    so, sb = csr(spec_ids)
    fi, si = np.ascontiguousarray(file_id, np.uint32), np.ascontiguousarray(spec, np.uint32)
    inj = np.ascontiguousarray(injection, np.float32)
    pk = np.ascontiguousarray(peaks, np.float32).reshape(len(fi), -1)
    n = lib().mo_write_tmt(_p(fo), _p(fb), _p(so), _p(sb), _p(fi), _p(si), _p(inj), _p(pk), len(fi), pk.shape[1], int(user_labels),
                           int(threads or default_threads()))
    return _take(n)


class _WoTable(C.Structure):
    _fields_ = [(f, C.c_void_p) for f in ("res_off", "seq", "mods", "nterm", "cterm", "decoy", "semi", "prot_off", "prot_ids", "name_off",
                                          "name_bytes")] + [("tag", C.c_char_p), ("generate_decoys", C.c_int)]


_COLS = ("discriminant", "posterior", "spectrum_q", "peptide_q", "protein_q", "protein_group_q", "aligned_rt", "predicted_rt", "delta_rt",
         "predicted_ims", "delta_ims", "num_groups", "group_pass", "row_group_off", "row_groups", "group_off", "group_members", "group_decoy")


class _WoColumns(C.Structure):
    _fields_ = [(f, C.c_void_p) for f in _COLS]


def _csr(strs, keep):
    bs = [s.encode() if isinstance(s, str) else bytes(s) for s in strs]
    off = np.concatenate([[0], np.cumsum([len(b) for b in bs], dtype=np.uint64)]).astype(np.uint64)
    data = np.frombuffer(b"".join(bs) + b"\0", np.uint8)
    keep += [off, data]
    return _p(off), _p(data)


def _table(digest, decoy_tag, generate_decoys, keep):
    P = digest.peptides
    arrs = [np.ascontiguousarray(a, dt) for a, dt in ((P.seq_off, np.uint32), (P.seq, np.uint8), (P.mods, np.float32), (P.nterm, np.float32),
                                                       (digest.cterm, np.float32), (P.decoy, np.uint8), (digest.semi_enzymatic, np.uint8),
                                                       (digest.protein_offsets, np.uint32), (digest.protein_ids, np.uint32))]
    keep += arrs
    no, nb = _csr(digest.names, keep)
    tag = decoy_tag.encode()
    keep.append(tag)
    return _WoTable(*[_p(a) for a in arrs], no, nb, tag, int(bool(generate_decoys)))


def _column(d, key, dt, keep):
    if d is None or d.get(key) is None:
        return None
    a = np.ascontiguousarray(d[key], dt)
    keep.append(a)
    return _p(a)


def write_results(digest, rows, psm_id, file_id, spec_index, filenames, spec_ids, fdr=None, rt=None, picked=None, groups=None, decoy_tag="rev_",
                  generate_decoys=True, pin=False, threads=None) -> bytes:
    """results.sage.tsv (pin=False) or results.sage.pin; the dicts are those of the library's spectrum_fdr, predict_rt, picked_fdr, protein_groups."""
    keep = []
    rows = np.ascontiguousarray(rows)
    t = _table(digest, decoy_tag, generate_decoys, keep)
    src = dict(discriminant=(fdr, "discriminant_score", np.float32), posterior=(fdr, "posterior_error", np.float32), spectrum_q=(fdr, "spectrum_q", np.float32),
               peptide_q=(picked, "peptide_q", np.float32), protein_q=(picked, "protein_q", np.float32),
               protein_group_q=(groups, "protein_group_q", np.float32), aligned_rt=(rt, "aligned_rt", np.float32), predicted_rt=(rt, "predicted_rt", np.float32),
               delta_rt=(rt, "delta_rt_model", np.float32), predicted_ims=(rt, "predicted_ims", np.float32), delta_ims=(rt, "delta_ims_model", np.float32),
               num_groups=(groups, "num_protein_groups", np.uint32), group_pass=(groups, "pass", np.uint8), row_group_off=(groups, "row_group_offsets", np.uint64),
               row_groups=(groups, "row_groups", np.uint32), group_off=(groups, "group_offsets", np.uint64), group_members=(groups, "group_members", np.uint32),
               group_decoy=(groups, "group_decoy", np.uint8))
    c = _WoColumns(*[_column(*src[k], keep) for k in _COLS])
    fo, fb = _csr(filenames, keep)
    so, sb = _csr(spec_ids, keep)
    a = [np.ascontiguousarray(psm_id, np.uint64), np.ascontiguousarray(file_id, np.uint32), np.ascontiguousarray(spec_index, np.uint32)]
    n = lib().mo_write_results(int(pin), _p(rows), _p(a[0]), _p(a[1]), _p(a[2]), len(rows), fo, fb, so, sb, C.byref(t), C.byref(c),
                               int(threads or default_threads()))
    return _take(n)


def write_lfq(digest, lfq_rows, areas, q_value, filenames, decoy_tag="rev_", generate_decoys=True, threads=None) -> bytes:
    """lfq.tsv over sage_b200_lfq_integrate's rows (a structured array in sage_b200_lfq_row's layout), areas [n, files] and q-values."""
    keep = []
    t = _table(digest, decoy_tag, generate_decoys, keep)
    r = np.ascontiguousarray(lfq_rows)
    ar = np.ascontiguousarray(areas, np.float64).reshape(len(r), len(filenames))
    q = np.ascontiguousarray(q_value, np.float32)
    fo, fb = _csr(filenames, keep)
    n = lib().mo_write_lfq(_p(r), _p(ar), _p(q), len(r), fo, fb, len(filenames), C.byref(t), int(threads or default_threads()))
    return _take(n)
