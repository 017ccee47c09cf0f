"""Result files on the device: every f32 in both layouts and 10^8 f64 format as the C++ oracle's std::to_chars restatement does, and
matched_fragments.sage.tsv / tmt.tsv are byte-identical to the oracle's, for any chunk budget."""
import csv
import io
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import write_reference as W  # noqa: E402
from oracle_ml import ml_oracle as M  # noqa: E402
from sage_b200 import Scorer, Tolerance, api, synth  # noqa: E402
from sage_b200.api import IndexedDatabase  # noqa: E402
from test_write_no_gpu import edge_f32, edge_f64  # noqa: E402

pytestmark = pytest.mark.gpu
BLOCK = 1 << 16


def first_mismatch(fmt, dev, ref, first=0, values=None):
    b = int(np.nonzero(dev != ref)[0][0])
    lo = b * BLOCK
    for i in range(lo, lo + BLOCK):   # drill down: one value per block
        if values is None:
            d = api.format_hashes(fmt, first + i, n=1, block=1)
            r = M.format_hashes(fmt, first + i, n=1, block=1)
            x = np.uint32(first + i).view(np.float32)
        else:
            d = api.format_hashes(fmt, values=values[i:i + 1], block=1)
            r = M.format_hashes(fmt, values=values[i:i + 1], block=1)
            x = values[i]
        if d[0] != r[0]:
            return f"format {fmt}: value {x!r} (index {i}) oracle {M.format_one(fmt, float(x))!r}"
    return f"format {fmt}: block {b} differs"


@pytest.mark.parametrize("fmt", [0, 1])
def test_every_f32(fmt):
    n = 1 << 32
    dev = api.format_hashes(fmt, 0, n=n, block=BLOCK)
    ref = M.format_hashes(fmt, 0, n=n, block=BLOCK)
    assert np.array_equal(dev, ref), first_mismatch(fmt, dev, ref)


def test_random_f64_and_edges():
    rng = np.random.default_rng(5)
    n = 100_000_000 // BLOCK * BLOCK
    edges = np.concatenate([edge_f64(), edge_f32()])
    x = rng.integers(0, 1 << 64, n, dtype=np.uint64).view(np.float64)
    x[:len(edges)] = edges
    dev = api.format_hashes(2, values=x, block=BLOCK)
    ref = M.format_hashes(2, values=x[:n // BLOCK * BLOCK], block=BLOCK)
    assert np.array_equal(dev, ref), first_mismatch(2, dev, ref, values=x)


def check_all_budgets(write, want):
    stats = {}
    assert write(0, stats) == want
    assert stats["chunks"] == 1 and stats["records"] > 0
    for budget in (1, 4096 * 40, len(want) // 3 + 1):
        st = {}
        assert write(budget, st) == want
        assert st["chunks"] >= 1


def test_fragments_from_search():
    pep = synth.make_peptides(20000, seed=41, static_c=True)
    spectra = synth.make_spectra(pep, 12000, seed=42)
    db = IndexedDatabase.build_from_peptides(pep, device=0)
    sc = Scorer(db, precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), report_psms=2, annotate_matches=True)
    feats, counts = sc.score_batch(spectra)
    frags = sc.last_fragments
    rows = np.concatenate([feats[i * 2:i * 2 + int(counts[i])] for i in range(len(counts))])
    assert len(rows) > 5000 and int(rows["fragment_count"].sum()) > 8192
    rows["fragment_count"][::97] = 0   # rows with no fragments
    pid = np.arange(len(rows), dtype=np.uint64) * 3 + 7
    want = M.write_fragments(pid, rows["fragment_offset"], rows["fragment_count"], frags)
    check_all_budgets(lambda b, st: api.write_fragments(rows, frags, pid, text_budget=b, stats=st), want)


def test_fragments_adversarial():
    rng = np.random.default_rng(8)
    specials = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 1e-45, -1e-45, 1.1754942e-38, 3.4028235e38, 1e13, 1e12, 1e-5, 1e-4], np.float32)
    n = 20000
    fr = np.zeros(n, api.FRAGMENT_DTYPE)
    fr["kind"] = rng.integers(0, 6, n)
    fr["charge"] = rng.integers(-2, 5, n)
    fr["ordinal"] = rng.integers(-1, 50, n)
    for f in ("intensity", "mz_calculated", "mz_experimental"):
        v = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
        v[::3] = specials[rng.integers(0, len(specials), len(v[::3]))]
        fr[f] = v
    rows = np.zeros(3000, api.FEATURE_DTYPE)
    rows["fragment_count"] = rng.integers(0, 12, len(rows))
    rows["fragment_offset"] = rng.integers(0, n - 12, len(rows))   # ranges anywhere in the array, overlapping
    pid = rng.integers(0, 1 << 63, len(rows), dtype=np.uint64)
    want = M.write_fragments(pid, rows["fragment_offset"], rows["fragment_count"], fr)
    assert want == W.write_fragments(pid, rows, fr)
    check_all_budgets(lambda b, st: api.write_fragments(rows, fr, pid, text_budget=b, stats=st), want)


@pytest.mark.parametrize("user", [False, True])
def test_tmt(user):
    rng = np.random.default_rng(9)
    files = ["run1.mzML", 'odd "name"\twith tab.mzML', "line\nbreak.mzML", ""]
    ids = ["controllerType=0 controllerNumber=1 scan=%d" % i for i in range(5000)] + ['quote"d', "cr\rid"]
    n = 30000
    fi, si = rng.integers(0, len(files), n), rng.integers(0, len(ids), n)
    inj = (rng.random(n) * 100).astype(np.float32)
    inj[::11] = np.float32(np.nan)
    ch = 18 if not user else 3
    peaks = (rng.random((n, ch)) * 1e7).astype(np.float32)
    peaks[::5, 0] = 0.0
    peaks[::7, -1] = -0.0
    peaks[1, :] = np.float32(np.inf)
    peaks[2, :] = rng.integers(0, 1 << 23, ch).astype(np.uint32).view(np.float32)   # subnormals
    want = M.write_tmt([f.encode() for f in files], [s.encode() for s in ids], fi, si, inj, peaks, user)
    check_all_budgets(lambda b, st: api.write_tmt(files, ids, fi, si, inj, peaks, user_labels=user, text_budget=b, stats=st), want)


def test_size_query_equals_written_length():
    import ctypes as C
    rows = np.zeros(2, api.FEATURE_DTYPE)
    rows["fragment_count"] = [1, 2]
    rows["fragment_offset"] = [0, 1]
    fr = np.zeros(3, api.FRAGMENT_DTYPE)
    fr["mz_calculated"] = [1.5, 2.5, 1e20]
    pid = np.array([1, 2], np.uint64)
    ci = api.CWriteInputs(rows=api._ptr(rows), psm_id=api._ptr(pid), n_rows=2, fragments=api._ptr(fr), n_fragments=3)
    lib = api.load_library()
    size = C.c_uint64()
    assert lib.sage_b200_write_tsv(0, api.FILE_FRAGMENTS, C.byref(ci), None, C.c_uint64(0), C.byref(size)) == 0
    want = W.write_fragments(pid, rows, fr)
    assert size.value == len(want)
    small = C.create_string_buffer(size.value)
    got = C.c_uint64()
    assert lib.sage_b200_write_tsv(0, api.FILE_FRAGMENTS, C.byref(ci), small, C.c_uint64(size.value - 1), C.byref(got)) == -5   # ELIMIT
    assert got.value == size.value and small.raw == b"\0" * size.value   # nothing written
    assert api.write_fragments(rows, fr, pid) == want


# ------------------------------------------------------------------------------------------------ results.sage.tsv, .pin, lfq.tsv
def fake_digest(pep, rng, n_names=400, quoted=False):
    """A DigestResult over a synthetic peptide table: 1..3 proteins per peptide (ids ascending, a repeat allowed), random cterm / semi."""
    n = len(pep)
    counts = rng.integers(1, 4, n)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
    ids = np.concatenate([np.sort(rng.integers(0, n_names, c)) for c in counts]).astype(np.uint32)
    names = sorted({"sp|P%05d|PROT_%d" % (i, i) for i in range(n_names)})
    if quoted:
        names[3], names[7] = 'sp|Q"uote"', "tab\tname"
        names = sorted(names)
    cterm = np.where(rng.random(n) < 0.05, np.float32(0.984), np.float32(np.nan)).astype(np.float32)
    semi = (rng.random(n) < 0.1).astype(np.uint8)
    return api.DigestResult(peptides=pep, cterm=cterm, semi_enzymatic=semi, protein_offsets=off, protein_ids=ids, names=names, info={})


def spec_ids_for(n, rng):
    ids = ["controllerType=0 controllerNumber=1 scan=%d" % (i + 1) for i in range(n)]
    for i in range(0, n, 13):
        ids[i] = ["index=%d" % i, "scan=12 scan=%d" % i, "scan= scan=x%d" % i, 'we"ird\tid scan=%d' % i, "scan=007 frame=%d scan=" % i][i % 5]
    return ids


def check_rows_files(digest, rows, fdr=None, rt=None, picked=None, groups=None, generate_decoys=True, budgets=True):
    rng = np.random.default_rng(11)
    n = len(rows)
    pid = np.arange(n, dtype=np.uint64) + 1000
    files = ["a.mzML", "b file.mzML", 'c"q.mzML']
    fid = (np.arange(n) % 3).astype(np.uint32)
    ids = spec_ids_for(n, rng)
    six = rng.permutation(n).astype(np.uint32)
    kw = dict(decoy_tag="rev_", generate_decoys=generate_decoys)
    want = M.write_results(digest, rows, pid, fid, six, files, ids, fdr=fdr, rt=rt, picked=picked, groups=groups, **kw)
    got = lambda b, st: api.write_results(digest, rows, pid, fid, six, files, ids, fdr=fdr, rt=rt, picked=picked, groups=groups, text_budget=b, stats=st, **kw)
    if budgets:
        check_all_budgets(got, want)
    else:
        assert got(0, {}) == want
    want = M.write_results(digest, rows, pid, fid, six, files, ids, fdr=fdr, rt=rt, pin=True, **kw)
    got = lambda b, st: api.write_pin(digest, rows, pid, fid, six, files, ids, fdr=fdr, rt=rt, text_budget=b, stats=st, **kw)
    if budgets:
        check_all_budgets(got, want)
    else:
        assert got(0, {}) == want
    return want


@pytest.mark.parametrize("generate_decoys", [True, False])
def test_results_pin_through_every_stage(generate_decoys):
    """search (annotate_matches) -> predict_rt -> spectrum_fdr -> rows in its order -> picked_fdr -> protein_groups, then results.sage.tsv,
    results.sage.pin and matched_fragments.sage.tsv against the oracle's writer."""
    rng = np.random.default_rng(21)
    pep = synth.make_peptides(30000, seed=401, static_c=True)
    digest = fake_digest(pep, rng, quoted=True)
    spectra = synth.make_spectra(pep, 50000, seed=402)
    db = IndexedDatabase.build_from_peptides(pep)
    sc = Scorer(db, precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), annotate_matches=True)
    f, counts = sc.score_batch(spectra)
    frags = sc.last_fragments
    rows = f[counts > 0]
    fid = (rows["spectrum"] % 3).astype(np.uint32)
    rt = api.predict_rt(db, pep, rows, fid, 3)
    fd = api.spectrum_fdr(rows, Tolerance.ppm(-20, 20), aligned_rt=rt["aligned_rt"], delta_rt_model=rt["delta_rt_model"],
                          delta_ims_model=rt["delta_ims_model"])
    order = fd["order"]
    srows = rows[order]
    fd_s = {k: fd[k][order] for k in ("discriminant_score", "posterior_error", "spectrum_q")}
    rt_s = {k: rt[k][order] for k in ("aligned_rt", "predicted_rt", "delta_rt_model", "predicted_ims", "delta_ims_model")}
    picked = api.picked_fdr(pep, srows, fd_s["discriminant_score"], digest.n_proteins, digest.protein, cterm=digest.cterm, generate_decoys=generate_decoys)
    groups = api.protein_groups(pep, srows, picked["peptide_q"], fd_s["discriminant_score"], digest.protein_offsets, digest.protein_ids,
                                len(digest.names), threshold=float(np.quantile(picked["peptide_q"], 0.3)), generate_decoys=generate_decoys)
    assert len(srows) > 20000 and groups["annotated"][0] + groups["annotated"][1] > 0 and (srows["label"] == -1).any()
    check_rows_files(digest, srows, fdr=fd_s, rt=rt_s, picked=picked, groups=groups, generate_decoys=generate_decoys)
    # the reference's Feature::protein_groups strings, built by the library's host helper, appear as the results' fourth column
    res = M.write_results(digest, srows, np.arange(len(srows)), np.zeros(len(srows)), np.arange(len(srows)), ["f"],
                          ["s%d" % i for i in range(len(srows))], groups=groups, generate_decoys=generate_decoys)
    col = [rec[3] for rec in list(csv.reader(io.StringIO(res.decode(), newline=""), delimiter="\t"))[1:]]
    helper = api.protein_group_strings(groups, srows, pep, digest.protein_offsets, digest.protein_ids, digest.names, "rev_", generate_decoys)
    assert helper == col
    pid = np.arange(len(srows), dtype=np.uint64)
    assert api.write_fragments(srows, frags, pid) == M.write_fragments(pid, srows["fragment_offset"], srows["fragment_count"], frags)


def test_results_pin_adversarial_rows():
    """NaN / inf / -0.0 / subnormals in every float column, poisson -inf, Some(0.0) and -0.0 terminal mods, decoys, defaults (no stage dicts)."""
    rng = np.random.default_rng(23)
    pep = synth.make_peptides(3000, seed=403, static_c=True)
    pep.nterm[::7] = np.float32(0.0)
    pep.nterm[1::7] = np.float32(-0.0)
    pep.nterm[2::7] = np.float32(42.010565)
    pep.mods[::11] = np.float32(-0.0)
    pep.mods[3::17] = np.float32(np.nan)
    digest = fake_digest(pep, rng)
    digest.cterm[::9] = np.float32(0.0)
    n = 6000
    rows = np.zeros(n, api.FEATURE_DTYPE)
    rows["peptide_idx"] = rng.integers(0, len(pep), n)
    rows["label"] = np.where(pep.decoy[rows["peptide_idx"]] != 0, -1, 1)
    rows["charge"] = rng.integers(0, 9, n)
    rows["rank"] = rng.integers(1, 5, n)
    specials32 = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 1e-45, -1e-45, 1e13, 1e-5, 3.4e38], np.float32)
    specials64 = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 5e-324, 1e16, 1e-5, -1.0, -0.5], np.float64)
    for name in rows.dtype.names:
        kind = rows.dtype[name]
        if name in ("peptide_idx", "label", "charge", "rank", "fragment_offset", "fragment_count", "_pad0"):
            continue
        if kind == np.float32:
            v = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
            v[::2] = specials32[rng.integers(0, len(specials32), len(v[::2]))]
            rows[name] = v
        elif kind == np.float64:
            v = rng.integers(0, 1 << 64, n, dtype=np.uint64).view(np.float64)
            v[::2] = specials64[rng.integers(0, len(specials64), len(v[::2]))]
            rows[name] = v
        else:
            rows[name] = rng.integers(0, 1 << 31, n)
    rows["poisson"][::5] = -np.inf
    check_rows_files(digest, rows, generate_decoys=True)
    cols = {k: rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32) for k in
            ("discriminant_score", "posterior_error", "spectrum_q", "aligned_rt", "predicted_rt", "delta_rt_model", "predicted_ims", "delta_ims_model")}
    cols["delta_rt_model"][::3] = specials32[rng.integers(0, len(specials32), len(cols["delta_rt_model"][::3]))]
    check_rows_files(digest, rows, fdr=cols, rt=cols, picked=dict(peptide_q=cols["spectrum_q"], protein_q=cols["posterior_error"]),
                     generate_decoys=False, budgets=False)


def test_lfq_file():
    rng = np.random.default_rng(25)
    pep = synth.make_peptides(3000, seed=405, static_c=True)
    digest = fake_digest(pep, rng, quoted=True)
    n, files = 20000, ["run1.mzML", 'run "2".mzML', "run\t3.mzML"]
    quant = dict(id=rng.integers(0, len(pep), n).astype(np.uint32), charge=rng.integers(0, 5, n).astype(np.uint8),
                 decoy=rng.random(n) < 0.3, rt=rng.integers(0, 100, n).astype(np.uint32), spectral_angle=rng.random(n),
                 score=rng.standard_normal(n), areas=rng.random((n, 3)) * 1e7)
    quant["areas"][::4, 1] = 0.0
    quant["score"][::9] = np.nan
    q = rng.random(n).astype(np.float32)
    rows = np.zeros(n, api.LFQ_ROW_DTYPE)
    for k, c in (("peptide", "id"), ("charge", "charge"), ("decoy", "decoy"), ("rt", "rt"), ("spectral_angle", "spectral_angle"), ("score", "score")):
        rows[k] = quant[c]
    for gen in (True, False):
        want = M.write_lfq(digest, rows, quant["areas"], q, files, generate_decoys=gen)
        assert want.count(b"\n") == 1 + int((~quant["decoy"]).sum()) and b"\t-1\t" in want
        check_all_budgets(lambda b, st: api.write_lfq(digest, quant, q, files, generate_decoys=gen, text_budget=b, stats=st), want)
