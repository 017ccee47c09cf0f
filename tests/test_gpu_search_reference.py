"""The device search-and-score path against BOTH CPU authorities, the numpy restatement (tests/search_reference.py) and the C++
oracle, on every edge workload of tests/search_cases.py, under every counting and scoring strategy the library can take: the
small-block copy of the index and the page index (narrow_index), the peptide-centric path (pep_cap), fused and split scoring
(score_split), the straight-line and generic task bodies (score_fast), the open-search block index and page streaming
(SAGE_B200_NO_WIDE_INDEX), and block / tile sizes placed on the workloads' window bounds. Integer, f32 and f64 fields bit for bit."""
import os

import numpy as np
import pytest

from sage_b200 import IndexedDatabase, Scorer, api

import search_cases as SC
import search_reference as R
from helpers import assert_features_equal, f64_exact_default, oracle_cfg, oracle_db_from_peptides

pytestmark = pytest.mark.gpu

STRATEGIES = [dict(), dict(narrow_index=0), dict(pep_cap=8192), dict(score_split=0), dict(score_split=1, score_fast=0), dict(score_split=0, score_fast=0)]
EXTRA = {"block_boundaries": [dict(narrow_block=256), dict(narrow_block=256, narrow_index=0)],
         "block_boundaries_wide": [dict(wide_tile=4096), dict(wide_tile=4096, score_split=0)],
         "window_8193": [dict(wide_tile=4096)]}

def _device(db, cfg, sp, opts):
    sc = Scorer(db, **cfg)
    for k, v in opts.items():
        sc.set_option(k, v)
    return sc.score_batch(sp)


def _compare_all(name, pep, db_kw, sp, cfg, no_wide=False):
    rf, rc, _, _ = SC.restated(pep, db_kw, sp, cfg)
    odb = oracle_db_from_peptides(pep, **db_kw)
    of, oc, _, _ = odb.score_batch(oracle_cfg(**cfg), sp.as_dict())
    k = cfg.get("report_psms", 1)
    n = SC.assert_rows_bits_equal(rf, rc, of, oc, k, f"{name}: restatement vs oracle")
    old = os.environ.get("SAGE_B200_NO_WIDE_INDEX")
    if no_wide:
        os.environ["SAGE_B200_NO_WIDE_INDEX"] = "1"
    try:
        db = IndexedDatabase.build_from_peptides(pep, **db_kw)
        fp, fm, bm = db.export_index()
        e = odb.export()
        assert np.array_equal(fp, e["frag_pep"]) and np.array_equal(fm.view(np.uint32), e["frag_mz"].view(np.uint32))
        assert np.array_equal(bm.view(np.uint32), e["bucket_min"].view(np.uint32))
        exact = f64_exact_default(cfg.get("score_type", 0))
        for opts in STRATEGIES + EXTRA.get(name, []):
            gf, gc = _device(db, cfg, sp, opts)
            what = f"{name} {opts} no_wide={no_wide}"
            # integer and f32 fields always bit for bit; the f64 scores too where the device reproduces this host's libm log (helpers.py)
            SC.assert_rows_bits_equal(gf, gc, rf, rc, k, what + ": device vs restatement", f64=exact)
            SC.assert_rows_bits_equal(gf, gc, of, oc, k, what + ": device vs oracle", f64=exact)
            if not exact:
                assert_features_equal(gf, gc, of, oc, k, what=what, f64_exact=False)
    finally:
        if no_wide:
            if old is None:
                os.environ.pop("SAGE_B200_NO_WIDE_INDEX", None)
            else:
                os.environ["SAGE_B200_NO_WIDE_INDEX"] = old
    return n


@pytest.mark.parametrize("name", [f.__name__ for f in SC.WORKLOADS])
def test_device_equals_restatement_and_oracle(name):
    pep, db_kw, sp, cfg = SC.BY_NAME[name]()
    n = _compare_all(name, pep, db_kw, sp, cfg)
    print(f"{name}: {n} rows compared")
    if name in SC.COUNTED:
        assert n > 0


@pytest.mark.parametrize("name", ["overflow_warp", "overflow_narrow"])
@pytest.mark.parametrize("opts", [dict(), dict(narrow_index=0), dict(pep_cap=8192)])
def test_u16_count_wraps_like_the_reference(name, opts):
    """k_prelim_exact: a (query, peptide) count past 2^16 on an even slot wraps as the reference's u16 PreScore::matched does, without
    carrying into its matching odd neighbour, and scored_candidates counts the wrapped slot again (scoring.rs:363-372). Before the exact
    path, the packed u16 pair carried the overflow into the neighbour's count. Checked on the trimmed preliminary list in heap order
    (matched, PeptideIx, charge, isotope) and on the rows, under the index, page-index and peptide-centric counting paths."""
    pep, db_kw, sp, cfg = SC.BY_NAME[name]()
    db = R.build_from_peptides(pep, **db_kw)
    h = R.initial_hits_one(db, cfg, sp)
    gdb = IndexedDatabase.build_from_peptides(pep, **db_kw)
    sc = Scorer(gdb, **cfg)
    for k, v in opts.items():
        sc.set_option(k, v)
    g = sc.initial_hits(sp)
    got = list(zip(g["matched"].tolist(), g["peptide"].tolist(), g["charge"].tolist(), g["iso"].tolist()))
    assert got == [tuple(x) for x in h.preliminary]
    assert (g["matched_peaks"], g["scored_candidates"]) == (h.matched_peaks, h.scored_candidates)
    assert h.matched_peaks > 0x10000
    rf, rc, _, _ = SC.restated(pep, db_kw, sp, cfg)
    gf, gc = _device(gdb, cfg, sp, opts)
    n = SC.assert_rows_bits_equal(gf, gc, rf, rc, cfg["report_psms"], f"{name} {opts}", f64=f64_exact_default())
    print(f"{name} {opts}: {n} rows compared")
    assert n > 0


@pytest.mark.parametrize("name", ["window_8193", "block_boundaries_wide", "negative_fragment_mz", "two_charges_unknown"])
def test_device_equals_restatement_page_streaming(name):
    """Open-search windows counted by streaming page slices as the reference does (SAGE_B200_NO_WIDE_INDEX=1)."""
    pep, db_kw, sp, cfg = SC.BY_NAME[name]()
    _compare_all(name, pep, db_kw, sp, cfg, no_wide=True)


@pytest.mark.parametrize("name", ["isobaric_isomers", "equal_intensities", "ion_index_zero_two_charges", "odd_peaks", "peptide_lengths",
                                  "fragment_charges_1_to_8", "fmax_intensity_sage", "duplicate_peaks"])
def test_device_fragments_and_chimera(name):
    """annotate_matches fragments and the chimera loop (remove_matched_peaks, TIC re-sum, the first round's hits reused)."""
    pep, db_kw, sp, cfg = SC.BY_NAME[name]()
    db = IndexedDatabase.build_from_peptides(pep, **db_kw)
    odb = oracle_db_from_peptides(pep, **db_kw)
    for extra in (dict(annotate_matches=True), dict(chimera=True, report_psms=max(3, cfg.get("report_psms", 1)))):
        c = dict(cfg, **extra)
        rf, rc, rfr, _ = SC.restated(pep, db_kw, sp, c)
        of, oc, ofr, _ = odb.score_batch(oracle_cfg(**c), sp.as_dict())
        sc = Scorer(db, **c)
        gf, gc = sc.score_batch(sp)
        SC.assert_rows_bits_equal(gf, gc, rf, rc, c["report_psms"], f"{name} {extra}: device vs restatement")
        SC.assert_rows_bits_equal(gf, gc, of, oc, c["report_psms"], f"{name} {extra}: device vs oracle")
        if c.get("annotate_matches"):
            SC.assert_fragments_equal(gf, gc, sc.last_fragments, rf, rc, rfr, c["report_psms"], name)


@pytest.mark.parametrize("name", ["isobaric_isomers", "isotope_defaults_r64", "two_charges_unknown", "asymmetric_da", "window_bounds"])
@pytest.mark.parametrize("low_memory", [False, True])
def test_device_quick_score(name, low_memory):
    pep, db_kw, sp, cfg = SC.BY_NAME[name]()
    want = R.quick_score_batch(R.build_from_peptides(pep, **db_kw), cfg, sp, low_memory)
    assert np.array_equal(want, oracle_db_from_peptides(pep, **db_kw).quick_score(oracle_cfg(**cfg), sp.as_dict(), low_memory))
    got = Scorer(IndexedDatabase.build_from_peptides(pep, **db_kw), **cfg).quick_score(sp, low_memory)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("name", ["isotope_defaults_r1", "isotope_defaults_r5", "two_charges_unknown", "window_bounds", "window_1025"])
def test_device_initial_hits_order(name):
    """The trimmed preliminary list in heap order (the white-box hook), with matched_peaks and scored_candidates."""
    pep, db_kw, sp, cfg = SC.BY_NAME[name]()
    db = R.build_from_peptides(pep, **db_kw)
    sc = Scorer(IndexedDatabase.build_from_peptides(pep, **db_kw), **cfg)
    for i in range(min(len(sp), 10)):
        one = sp.slice(i, i + 1)
        h = R.initial_hits_one(db, cfg, one)
        g = sc.initial_hits(one)
        got = list(zip(g["matched"].tolist(), g["peptide"].tolist(), g["charge"].tolist(), g["iso"].tolist()))
        assert got == [tuple(x) for x in h.preliminary], f"{name} spectrum {i}"
        assert (g["matched_peaks"], g["scored_candidates"]) == (h.matched_peaks, h.scored_candidates)


def _elimit(fn, needle):
    with pytest.raises(api.SageB200Error) as e:
        fn()
    assert e.value.code == -5 and needle in str(e.value), str(e.value)


def test_limits_and_one_past():
    """report_psms 64, an isotope range of 32 and a charge range of 16 are accepted (their rows are compared above); one past each is
    ELIMIT with its message."""
    pep, db_kw, sp, cfg = SC.report_psms_64()
    db = IndexedDatabase.build_from_peptides(pep, **db_kw)
    _elimit(lambda: Scorer(db, **dict(cfg, report_psms=65)), "report_psms 65 > 64")
    _elimit(lambda: Scorer(db, **dict(cfg, min_isotope_err=-16, max_isotope_err=16)), "isotope range > 32")
    _elimit(lambda: Scorer(db, **dict(cfg, min_precursor_charge=1, max_precursor_charge=17)), "charge range > 16")


def test_largest_peak_count():
    """The largest spectrum k_score's shared-memory budget accepts is scored like the CPU authorities; one more peak is ELIMIT with the
    message (the staged peak copies are 16-byte granular, so the largest accepted count is a multiple of four)."""
    pep, db_kw, sp, cfg = SC.many_peaks(8)
    db = IndexedDatabase.build_from_peptides(pep, **db_kw)

    def ok(n):
        try:
            _device(db, cfg, SC.many_peaks(n)[2], {})
            return True
        except api.SageB200Error as e:
            assert e.code == -5 and "exceeds the shared-memory budget" in str(e), str(e)
            return False

    lo, hi = 8, 1 << 16
    assert ok(lo) and not ok(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if ok(mid) else (lo, mid)
    print(f"largest accepted peak count: {lo}")
    assert lo % 4 == 0
    pep, db_kw, sp, cfg = SC.many_peaks(lo)
    n = _compare_all(f"many_peaks({lo})", pep, db_kw, sp, cfg)
    assert n > 0
    _elimit(lambda: _device(db, cfg, SC.many_peaks(lo + 1)[2], {}), "exceeds the shared-memory budget")
