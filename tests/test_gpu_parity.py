"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs."""
import os

import numpy as np
import pytest

import sage_b200
from sage_b200 import IndexedDatabase, Precursor, ProcessedSpectrum, Scorer, SpectraBatch, Tolerance, synth
from oracle import oracle as O

from helpers import assert_features_equal, f64_exact_default, oracle_cfg, oracle_db_from_peptides, peptides_from_oracle, valid_rows

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def small():
    pep = synth.make_peptides(20000, seed=11, static_c=True)
    odb = oracle_db_from_peptides(pep)
    gdb = IndexedDatabase.build_from_peptides(pep)
    spectra = synth.make_spectra(pep, 1500, seed=12)
    return pep, odb, gdb, spectra


def run_both(odb, gdb, spectra, pep_caps=(2048, 0), **kw):
    """Scores with the CUDA path under each preliminary-scoring strategy — peptide-centric counting for small windows (pep_cap > 0), probing
    the small-block copy of the index (pep_cap 0, narrow_index 1: the default), probing the page index in the reference's loop order
    (narrow_index 0; last, so that the returned scorer's counters are the reference's work terms) — and requires each to equal the oracle."""
    of, oc, _, octr = odb.score_batch(oracle_cfg(**kw), spectra.as_dict(), counters=True)
    modes = [(cap, 1) for cap in pep_caps] + [(0, 0)]
    for cap, narrow_index in modes:
        sc = Scorer(gdb, **kw)
        if cap is not None:
            sc.set_option("pep_cap", cap)
        sc.set_option("narrow_index", narrow_index)
        gf, gc = sc.score_batch(spectra)
        n = assert_features_equal(gf, gc, of, oc, kw.get("report_psms", 1),
                                  what=str({"pep_cap": cap, "narrow_index": narrow_index, **{k: v for k, v in kw.items() if "tol" not in k}}),
                                  f64_exact=f64_exact_default(kw.get("score_type", 0)))
    return sc, n, octr


def test_index_build_matches_oracle(small):
    pep, odb, gdb, _ = small
    fp, fm, bm = gdb.export_index()
    e = odb.export()
    assert np.array_equal(bm.view(np.uint32), e["bucket_min"].view(np.uint32))
    assert np.array_equal(fp, e["frag_pep"])
    assert np.array_equal(fm.view(np.uint32), e["frag_mz"].view(np.uint32))


def test_reference_layout_upload_roundtrip(small):
    pep, odb, _, spectra = small
    e = odb.export()
    gdb2 = IndexedDatabase.from_reference_layout(pep, e["frag_pep"], e["frag_mz"], e["bucket_min"], e["bucket_size"])
    fp, fm, bm = gdb2.export_index()
    assert np.array_equal(fp, e["frag_pep"]) and np.array_equal(fm.view(np.uint32), e["frag_mz"].view(np.uint32))
    run_both(odb, gdb2, spectra.slice(0, 300), precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20))


def test_config1_known_answer(config1):
    # crates/sage-cli/tests/integration.rs: psm.len()==1, matched_peaks==21, through the C ABI
    odb = O.OracleDB.from_fasta(config1["fasta"])
    pep = peptides_from_oracle(odb)
    gdb = IndexedDatabase.build_from_peptides(pep)
    masses, intens, tic = O.process_ms2(config1["mz"], config1["intensity"], config1["precursor_charge"], 100, True, 0.0)
    spec = ProcessedSpectrum(level=2, id=config1["spectrum_id"], scan_start_time=config1["scan_start_time_min"],
                             precursors=[Precursor(mz=config1["precursor_mz"], charge=config1["precursor_charge"],
                                                   isolation_window=Tolerance.da(*config1["isolation_window_da"]))],
                             masses=masses, intensities=intens, total_ion_current=float(tic))
    scorer = Scorer(gdb, precursor_tol=Tolerance.ppm(-50.0, 50.0), fragment_tol=Tolerance.ppm(-10.0, 10.0), min_matched_peaks=4, min_isotope_err=-1,
                    max_isotope_err=3, min_precursor_charge=2, max_precursor_charge=4, override_precursor_charge=False, max_fragment_charge=1,
                    chimera=False, report_psms=1, wide_window=False, annotate_matches=False, score_type=0)
    psm = scorer.score(spec)
    assert len(psm) == 1
    assert psm[0]["matched_peaks"] == 21
    assert pep.sequence(int(psm[0]["peptide_idx"])) == "LQSRPAAPPAPGPGQLTLR"
    assert abs(psm[0]["hyperscore"] - 69.90865222) < 1e-6
    assert psm[0]["rt"] == np.float32(config1["scan_start_time_min"])


def test_narrow_search(small):
    pep, odb, gdb, spectra = small
    sc, n, octr = run_both(odb, gdb, spectra, precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20))
    assert n > 1000
    c = sc.counters()  # last run: pep_cap = 0, i.e. the reference's loop order -> identical work counters
    for k in ("queries", "pages", "entries_scanned", "candidates_scored", "psms"):
        assert c[k] == octr[k], (k, c[k], octr[k])
    assert c["peptide_record_floats"] == octr["peptide_record_floats"] and c["pep_queries"] == 0
    sc2 = Scorer(gdb, precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20))
    sc2.set_option("pep_cap", 8192)
    sc2.score_batch(spectra)
    c2 = sc2.counters()
    assert c2["pep_queries"] == c2["queries"] and c2["pep_fallbacks"] == 0 and c2["matched_fragments"] == c["matched_fragments"]


def test_narrow_block_index_block_sizes(small):
    """The small-block copy of the index with blocks of 64 .. 8192 peptides (windows inside one block, straddling two, spanning many) and the page
    index give the same rows and the same matched-fragment / candidate counts."""
    pep, odb, gdb, spectra = small
    kw = dict(precursor_tol=Tolerance.ppm(-50, 50), fragment_tol=Tolerance.ppm(-20, 20), report_psms=3, min_isotope_err=-1, max_isotope_err=2)
    ref = Scorer(gdb, **kw)
    ref.set_option("narrow_index", 0)
    rf, rc = ref.score_batch(spectra)
    rf, rc, rctr = valid_rows(rf, rc, 3).copy(), rc.copy(), ref.counters()
    assert rc.sum() > 500 and rctr["pages"] > 0
    for block in (64, 300, 1024, 8192):
        sc = Scorer(gdb, **kw)
        sc.set_option("narrow_block", block)
        f, c = sc.score_batch(spectra)
        ctr = sc.counters()
        assert np.array_equal(c, rc) and valid_rows(f, c, 3).tobytes() == rf.tobytes(), block
        assert ctr["matched_fragments"] == rctr["matched_fragments"] and ctr["candidates_scored"] == rctr["candidates_scored"] and ctr["pages"] == 0, block


def test_split_scoring_equals_fused(small):
    """k_score<true> -> k_fold -> k_features (default for non-chimeric scoring) against the fused kernel: same rows, same counters; also with a hit
    arena that is too small at first (the chunk is re-run with the exact size)."""
    pep, odb, gdb, spectra = small
    for kw in (dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20)),
               dict(precursor_tol=Tolerance.ppm(-50, 50), fragment_tol=Tolerance.ppm(-20, 20), report_psms=5, min_isotope_err=-1, max_isotope_err=2, min_matched_peaks=1),
               dict(precursor_tol=Tolerance.da(-2, 2), fragment_tol=Tolerance.da(-0.02, 0.02), report_psms=3, max_fragment_charge=1, score_type=1),
               dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), report_psms=64, min_matched_peaks=2)):
        r = kw.get("report_psms", 1)
        fused = Scorer(gdb, **kw)
        fused.set_option("score_split", 0)
        ff, fc = fused.score_batch(spectra)
        ff, fc, fctr = valid_rows(ff, fc, r).copy(), fc.copy(), fused.counters()
        assert fc.sum() > 100
        for fast, reset in ((1, 0), (0, 0), (1, 1)):
            sc = Scorer(gdb, **kw)
            sc.set_option("score_fast", fast)
            if reset:
                sc.set_option("worklist_reset", 1)
            f, c = sc.score_batch(spectra)
            ctr = sc.counters()
            assert np.array_equal(c, fc) and valid_rows(f, c, r).tobytes() == ff.tobytes(), (kw, fast, reset)
            for k in ("psms", "candidates_scored", "peptide_record_floats", "matched_fragments"):
                assert ctr[k] == fctr[k], (k, ctr[k], fctr[k])
            if reset:
                assert ctr["chunk_retries"] >= 1


def test_narrow_report5_fragcharge1(small):
    pep, odb, gdb, spectra = small
    run_both(odb, gdb, spectra, precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), report_psms=5, max_fragment_charge=1,
             min_matched_peaks=2)


def test_isotope_errors(small):
    pep, odb, gdb, spectra = small
    run_both(odb, gdb, spectra, precursor_tol=Tolerance.ppm(-50, 50), fragment_tol=Tolerance.ppm(-10, 10), min_isotope_err=-1, max_isotope_err=3,
             report_psms=2)


def test_isotope_min_eq_max_nonzero(small):
    # scoring.rs:391-415: min == max (even non-zero) searches isotope 0 only
    pep, odb, gdb, spectra = small
    run_both(odb, gdb, spectra.slice(0, 400), precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), min_isotope_err=1, max_isotope_err=1)


def test_unknown_charge_and_override(small):
    pep, odb, gdb, spectra = small
    unk = SpectraBatch(**{**spectra.__dict__, "prec_charge": np.where(np.arange(len(spectra)) % 3 == 0, 0, spectra.prec_charge).astype(np.uint8)})
    run_both(odb, gdb, unk, precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), report_psms=3)
    run_both(odb, gdb, spectra.slice(0, 500), precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), override_precursor_charge=True,
             min_precursor_charge=1, max_precursor_charge=4)


def test_wide_window(small):
    pep, odb, gdb, spectra = small
    n = len(spectra)
    iso_lo = np.where(np.arange(n) % 2 == 0, np.float32(-1.5), np.float32(np.nan)).astype(np.float32)
    iso_hi = np.where(np.arange(n) % 2 == 0, np.float32(1.5), np.float32(np.nan)).astype(np.float32)
    ww = SpectraBatch(**{**spectra.__dict__, "iso_lo": iso_lo, "iso_hi": iso_hi})
    run_both(odb, gdb, ww.slice(0, 600), precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), wide_window=True, report_psms=2,
             min_precursor_charge=2, max_precursor_charge=3)


def test_open_search_wide_path(small):
    pep, odb, gdb, spectra = small
    sc, n, _ = run_both(odb, gdb, spectra.slice(0, 400), precursor_tol=Tolerance.da(-500, 500), fragment_tol=Tolerance.ppm(-20, 20), report_psms=2)
    assert sc.counters()["wide_queries"] > 100  # exercised the streaming kernel
    run_both(odb, gdb, spectra.slice(400, 600), precursor_tol=Tolerance.da(-500, 100), fragment_tol=Tolerance.ppm(-20, 20), min_isotope_err=-1,
             max_isotope_err=1)


def test_open_search_multi_tile(small):
    # the wide kernel walks the window in shared-memory tiles; small tiles force several tiles per query on this small database
    pep, odb, gdb, spectra = small
    kw = dict(precursor_tol=Tolerance.da(-800, 800), fragment_tol=Tolerance.ppm(-20, 20), report_psms=3)
    sub = spectra.slice(0, 200)
    of, oc, _, octr = odb.score_batch(oracle_cfg(**kw), sub.as_dict(), counters=True)
    # both counting strategies of k_prelim_wide: the block-major m/z-sorted index copy (default) and page-slice streaming (the reference's loop)
    for tile, pages_mode in ((1024, False), (4096, False), (32768, False), (512, False), (1024, True), (32768, True)):
        os.environ["SAGE_B200_NO_WIDE_INDEX"] = "1" if pages_mode else "0"
        try:
            sc = Scorer(gdb, **kw)
            sc.set_option("wide_tile", tile)
            gf, gc = sc.score_batch(sub)
        finally:
            os.environ.pop("SAGE_B200_NO_WIDE_INDEX", None)
        assert_features_equal(gf, gc, of, oc, 3, what=f"wide_tile={tile} pages_mode={pages_mode}")
        c = sc.counters()
        if c["wide_queries"] == c["queries"]:   # the reference-terms work counters are the oracle's in both modes
            assert c["pages"] == octr["pages"] and c["entries_scanned"] == octr["entries_scanned"], (tile, pages_mode, c["pages"], octr["pages"])
    # survivor-list overflow at various points -> the counting CTA replays and continues serially
    for lmax, tile in ((128, 1024), (200, 4096), (600, 2048), (3000, 1024)):
        sc = Scorer(gdb, **kw)
        sc.set_option("wide_tile", tile)
        sc.set_option("wide_lmax", lmax)
        gf, gc = sc.score_batch(sub)
        assert_features_equal(gf, gc, of, oc, 3, what=f"wide_lmax={lmax} wide_tile={tile}")
        assert lmax > 1000 or sc.counters()["wide_overflows"] > 0
    kw = dict(precursor_tol=Tolerance.da(-800, 800), fragment_tol=Tolerance.da(-1.5, 1.5), min_isotope_err=-1, max_isotope_err=1)  # many pages per probe
    of, oc, _, _ = odb.score_batch(oracle_cfg(**kw), sub.slice(0, 40).as_dict())
    sc = Scorer(gdb, **kw)
    sc.set_option("wide_tile", 2048)
    gf, gc = sc.score_batch(sub.slice(0, 40))
    assert_features_equal(gf, gc, of, oc, 1, what="wide, Da fragment tolerance")


def test_open_search_arena_budget_forces_smaller_chunks(small):
    # ADVICE r1: the survivor-list arena (96 KiB per open-search query and lane) is bounded by a budget; a first chunk that would need more is
    # not re-run at its size (that used to end in a hard cudaMalloc failure for very large batches) — the call restarts with smaller chunks
    pep, odb, gdb, spectra = small
    kw = dict(precursor_tol=Tolerance.da(-500, 500), fragment_tol=Tolerance.ppm(-20, 20), min_isotope_err=-1, max_isotope_err=1, report_psms=2)
    sub = spectra.slice(0, 400)
    of, oc, _, _ = odb.score_batch(oracle_cfg(**kw), sub.as_dict())
    os.environ["SAGE_B200_WIDE_ARENA_MB"] = "16"   # 170 lists: 400 spectra x 3 isotope queries do not fit one chunk
    try:
        sc = Scorer(gdb, **kw)
        gf, gc = sc.score_batch(sub)
        c = sc.counters()
        g2, c2 = sc.score_batch(sub)   # second call: chunk size already learned, no restart
    finally:
        os.environ.pop("SAGE_B200_WIDE_ARENA_MB", None)
    assert_features_equal(gf, gc, of, oc, 2, what="arena budget, first call")
    assert_features_equal(g2, c2, of, oc, 2, what="arena budget, second call")
    assert c["chunk_retries"] > 0 and c["wide_queries"] > 300


def test_chimera(small):
    pep, odb, gdb, _ = small
    chim = synth.make_spectra(pep, 800, seed=13, chimeric=True)
    run_both(odb, gdb, chim, precursor_tol=Tolerance.da(-1.5, 1.5), fragment_tol=Tolerance.ppm(-20, 20), chimera=True, report_psms=5)
    run_both(odb, gdb, chim.slice(0, 200), precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), chimera=True, report_psms=2)


def test_tolerance_kinds_and_openms_score(small):
    pep, odb, gdb, spectra = small
    run_both(odb, gdb, spectra.slice(0, 400), precursor_tol=Tolerance.pct(-0.01, 0.01), fragment_tol=Tolerance.da(-0.02, 0.02), score_type=1)


def test_annotate_matches_fragments(small):
    # Fragments of every reported PSM (scoring.rs:738-751), standard and chimera paths
    pep, odb, gdb, spectra = small
    for kw, sub in ((dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), report_psms=3, annotate_matches=True), spectra.slice(0, 500)),
                    (dict(precursor_tol=Tolerance.da(-1.5, 1.5), fragment_tol=Tolerance.ppm(-20, 20), chimera=True, report_psms=3, annotate_matches=True,
                          max_fragment_charge=2), synth.make_spectra(pep, 300, seed=14, chimeric=True))):
        sc = Scorer(gdb, **kw)
        gf, gc = sc.score_batch(sub)
        gfr = sc.last_fragments
        of, oc, ofr, _ = odb.score_batch(oracle_cfg(**kw), sub.as_dict())
        n = assert_features_equal(gf, gc, of, oc, 3, what="annotate")
        sel = (np.arange(len(gf)) % 3) < np.repeat(gc, 3)
        g, o = gf[sel], of[sel]
        assert n > 100 and len(gfr) == len(ofr) == int(g["fragment_count"].sum())
        for a, b_ in zip(g, o):
            assert a["fragment_count"] == b_["frag_count"] == a["matched_peaks"]
            x = gfr[a["fragment_offset"]:a["fragment_offset"] + a["fragment_count"]]
            y = ofr[b_["frag_offset"]:b_["frag_offset"] + b_["frag_count"]]
            for f in ("kind", "charge", "ordinal"):
                assert np.array_equal(x[f], y[f]), f
            for f in ("intensity", "mz_calculated", "mz_experimental"):
                assert np.array_equal(x[f].view(np.uint32), y[f].view(np.uint32)), f
    # capacity too small -> ELIMIT with the required size reported, features still complete
    sc = Scorer(gdb, precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), annotate_matches=True)
    sc.fragment_capacity = 16
    with pytest.raises(sage_b200.SageB200Error) as e:
        sc.score_batch(spectra.slice(0, 100))
    assert e.value.code == -5 and "fragment_capacity" in e.value.message


def test_score_batch_multi_single_process(small):
    # one process driving every visible GPU (falls back to two scorers on one device when only one GPU is visible)
    from sage_b200.api import score_batch_multi
    pep, odb, gdb, spectra = small
    kw = dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), report_psms=2)
    ndev = max(1, sage_b200.device_count())
    dbs = [gdb] + [IndexedDatabase.build_from_peptides(pep, device=d) for d in range(1, ndev)]
    scorers = [Scorer(dbs[d % ndev], **kw) for d in range(max(2, ndev))] + [Scorer(gdb, **kw)]   # odd count: uneven blocks
    gf, gc = score_batch_multi(scorers, spectra)
    of, oc, _, _ = odb.score_batch(oracle_cfg(**kw), spectra.as_dict())
    assert_features_equal(gf, gc, of, oc, 2, what=f"score_batch_multi over {len(scorers)} scorers / {ndev} device(s)")


def test_scorers_on_one_db_in_two_threads(small):
    """A narrow and an open-search scorer on one fresh db, each scoring from its own thread: both lazily build their block-index copy of the
    fragments while the other scorer's kernels run. Rows, counts and work counters equal the same searches run one after the other on
    another fresh db, and the oracle's rows."""
    import threading
    from sage_b200.api import COUNTER_U64
    pep, odb, _, spectra = small
    kws = (dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), report_psms=2),
           dict(precursor_tol=Tolerance.da(-500, 500), fragment_tol=Tolerance.ppm(-20, 20), report_psms=2))
    subs = (spectra, spectra.slice(0, 400))

    def search(db, kw, sub):
        sc = Scorer(db, **kw)
        f, c = sc.score_batch(sub)
        return f, c, {k: v for k, v in sc.counters().items() if k in COUNTER_U64}

    seq_db = IndexedDatabase.build_from_peptides(pep)
    seq = [search(seq_db, kw, sub) for kw, sub in zip(kws, subs)]
    par_db = IndexedDatabase.build_from_peptides(pep)
    par, errors = [None, None], []

    def run(i):
        try:
            par[i] = search(par_db, kws[i], subs[i])
        except Exception as e:   # re-raised in the main thread
            errors.append(e)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for (pf, pc, pctr), (sf, sc_, sctr), kw, sub in zip(par, seq, kws, subs):
        assert np.array_equal(pc, sc_)
        pv, sv = valid_rows(pf, pc, 2), valid_rows(sf, sc_, 2)
        for f in pv.dtype.names:
            if not f.startswith("_"):
                assert np.array_equal(np.ascontiguousarray(pv[f]).view(np.uint8), np.ascontiguousarray(sv[f]).view(np.uint8)), f
        assert pctr == sctr
        of, oc, _, _ = odb.score_batch(oracle_cfg(**kw), sub.as_dict())
        assert_features_equal(pf, pc, of, oc, 2, what="two threads, one db")
    assert seq[1][2]["wide_queries"] > 100
    assert par_db.device_bytes() == seq_db.device_bytes()


def test_quick_score_prefilter(small):
    # Scorer::quick_score (scoring.rs:255-298): both branches, incl. isotope fold and unknown charges
    pep, odb, gdb, spectra = small
    sub = SpectraBatch(**{**spectra.slice(0, 600).__dict__, "prec_charge": np.where(np.arange(600) % 4 == 0, 0, spectra.prec_charge[:600]).astype(np.uint8)})
    for kw in (dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), report_psms=1),
               dict(precursor_tol=Tolerance.da(-3, 3), fragment_tol=Tolerance.ppm(-10, 10), min_isotope_err=-1, max_isotope_err=2, report_psms=3,
                    min_matched_peaks=3)):
        sc = Scorer(gdb, **kw)
        for low in (False, True):
            g = sc.quick_score(sub, low)
            o = odb.quick_score(oracle_cfg(**kw), sub.as_dict(), low)
            assert g.sum() > 100 and np.array_equal(g, o), (kw, low, int(g.sum()), int(o.sum()))
        # OR semantics
        k0 = np.zeros(len(pep), np.uint8)
        k0[:10] = 1
        assert np.array_equal(sc.quick_score(sub, True, k0)[:10], np.ones(10, np.uint8))


def test_quick_score_fresh_scorer_rerun_leaves_no_stale_marks(small):
    # ADVICE r1: a chunk whose work lists overflow is re-run with exact sizes; keep[] is OR-accumulated, so the partial hit sets of the
    # overflowed attempt must not leave marks behind. Fresh scorers start with an empty open-search work list (wide_cap = 0) and a tiny
    # narrow arena, so the first chunk of each of these calls is re-run; with charge / isotope folds a partial set changes the final trim.
    pep, odb, gdb, spectra = small
    sub = SpectraBatch(**{**spectra.slice(0, 300).__dict__, "prec_charge": np.where(np.arange(300) % 3 == 0, 0, spectra.prec_charge[:300]).astype(np.uint8)})
    for kw, reset in ((dict(precursor_tol=Tolerance.da(-500, 500), fragment_tol=Tolerance.ppm(-20, 20), min_isotope_err=-1, max_isotope_err=1, report_psms=2), None),
                      (dict(precursor_tol=Tolerance.da(-30, 30), fragment_tol=Tolerance.ppm(-20, 20), min_isotope_err=-1, max_isotope_err=2, report_psms=1), 0)):
        for low in (False, True):
            sc = Scorer(gdb, **kw)   # fresh: nothing learned yet
            if reset is not None:
                sc.set_option("worklist_reset", reset)
            g = sc.quick_score(sub, low)
            assert sc.counters()["chunk_retries"] > 0
            o = odb.quick_score(oracle_cfg(**kw), sub.as_dict(), low)
            assert g.sum() > 100 and np.array_equal(g, o), (kw, low, int(g.sum()), int(o.sum()), int((g != o).sum()))


def test_initial_hits_heap_order(small):
    # white box: the preliminary list must come back in the reference's bounded_min_heapify order
    pep, odb, gdb, spectra = small
    kw = dict(precursor_tol=Tolerance.da(-30, 30), fragment_tol=Tolerance.ppm(-20, 20), min_isotope_err=-1, max_isotope_err=2)
    sc = Scorer(gdb, **kw)
    for i in (0, 7, 19, 123):
        one = spectra.slice(i, i + 1)
        g = sc.initial_hits(one)
        o = odb.initial_hits(oracle_cfg(**kw), one.masses, one.intensities, float(one.prec_mz[0]), int(one.prec_charge[0]))
        for k in ("matched", "peptide", "charge", "iso"):
            assert np.array_equal(g[k], o[k]), (i, k)
        assert g["matched_peaks"] == o["matched_peaks"] and g["scored_candidates"] == o["scored_candidates"]


def test_edge_cases(small):
    pep, odb, gdb, spectra = small
    # ragged spectra: empty, 1 peak, precursor far outside the peptide mass range, duplicate masses
    specs = [
        ProcessedSpectrum(precursors=[Precursor(mz=500.0, charge=2)]),
        ProcessedSpectrum(precursors=[Precursor(mz=800.0, charge=2)], masses=np.float32([500.0]), intensities=np.float32([10.0]), total_ion_current=10.0),
        ProcessedSpectrum(precursors=[Precursor(mz=90000.0, charge=3)], masses=np.float32([100, 200, 300]), intensities=np.float32([1, 2, 3]), total_ion_current=6.0),
        ProcessedSpectrum(precursors=[Precursor(mz=1.0, charge=1)], masses=np.float32([100, 200, 300]), intensities=np.float32([1, 2, 3]), total_ion_current=6.0),
    ]
    one = spectra.slice(3, 4)
    m = np.repeat(one.masses, 2)
    specs.append(ProcessedSpectrum(precursors=[Precursor(mz=float(one.prec_mz[0]), charge=int(one.prec_charge[0]))], masses=m,
                                   intensities=np.repeat(one.intensities, 2), total_ion_current=float(one.tic[0]) * 2))
    batch = SpectraBatch.from_spectra(specs)
    run_both(odb, gdb, batch, precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), report_psms=2)
    run_both(odb, gdb, batch, precursor_tol=Tolerance.da(-500, 500), fragment_tol=Tolerance.ppm(-20, 20), min_isotope_err=-1, max_isotope_err=1, chimera=True,
             report_psms=2)


def test_unsorted_peaks_fall_back_to_index_path(small):
    # the reference never assumes sorted peaks in the preliminary pass; the peptide-centric path does, so it must detect and fall back
    pep, odb, gdb, spectra = small
    sub = spectra.slice(0, 64)
    rng = np.random.default_rng(5)
    m = sub.masses.reshape(64, 200).copy()
    it = sub.intensities.reshape(64, 200).copy()
    for r in range(0, 64, 2):
        perm = rng.permutation(200)
        m[r], it[r] = m[r][perm], it[r][perm]
    shuffled = SpectraBatch(**{**sub.__dict__, "masses": m.ravel(), "intensities": it.ravel()})
    kw = dict(precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), min_matched_peaks=1)
    run_both(odb, gdb, shuffled, pep_caps=(2048,), **kw)
    sc = Scorer(gdb, **kw)
    sc.set_option("pep_cap", 2048)
    sc.score_batch(shuffled)
    assert sc.counters()["pep_fallbacks"] == 32


def test_reference_panics_become_errors(small):
    pep, odb, gdb, spectra = small
    sc = Scorer(gdb, precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20))
    with pytest.raises(sage_b200.SageB200Error) as e:
        sc.score(ProcessedSpectrum(level=1, precursors=[Precursor(mz=500.0, charge=2)]))
    assert e.value.code == -3 and "non-MS2" in e.value.message
    with pytest.raises(sage_b200.SageB200Error) as e:
        sc.score(ProcessedSpectrum(level=2, precursors=[]))
    assert e.value.code == -4 and "missing MS1 precursor" in e.value.message


def test_small_bucket_sizes():
    # bucket sizes down to 1 (the reference's quickcheck range) through both index paths
    pep = synth.make_peptides(3000, seed=21)
    spectra = synth.make_spectra(pep, 200, seed=22)
    for bs in (1, 2, 64, 1024):
        odb = oracle_db_from_peptides(pep, bucket_size=bs)
        gdb = IndexedDatabase.build_from_peptides(pep, bucket_size=bs)
        run_both(odb, gdb, spectra, precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20))
        run_both(odb, gdb, spectra.slice(0, 50), precursor_tol=Tolerance.da(-2000, 2000), fragment_tol=Tolerance.da(-0.5, 0.5))


def test_worklist_undersized_chunk_is_rerun(small):
    """Device work lists (narrow key-list arena, open-search item list) are sized from earlier chunks with no host round trip inside a
    chunk; a chunk that needs more is re-run with the exact sizes it counted. Results must not depend on that."""
    pep, odb, gdb, spectra = small
    sub = spectra.slice(0, 400)
    for kw in (dict(precursor_tol=Tolerance.da(-30.0, 30.0), fragment_tol=Tolerance.ppm(-20, 20)),        # narrow windows > k: arena in use
               dict(precursor_tol=Tolerance.da(-800.0, 800.0), fragment_tol=Tolerance.ppm(-20, 20))):      # open search: wide item list
        of, oc, _, _ = odb.score_batch(oracle_cfg(**kw), sub.as_dict())
        sc = Scorer(gdb, **kw)
        sc.set_option("worklist_reset", 0)
        gf, gc = sc.score_batch(sub)
        assert sc.counters()["chunk_retries"] >= 1
        assert_features_equal(gf, gc, of, oc, 1, what="first batch (undersized work lists)")
        gf, gc = sc.score_batch(sub)
        assert sc.counters()["chunk_retries"] == 0   # sizes learned
        assert_features_equal(gf, gc, of, oc, 1, what="second batch (learned sizes)")
