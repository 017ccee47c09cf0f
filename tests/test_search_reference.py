"""The numpy restatement of the search-and-score path (tests/search_reference.py) against the C++ oracle, bit for bit, on every edge
workload of tests/search_cases.py and on random index shapes; and against the reference's own known answers and 200-bit arithmetic.
The two CPU authorities share no code, so a misreading of the Rust in one of them fails here before any device comparison."""
import ctypes
import ctypes.util

import numpy as np
import pytest

from oracle import oracle as O
from sage_b200 import Tolerance, synth

import search_cases as SC
import search_reference as R
from helpers import oracle_cfg, oracle_db_from_peptides, peptides_from_oracle

f32 = np.float32


def _oracle(pep, db_kw, sp, cfg, counters=True):
    odb = oracle_db_from_peptides(pep, **db_kw)
    return odb, odb.score_batch(oracle_cfg(**cfg), sp.as_dict(), counters=counters)


@pytest.mark.parametrize("name", [f.__name__ for f in SC.WORKLOADS])
def test_restatement_equals_oracle(name):
    pep, db_kw, sp, cfg = SC.BY_NAME[name]()
    odb, (of, oc, _, octr) = _oracle(pep, db_kw, sp, cfg)
    rf, rc, _, rctr = SC.restated(pep, db_kw, sp, cfg, counters=True)
    n = SC.assert_rows_bits_equal(rf, rc, of, oc, cfg.get("report_psms", 1), name)
    assert (rctr["pages"], rctr["entries_scanned"]) == (octr["pages"], octr["entries_scanned"])
    if name in SC.COUNTED:
        print(f"{name}: {n} rows compared")
        assert n > 0


@pytest.mark.parametrize("name", ["isobaric_isomers", "isotope_defaults_r5", "equal_intensities", "odd_peaks", "ion_index_zero_two_charges",
                                  "peptide_lengths", "fragment_charges_1_to_8", "duplicate_peaks"])
def test_restatement_equals_oracle_fragments_and_chimera(name):
    """annotate_matches fragments (kind, charge, ordinal, intensity, calculated and experimental m/z), then the chimera loop."""
    pep, db_kw, sp, cfg = SC.BY_NAME[name]()
    for extra in (dict(annotate_matches=True), dict(chimera=True, report_psms=max(3, cfg.get("report_psms", 1)))):
        c = dict(cfg, **extra)
        _, (of, oc, ofr, _) = _oracle(pep, db_kw, sp, c, counters=False)
        rf, rc, rfr, _ = SC.restated(pep, db_kw, sp, c)
        SC.assert_rows_bits_equal(rf, rc, of, oc, c["report_psms"], f"{name} {extra}")
        if c.get("annotate_matches"):
            SC.assert_fragments_equal(rf, rc, rfr, of, oc, ofr, c["report_psms"], name)


@pytest.mark.parametrize("name", ["isobaric_isomers", "isotope_defaults_r64", "two_charges_unknown", "asymmetric_da", "overflow_warp"])
@pytest.mark.parametrize("low_memory", [False, True])
def test_quick_score_equals_oracle(name, low_memory):
    """Both branches of quick_score; the low-memory heap compares Score by its derived PartialOrd (peptide first)."""
    pep, db_kw, sp, cfg = SC.BY_NAME[name]()
    odb = oracle_db_from_peptides(pep, **db_kw)
    want = odb.quick_score(oracle_cfg(**cfg), sp.as_dict(), low_memory)
    got = R.quick_score_batch(R.build_from_peptides(pep, **db_kw), cfg, sp, low_memory)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("name", ["isotope_defaults_r1", "isotope_defaults_r64", "two_charges_unknown", "window_bounds", "overflow_warp",
                                  "overflow_narrow"])
def test_initial_hits_order_equals_oracle(name):
    """The trimmed preliminary list in heap order, with matched_peaks and scored_candidates, spectrum by spectrum."""
    pep, db_kw, sp, cfg = SC.BY_NAME[name]()
    odb = oracle_db_from_peptides(pep, **db_kw)
    db = R.build_from_peptides(pep, **db_kw)
    d = sp.as_dict()
    for i in range(min(len(sp), 12)):
        one = sp.slice(i, i + 1)
        h = R.initial_hits_one(db, cfg, one)
        o = odb.initial_hits(oracle_cfg(**cfg), d["masses"][int(d["peak_off"][i]):int(d["peak_off"][i + 1])],
                             d["intensities"][int(d["peak_off"][i]):int(d["peak_off"][i + 1])], float(one.prec_mz[0]), int(one.prec_charge[0]),
                             float(one.iso_lo[0]), float(one.iso_hi[0]))
        got = [(m, p, c, e) for (m, p, c, e) in h.preliminary]
        want = list(zip(o["matched"].tolist(), o["peptide"].tolist(), o["charge"].tolist(), o["iso"].tolist()))
        assert got == want, f"{name} spectrum {i}"
        assert (h.matched_peaks, h.scored_candidates) == (o["matched_peaks"], o["scored_candidates"])


def test_overflow_workloads_wrap():
    """The overflow workloads really pass 2^16 on one (query, peptide) pair whose slot is even, and its odd neighbour matches too:
    the wrapped count, the second `scored_candidates` increment and the neighbour's own count are what the rows must show."""
    for name in ("overflow_warp", "overflow_narrow"):
        pep, db_kw, sp, cfg = SC.BY_NAME[name]()
        db = R.build_from_peptides(pep, **db_kw)
        s = R.spectra_from_batch(sp)[0]
        q = R.db_query(db, (s.prec_mz - R.PROTON) * f32(2), R.Tol.of(cfg["precursor_tol"]), R.Tol.of(cfg["fragment_tol"]))
        _, peps = R.page_search_counts(db, q, s.masses)
        total = np.bincount(peps - q.pre_idx_lo, minlength=q.pre_idx_hi - q.pre_idx_lo + 1)
        big = int(np.argmax(total))
        assert total[big] > 65536 and big % 2 == 0 and total[big + 1] > 0, name
        h = R.Scorer(db, **cfg).initial_hits(s)
        assert h.scored_candidates == int((total > 0).sum()) + 1
        assert (total[big] & 0xFFFF, q.pre_idx_lo + big) in [(m, p) for (m, p, _, _) in h.preliminary]


@pytest.mark.parametrize("seed", range(12))
def test_random_configuration_restatement_equals_oracle(seed):
    """Random index shapes (ion kinds a/b/c/x/y/z, bucket sizes 16..32768, min_ion_index 0..3) and Scorer settings, in the style of
    test_gpu_random.py, including one-sided fragment windows."""
    rng = np.random.default_rng(9100 + seed)
    pep = synth.make_peptides(int(rng.choice([400, 1500])), seed=300 + seed, static_c=bool(rng.integers(2)), var_mod_m=bool(rng.integers(2)))
    kinds = [("b", "y"), ("a", "b", "y"), ("c", "z"), ("y",), ("b", "x", "y"), ("a", "c", "x", "z")][seed % 6]
    db_kw = dict(bucket_size=[16, 256, 4096, 8192, 32768, 64][seed % 6], ion_kinds=kinds, min_ion_index=seed % 4)
    sp = synth.make_spectra(pep, 40, seed=int(rng.integers(1 << 30)), n_peaks=int(rng.choice([30, 90])), charge_known=bool(rng.integers(2)))
    frag = [Tolerance.ppm(-20, 20), Tolerance.da(0.0, 0.03), Tolerance.ppm(-40, -5), Tolerance.pct(-0.002, 0.001)][seed % 4]
    cfg = dict(precursor_tol=[Tolerance.ppm(-20, 20), Tolerance.da(-2, 0.5), Tolerance.ppm(0, 50)][seed % 3], fragment_tol=frag,
               min_matched_peaks=int(rng.choice([0, 1, 4])), min_isotope_err=int(rng.choice([0, -1])), max_isotope_err=int(rng.choice([0, 2])),
               min_precursor_charge=2, max_precursor_charge=int(rng.choice([3, 4])), max_fragment_charge=[None, 1, 2][seed % 3],
               report_psms=int(rng.choice([1, 3, 7])), wide_window=seed % 5 == 4, chimera=seed % 6 == 5, score_type=seed % 2)
    _, (of, oc, _, octr) = _oracle(pep, db_kw, sp, cfg)
    rf, rc, _, rctr = SC.restated(pep, db_kw, sp, cfg, counters=True)
    SC.assert_rows_bits_equal(rf, rc, of, oc, cfg["report_psms"], f"seed {seed}")
    assert (rctr["pages"], rctr["entries_scanned"]) == (octr["pages"], octr["entries_scanned"])


@pytest.mark.parametrize("name,db_kw", [("isobaric_isomers", dict(bucket_size=8192, ion_kinds=("b", "y"), min_ion_index=2)),
                                        ("peptide_lengths", dict(bucket_size=16, ion_kinds=("a", "b", "c", "x", "y", "z"), min_ion_index=0)),
                                        ("window_bounds", dict(bucket_size=100, ion_kinds=("y",), min_ion_index=3))])
def test_index_equals_oracle_export(name, db_kw):
    """build_from_peptides: frag_pep, frag_mz and bucket_min equal the oracle's export() (the device's export_index() is compared on the GPU)."""
    pep = SC.BY_NAME[name]()[0]
    e = oracle_db_from_peptides(pep, **db_kw).export()
    db = R.build_from_peptides(pep, **db_kw)
    assert np.array_equal(db.frag_pep, e["frag_pep"])
    assert np.array_equal(db.frag_mz.view(np.uint32), e["frag_mz"].view(np.uint32))
    assert np.array_equal(db.bucket_min.view(np.uint32), e["bucket_min"].view(np.uint32))


def test_next_power_of_two():
    # database.rs:97: Builder::make_parameters rounds the bucket size up
    assert [R.next_power_of_two(n) for n in (1, 2, 3, 1000, 8192, 8193)] == [1, 2, 4, 1024, 8192, 16384]


# ------------------------------------------------------------------------------------------------ the reference's own known answers
def _config1_spectrum(config1, top_n):
    masses, intens, tic = O.process_ms2(config1["mz"], config1["intensity"], config1["precursor_charge"], top_n, True, 0.0)
    return dict(peak_off=np.array([0, len(masses)], np.uint64), masses=masses, intensities=intens, prec_mz=f32([config1["precursor_mz"]]),
                prec_charge=np.array([config1["precursor_charge"]], np.uint8), iso_lo=f32([config1["isolation_window_da"][0]]),
                iso_hi=f32([config1["isolation_window_da"][1]]), tic=f32([tic]), level=None, ims=None)


def test_config1_matched_peaks_21(config1):
    # crates/sage-cli/tests/integration.rs:7-52; the peptide table is the oracle's digest (digestion is not restated)
    odb = O.OracleDB.from_fasta(config1["fasta"])
    db = R.build_from_peptides(peptides_from_oracle(odb), bucket_size=odb.bucket_size)
    cfg = dict(precursor_tol=(R.PPM, -50.0, 50.0), fragment_tol=(R.PPM, -10.0, 10.0), min_matched_peaks=4, min_isotope_err=-1, max_isotope_err=3,
               min_precursor_charge=2, max_precursor_charge=4, max_fragment_charge=1, report_psms=1)
    rows, _, _ = R.score_batch(db, cfg, _config1_spectrum(config1, 100))
    assert len(rows[0]) == 1
    r = rows[0][0]
    assert r["matched_peaks"] == 21 and odb.sequence(r["peptide_idx"]) == "LQSRPAAPPAPGPGQLTLR"
    assert abs(r["hyperscore"] - 69.90865222) < 1e-6


def test_config1_tests_config_json(config1):
    odb = O.OracleDB.from_fasta(config1["fasta"], bucket_size=16384, missed_cleavages=1, static_mods={"C": 57.0216})
    db = R.build_from_peptides(peptides_from_oracle(odb), bucket_size=odb.bucket_size)
    cfg = dict(precursor_tol=(R.PPM, -50.0, 50.0), fragment_tol=(R.PPM, -10.0, 10.0), min_isotope_err=-1, max_isotope_err=3, max_fragment_charge=1,
               report_psms=1)
    rows, _, _ = R.score_batch(db, cfg, _config1_spectrum(config1, 150))
    r = rows[0][0]
    assert r["matched_peaks"] == 22 and odb.sequence(r["peptide_idx"]) == "LQSRPAAPPAPGPGQLTLR"
    assert abs(r["hyperscore"] - 72.26591574) < 1e-6


@pytest.mark.parametrize("seed", range(10))
def test_check_all_ions_visited(seed):
    """crates/sage/tests/integration.rs:30-70 on the restated index: page_search visits every fragment in the window."""
    rng = np.random.default_rng(2000 + seed)
    pep = synth.make_peptides(600, seed=seed)
    bs = R.next_power_of_two(int(rng.integers(1, 8193)))
    db = R.build_from_peptides(pep, bucket_size=bs)
    target = f32(rng.uniform(0, 3000))
    q = R.db_query(db, f32(1000.0), R.Tol(R.DA, f32(-5000.0), f32(5000.0)), R.Tol(R.DA, f32(-100.0), f32(100.0)))
    _, peps = R.page_search_counts(db, q, np.array([target], np.float32))
    flo, fhi = R.Tol(R.DA, f32(-100.0), f32(100.0)).bounds(target)
    sel = (db.frag_mz >= flo) & (db.frag_mz <= fhi)
    assert np.array_equal(np.bincount(peps, minlength=db.n_peptides), np.bincount(db.frag_pep[sel], minlength=db.n_peptides))


@pytest.mark.parametrize("seed", range(20))
def test_heap_quickcheck(seed):
    # heap.rs:62-100: the k largest in min-heap order
    rng = np.random.default_rng(seed)
    data = rng.integers(-50, 50, int(rng.integers(0, 300))).tolist()
    k = min(int(rng.integers(0, 80)), len(data))
    want = sorted(data, reverse=True)[:k]
    got = list(data)
    R.bounded_min_heapify(got, k)
    assert R.check_heap(got[:k]) or k == len(data)
    assert sorted(got[:k], reverse=True) == want
    assert O.bounded_min_heapify(np.array(data, np.int32), k)[:k].tolist() == got[:k]


def test_run_and_max_fragment_charge_tables():
    # scoring.rs:799-830
    run = R.Run()
    for i in (1, 2, 3, 3, 3):
        run.matched(i)
    assert (run.length, run.longest) == (3, 3)
    run.matched(5)
    run.matched(5)
    assert (run.length, run.longest) == (1, 3)
    run.matched(6)
    assert run.length == 2
    zero = R.Run()
    zero.matched(0)
    assert zero.longest == 0   # `last` starts at 0: ion index 0 never starts a ladder
    table = [(None, 1, 2), (None, 2, 2), (None, 3, 3), (None, 4, 4), (1, 2, 2), (1, 3, 2), (2, 4, 3), (4, 1, 2)]
    for opt, z, want in table:
        assert R.max_fragment_charge(opt, z) == want == O.max_fragment_charge(opt, z)


# ------------------------------------------------------------------------------------------------ 200-bit arithmetic
def test_scores_against_high_precision_arithmetic():
    """hyperscore, lnfact and poisson of the restatement against mpmath from the same f32 / integer inputs.

    hyperscore: ln (< 1 ulp), four libm logs inside the two lnfact terms and three f64 additions: <= 8 ulp of the result, the bound
    test_hyperscore_against_high_precision_arithmetic derives for the oracle. lnfact: its terms cancel, so its error is bounded
    relative to its largest term n ln n: <= 8 ulp of that. poisson = (k ln(lambda) - lambda - lnfact(k)) / ln 10: the error of
    k ln(lambda) (1 ulp of ln, 0.5 of the product), of lnfact(k) (the bound above), two subtractions and the division (0.5 ulp each)
    are each at most a few ulp of the largest intermediate term T = max(|k ln lambda|, lambda, k ln k); the bound is 16 ulp of T / ln 10."""
    mpmath = pytest.importorskip("mpmath")
    mpmath.mp.prec = 200
    log1pf = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6").log1pf
    log1pf.restype, log1pf.argtypes = ctypes.c_float, [ctypes.c_float]
    rng = np.random.default_rng(0x5C0F)

    def x_lnfact(n):
        if n == 0:
            return mpmath.mpf(1)
        x = mpmath.mpf(n)
        return x * mpmath.log(x) - x + mpmath.mpf(0.5) * mpmath.log(x) + mpmath.mpf(0.5) * mpmath.log(mpmath.pi * 2 * x)

    ulp = lambda v: float(np.spacing(np.float64(abs(float(v)))))  # noqa: E731
    for _ in range(3000):
        mb, my = int(rng.integers(0, 80)), int(rng.integers(0, 80))
        sb, sy = f32(rng.uniform(0, 5e6)), f32(rng.uniform(0, 5e6))
        want = mpmath.log(mpmath.mpf(float(sb + f32(1.0))) * mpmath.mpf(float(sy + f32(1.0)))) + x_lnfact(mb) + x_lnfact(my)
        got = R.score_type_score(0, mb, my, sb, sy)
        assert abs(float(mpmath.mpf(got) - want)) <= 8 * ulp(want)
        want1 = mpmath.mpf(float(log1pf(ctypes.c_float(sb + sy)))) + x_lnfact(mb) + x_lnfact(my)
        assert abs(float(mpmath.mpf(R.score_type_score(1, mb, my, sb, sy)) - want1)) <= 8 * ulp(want1)
    for n in (1, 2, 3, 10, 59, 255, 1000, 65535):
        assert abs(R.lnfact(n) - float(x_lnfact(n))) <= 8 * np.spacing(np.float64(max(n * np.log(max(n, 2)), 1.0))), n
    ln10 = mpmath.log(10)
    for _ in range(3000):
        k = int(rng.integers(0, 200))
        mp_, scd = int(rng.integers(1, 10**6)), int(rng.integers(1, 5000))
        lam = mp_ / scd
        got = (float(k) * R.ln(lam) - lam - R.lnfact(k)) / R.LN_10
        L = mpmath.mpf(lam)   # lambda itself is the f64 quotient the reference computes
        want = (k * mpmath.log(L) - L - x_lnfact(k)) / ln10
        T = max(abs(k * float(mpmath.log(L))), lam, k * np.log(max(k, 2)), 1.0)
        assert abs(float(mpmath.mpf(got) - want)) <= 16 * ulp(T / 2.302585092994046), (k, lam)


def test_non_finite_hyperscore_is_255():
    big = f32(3.0e38)
    assert R.score_type_score(0, 3, 3, big + big, f32(1.0)) == 255.0     # (summed + 1) overflows to +inf
    assert R.score_type_score(1, 3, 3, big, big) == 255.0                # ln_1p(+inf)
    assert R.score_type_score(0, 3, 3, big, big) != 255.0                # each sum + 1 is finite and so is their f64 product
