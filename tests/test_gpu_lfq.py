"""Label-free quantification on the device (sage_b200.FeatureMap) against the CPU oracle (oracle_lfq/): the feature map and every grid cell
bit for bit; integration under the exactness contract of DESIGN.md §9 (identical presence, rt and areas wherever the oracle's acos-dependent
decisions are not near-ties; score and spectral_angle within 1e-12 relative)."""
import numpy as np
import pytest

import lfq_cases
from lfq_reference import LfqReference
from oracle_lfq import lfq_oracle as LO
from sage_b200 import FeatureMap, IndexedDatabase, LfqSettings, Ms1Batch, SageB200Error, synth
from sage_b200.api import ALIGNMENT_DTYPE

pytestmark = pytest.mark.gpu

REL = 1e-12
NEAR_TIE = 1e-9


@pytest.fixture(scope="module")
def pep():
    return lfq_cases.peptides()   # synth.make_peptides(20000, seed=41), the table of the edge workloads


@pytest.fixture(scope="module")
def db(pep):
    return IndexedDatabase.build_from_peptides(pep, device=0)


def grid_keys(fm, export, combine, charges):
    """(peptide, charge or 0, decoy) of every device grid: grids are (slot, [charge,] decoy) with slots in ascending PeptideIx."""
    slots = np.unique(export["ranges"]["peptide"])
    nch = charges[1] - charges[0] + 1
    g = np.arange(len(export["touched"]))
    sc = g // 2
    pepi = slots[sc if combine else sc // nch]
    ch = np.zeros_like(g) if combine else charges[0] + sc % nch
    return np.stack([pepi, ch, g % 2], axis=1).astype(np.uint32)


def run_both(db, pep, runs, settings, charges, splits=1):
    fm = FeatureMap.build(db, pep, settings, charges, runs["features"], runs["alignments"])
    orc = LO.LfqOracle(pep, settings, charges, runs["features"], runs["alignments"])
    b = runs["batch"]
    cuts = np.linspace(0, len(b), splits + 1).astype(int)
    for a, z in zip(cuts[:-1], cuts[1:]):
        fm.add_ms1(b.slice(a, z))
    orc.add_ms1(b)
    return fm, orc


def assert_map_and_grids_equal(fm, orc, combine, charges):
    ex = fm.export(grids=True)
    r, m = orc.export_map()
    assert ex["ranges"].tobytes() == r.tobytes(), "range arrays differ"
    assert ex["min_rts"].tobytes() == m.tobytes(), "min_rts differ"
    keys = grid_keys(fm, ex, combine, charges)
    ok, om = orc.export_grids()
    t = ex["touched"].astype(bool)
    assert keys[t].tolist() == ok.tolist(), "touched grids differ"
    assert not ex["grids"][~t].any()
    assert ex["grids"][t].tobytes() == om.tobytes(), "grid cells differ"
    return int(t.sum())


def assert_integration_matches(fm, orc, threads=8):
    d = fm.quantify()
    o = orc.quantify(threads=threads)
    okey = {k: i for i, k in enumerate(zip(o["id"].tolist(), o["charge"].tolist(), o["decoy"].tolist()))}
    seen = np.zeros(len(o["id"]), bool)
    near = 0
    for j, k in enumerate(zip(d["id"].tolist(), d["charge"].tolist(), d["decoy"].tolist())):
        i = okey[k]
        seen[i] = True
        if o["margin"][i] <= NEAR_TIE:
            near += 1
            continue
        assert o["present"][i], f"grid {k}: row on the device only"
        assert d["rt"][j] == o["rt"][i], f"grid {k}: rt {d['rt'][j]} vs {o['rt'][i]}"
        assert d["areas"][j].tobytes() == o["areas"][i].tobytes(), f"grid {k}: areas {d['areas'][j]} vs {o['areas'][i]}"
        for f in ("score", "spectral_angle"):
            assert abs(d[f][j] - o[f][i]) <= REL * max(abs(o[f][i]), 1e-300), f"grid {k}: {f} {d[f][j]!r} vs {o[f][i]!r}"
    missing = o["present"] & ~seen & (o["margin"] > NEAR_TIE)
    assert not missing.any(), f"{int(missing.sum())} oracle rows missing on the device"
    assert np.all(np.diff(np.stack([d["id"], d["charge"], d["decoy"]], 1).astype(np.int64) @ np.array([1 << 20, 1 << 2, 1])) > 0)
    return len(d["id"]), near


@pytest.mark.parametrize("combine", [True, False])
@pytest.mark.parametrize("mobility", [False, True])
def test_grids_bit_exact_across_batch_splits(db, pep, combine, mobility):
    runs = synth.make_ms1_runs(pep, n_ids=1500, n_files=3, spectra_per_file=200, peaks_per_spectrum=300, seed=7 + mobility, mobility=mobility)
    settings = LfqSettings(combine_charge_states=combine)
    charges = (2, 4)
    ref = None
    for splits in (1, 3, 37):
        fm, orc = run_both(db, pep, runs, settings, charges, splits)
        n = assert_map_and_grids_equal(fm, orc, combine, charges)
        assert n > 1000
        g = fm.export(grids=True)["grids"]
        if ref is None:
            ref = g
        assert g.tobytes() == ref.tobytes()
    rows, near = assert_integration_matches(fm, orc)
    assert rows > 500
    print(f"combine={combine} mobility={mobility}: {n} grids, {rows} rows, {near} near-tie grids not compared")


def test_wide_ppm_tolerance_keeps_the_mass_window(db, pep):
    # 3000 ppm is wider than the +-0.1 binary-search window for every m/z above ~33: entries outside the window are not visited
    runs = synth.make_ms1_runs(pep, n_ids=1500, n_files=2, spectra_per_file=200, peaks_per_spectrum=300, seed=11)
    settings = LfqSettings(ppm_tolerance=3000.0)
    fm, orc = run_both(db, pep, runs, settings, (2, 3), splits=2)
    assert assert_map_and_grids_equal(fm, orc, True, (2, 3)) > 1000
    assert_integration_matches(fm, orc)


@pytest.mark.parametrize("scoring", ["RetentionTime", "SpectralAngle", "Intensity", "Hybrid"])
@pytest.mark.parametrize("integration", ["Apex", "Sum"])
@pytest.mark.parametrize("threshold", [0.7, 0.0])
def test_integration_strategies(db, pep, scoring, integration, threshold):
    runs = synth.make_ms1_runs(pep, n_ids=1200, n_files=3, spectra_per_file=250, peaks_per_spectrum=300, seed=13, absent_fraction=0.4)
    settings = LfqSettings(peak_scoring=scoring, integration=integration, spectral_angle=threshold)
    fm, orc = run_both(db, pep, runs, settings, (2, 3), splits=2)
    assert_map_and_grids_equal(fm, orc, True, (2, 3))
    rows, near = assert_integration_matches(fm, orc)
    assert rows > 300 and near < rows // 10
    print(f"{scoring}/{integration}/{threshold}: {rows} rows, {near} near-tie grids not compared")


def _single_peptide(pep, rt=0.5):
    i = int(np.nonzero(pep.decoy == 0)[0][100])
    feats = dict(peptide_idx=np.array([i], np.uint32), peptide_q=np.zeros(1, np.float32), label=np.ones(1, np.int32), aligned_rt=np.array([rt], np.float32),
                 calcmass=pep.mono[[i]], file_id=np.array([1], np.uint32), ims=np.zeros(1, np.float32))
    align = np.zeros(3, ALIGNMENT_DTYPE)
    align["max_rt"], align["slope"], align["intercept"] = 1.0, 1.0, 0.0
    return i, feats, align


def test_zero_intensity_touch_creates_a_row_and_far_spectra_are_skipped(db, pep):
    i, feats, align = _single_peptide(pep)
    mz = np.float32(pep.mono[i] / np.float32(2))
    b = Ms1Batch(np.array([0, 1, 2, 3], np.uint64), np.array([mz, mz, 100.0], np.float32), np.array([0.0, 0.0, 5.0], np.float32),
                 np.array([0, 0, 2], np.uint32), np.array([0.5, 0.501, 7.0], np.float32))   # the last spectrum lies outside every page
    settings = LfqSettings(peak_scoring="Intensity", spectral_angle=0.0)
    fm = FeatureMap.build(db, pep, settings, (2, 2), feats, align)
    orc = LO.LfqOracle(pep, settings, (2, 2), feats, align)
    fm.add_ms1(b)
    orc.add_ms1(b)
    assert fm.info()["contributions"] == 4
    assert assert_map_and_grids_equal(fm, orc, True, (2, 2)) == 1
    rows, _ = assert_integration_matches(fm, orc)
    d = fm.quantify()
    assert rows == 1 and d["id"].tolist() == [i] and not d["decoy"][0] and d["score"][0] > 0 and not d["areas"].any()


def test_error_codes(db, pep):
    i, feats, align = _single_peptide(pep)
    bad = dict(feats, file_id=np.array([3], np.uint32))
    with pytest.raises(SageB200Error) as e:
        FeatureMap.build(db, pep, LfqSettings(), (2, 3), bad, align)
    assert e.value.code == -1 and "file_id" in e.value.message
    fm = FeatureMap.build(db, pep, LfqSettings(), (2, 3), feats, align)
    b = Ms1Batch(np.array([0, 1], np.uint64), np.array([500.0], np.float32), np.ones(1, np.float32), np.array([3], np.uint32), np.zeros(1, np.float32))
    with pytest.raises(SageB200Error) as e:
        fm.add_ms1(b)
    assert e.value.code == -1 and "file_id" in e.value.message
    # every peptide of the table (~18800) x 10 charges x 2 x 128 files x 300 f64 = 115 GB of grids: refused before allocating
    n = len(pep)
    f = dict(peptide_idx=np.arange(n, dtype=np.uint32), peptide_q=np.zeros(n, np.float32), label=np.ones(n, np.int32),
             aligned_rt=np.full(n, 0.5, np.float32), calcmass=pep.mono, file_id=np.zeros(n, np.uint32), ims=np.zeros(n, np.float32))
    align = np.zeros(128, ALIGNMENT_DTYPE)
    align["max_rt"] = 1.0
    with pytest.raises(SageB200Error) as e:
        FeatureMap.build(db, pep, LfqSettings(combine_charge_states=False), (1, 10), f, align)
    assert e.value.code == -5 and "bytes" in e.value.message


def test_bench_sized_workload(db, pep):
    pep_big = synth.make_peptides(120000, seed=43)
    dbb = IndexedDatabase.build_from_peptides(pep_big, device=0)
    runs = synth.make_ms1_runs(pep_big, n_ids=30000, n_files=4, spectra_per_file=3000, peaks_per_spectrum=1500, seed=17)
    fm, orc = run_both(dbb, pep_big, runs, LfqSettings(), (2, 4), splits=4)
    n = assert_map_and_grids_equal(fm, orc, True, (2, 4))
    rows, near = assert_integration_matches(fm, orc, threads=16)
    assert n > 30000 and rows > 20000
    print(f"bench-sized: {n} grids, {rows} rows, {near} near-tie grids not compared")


# ---------------------------------------------------------------------------------------------------- edge workloads (tests/lfq_cases.py)
def _build_case(db, c):
    fm = FeatureMap.build(db, c["peptides"], c["settings"], c["charges"], c["features"], c["alignments"])
    orc = LO.LfqOracle(c["peptides"], c["settings"], c["charges"], c["features"], c["alignments"])
    return fm, orc


@pytest.mark.parametrize("name", lfq_cases.NAMES)
def test_edge_workloads(db, name):
    """Device against the oracle on every edge workload, and against the restatement without the oracle: the contribution count (two per
    add_entry), the touched set; and quantify twice gives identical bytes."""
    c = lfq_cases.case(name)
    combine = c["settings"].combine_charge_states
    fm, orc = _build_case(db, c)
    ref = LfqReference(c["peptides"], c["settings"], c["charges"], c["features"], c["alignments"])
    for b in c["batches"]:
        fm.add_ms1(b)
        orc.add_ms1(b)
        ref.add_ms1(b)
    n = assert_map_and_grids_equal(fm, orc, combine, c["charges"])
    assert fm.info()["contributions"] == 2 * ref.matches
    ex = fm.export(grids=True)
    assert grid_keys(fm, ex, combine, c["charges"])[ex["touched"].astype(bool)].tolist() == ref.export_grids()[0].tolist()
    rows, near = assert_integration_matches(fm, orc)
    a, b = fm.quantify(), fm.quantify()
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), f"second quantify differs in {k}"
    if name != "no_kept_feature":
        assert rows > 0
    print(f"{name}: {n} grids compared, {rows} rows, {near} near-tie grids not compared")


def test_add_ms1_after_quantify(db):
    """Tracing more spectra after quantify adds to the same grids: the result equals the oracle fed every batch before integrating."""
    c = lfq_cases.case("files9")
    fm, orc = _build_case(db, c)
    b = c["batches"][0]
    half = len(b) // 2
    fm.add_ms1(b.slice(0, half))
    fm.quantify()
    fm.add_ms1(b.slice(half, len(b)))
    orc.add_ms1(b)
    assert assert_map_and_grids_equal(fm, orc, True, c["charges"]) > 100
    assert_integration_matches(fm, orc)


def test_big_batch_equals_small_calls(db):
    """One add_ms1 of 2^24 + 2^20 peaks (two tracing passes) gives the grids of the same spectra fed in calls of at most 2^22 peaks."""
    c = lfq_cases.case("big_batch")
    b = c["batches"][0]
    fm_big, _ = _build_case(db, dict(c, batches=[]))
    fm_big.add_ms1(b)
    fm_small = FeatureMap.build(db, c["peptides"], c["settings"], c["charges"], c["features"], c["alignments"])
    off = b.peak_off.astype(np.int64)
    a = 0
    calls = 0
    while a < len(b):
        z = int(np.searchsorted(off, off[a] + (1 << 22), side="right")) - 1
        z = max(z, a + 1)
        fm_small.add_ms1(b.slice(a, z))
        a = z
        calls += 1
    assert calls >= 5
    g1, g2 = fm_big.export(grids=True), fm_small.export(grids=True)
    assert g1["touched"].tobytes() == g2["touched"].tobytes() and g1["touched"].any()
    assert g1["grids"].tobytes() == g2["grids"].tobytes()
    assert fm_big.info()["contributions"] == fm_small.info()["contributions"]
