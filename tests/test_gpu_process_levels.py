"""SpectrumProcessor::process for every MS level on the device (sage_b200_process_raw, FeatureMap.add_raw_ms1, tmt_quantify) against the CPU
oracle (oracle_process/, which takes level 2 from oracle/'s process_ms2). Every comparison is bit for bit: offsets, masses, intensities,
mobilities (NaN where a spectrum has none), TIC, and for LFQ every grid cell and quantify row."""
import numpy as np
import pytest

import lfq_cases
from oracle import oracle as O
from oracle_lfq import lfq_oracle as LO
from oracle_process import process_oracle as PO
from sage_b200 import FeatureMap, IndexedDatabase, LfqSettings, Ms1Batch, RawSpectra, SageB200Error, SpectrumProcessor, Tolerance, api, synth
from test_gpu_lfq import assert_integration_matches, assert_map_and_grids_equal

pytestmark = pytest.mark.gpu

RAW_SMEM_PEAKS = 4096   # spectra.cuh: the largest unsorted spectrum sorted in shared memory
ELIMIT = -5


def bits(x):
    return np.atleast_1d(np.asarray(x, np.float32)).view(np.uint32)


def assert_same(got, want, what=""):
    assert got.peak_off.tolist() == want["peak_off"].tolist(), f"{what}: offsets"
    for k, g in (("masses", got.masses), ("intensities", got.intensities), ("mobilities", got.mobilities), ("tic", got.tic)):
        gb, wb = bits(g), bits(want[k])
        if not np.array_equal(gb, wb):
            i = int(np.nonzero(gb != wb)[0][0])
            raise AssertionError(f"{what}: {k} differ first at {i}: {gb[i]:08x} vs {wb[i]:08x}")
    assert got.has_mobilities.tolist() == want["has_mobilities"].tolist(), f"{what}: has_mobilities"
    assert got.level.tolist() == want["level"].tolist()


def run(raw, take_top_n=150, deisotope=False, min_deisotope_mz=0.0, what=""):
    got = SpectrumProcessor(take_top_n, deisotope, min_deisotope_mz).process_raw(raw)
    assert_same(got, PO.so_process(raw, take_top_n, deisotope, min_deisotope_mz), what)
    return got


def concat(parts):
    """One RawSpectra of several (mobility kept only when every part has it)."""
    off = [np.zeros(1, np.uint64)]
    total = 0
    for p in parts:
        off.append((np.asarray(p.peak_off[1:], np.uint64) - np.uint64(p.peak_off[0]) + np.uint64(total)))
        total += int(p.peak_off[-1] - p.peak_off[0])
    mob = None if any(p.mobility is None for p in parts) else np.concatenate([p.mobility for p in parts])
    chg = np.concatenate([np.zeros(len(p), np.uint8) if p.precursor_charge is None else p.precursor_charge for p in parts])
    return RawSpectra(np.concatenate(off), np.concatenate([p.mz for p in parts]), np.concatenate([p.intensity for p in parts]),
                      np.concatenate([p.level for p in parts]), chg, mob)


def spectrum(mz, it, level, mob=None, charge=0):
    mz, it = np.asarray(mz, np.float32), np.asarray(it, np.float32)
    return RawSpectra(np.array([0, len(mz)], np.uint64), mz, it, np.uint8([level]), np.uint8([charge]),
                      None if mob is None else np.asarray(mob, np.float32))


@pytest.mark.parametrize("mobility", [False, True])
@pytest.mark.parametrize("order", ["sorted", "reversed", "shuffled"])
def test_mixed_levels(order, mobility):
    raw = synth.make_raw_spectra(600, peaks=(0, 700), levels=(0, 1, 2, 3, 4), order=order, mobility=mobility, seed=11)
    run(raw, what=f"{order} mob={mobility}")
    run(raw, take_top_n=40, deisotope=True, min_deisotope_mz=131.0, what=f"{order} mob={mobility} deisotoped")


def test_level2_rows_equal_process_spectra():
    raw = synth.make_raw_spectra(400, peaks=(0, 500), levels=(1, 2, 3), order="sorted", seed=12)
    for kw in (dict(take_top_n=150, deisotope=False, min_deisotope_mz=0.0), dict(take_top_n=60, deisotope=True, min_deisotope_mz=0.0)):
        sp = SpectrumProcessor(kw["take_top_n"], kw["deisotope"], kw["min_deisotope_mz"])
        got = sp.process_raw(raw)
        rows = np.nonzero(raw.level == 2)[0]
        sub = concat([raw.slice(int(r), int(r) + 1) for r in rows])
        off, m, i, tic = sp.process_batch(sub.peak_off, sub.mz, sub.intensity, sub.precursor_charge)
        for j, r in enumerate(rows):
            a, b = int(got.peak_off[r]), int(got.peak_off[r + 1])
            c, d = int(off[j]), int(off[j + 1])
            assert bits(got.masses[a:b]).tolist() == bits(m[c:d]).tolist() and bits(got.intensities[a:b]).tolist() == bits(i[c:d]).tolist()
            assert bits(got.tic[r]).tolist() == bits(tic[j]).tolist()
            assert np.isnan(got.mobilities[a:b]).all()


def test_ms2_past_budget_is_elimit():
    big = spectrum(np.linspace(100.0, 2000.0, 10_000), np.ones(10_000), 2, charge=2)
    raw = concat([synth.make_raw_spectra(5, levels=(1, 3), seed=13), big])
    with pytest.raises(SageB200Error) as e:
        SpectrumProcessor(150, False, 0.0).process_raw(raw)
    assert e.value.code == ELIMIT
    # the same size at level 1 and 3 has no limit
    run(concat([spectrum(big.mz[::-1], big.intensity, 1), spectrum(big.mz[::-1], big.intensity, 3)]), what="10k peaks, levels 1 and 3")


def _f32(u):
    return np.array(u, np.uint32).view(np.float32)


@pytest.mark.parametrize("mobility", [False, True])
def test_special_values(mobility):
    nan_mz = _f32([0x7FC00000, 0xFFC00000, 0x7F812345, 0xFF800001, 0x7FA00000, 0xFFFFFFFF])
    mz = np.concatenate([nan_mz, np.float32([np.inf, -np.inf, -5.0, 0.0, -0.0, 1.0072764, 100.0, 100.0, 2.0, 1e30])])
    it = np.concatenate([_f32([0x7FC00001, 0xFF812345]), np.float32([np.inf, -np.inf, -1.0, 0.0, -0.0, 3.0, 7.0, 7.0]), np.arange(6, dtype=np.float32)])
    rng = np.random.default_rng(14)
    parts = []
    for level in (0, 1, 3, 4):
        for k in range(6):
            p = rng.permutation(len(mz))
            q = rng.permutation(len(it))
            n = len(mz) - k
            parts.append(spectrum(mz[p][:n], it[q][:n], level, rng.uniform(0.6, 1.4, n) if mobility else None))
        parts.append(spectrum(np.zeros(0), np.zeros(0), level, np.zeros(0) if mobility else None))
        parts.append(spectrum(mz[:1], it[:1], level, np.ones(1) if mobility else None))
        parts.append(spectrum([np.inf, 1.0], [np.inf, -np.inf], level, np.ones(2) if mobility else None))   # TIC: inf + -inf
        parts.append(spectrum([5.0, 5.0, 5.0], [-0.0, -0.0, -0.0], level, np.ones(3) if mobility else None))   # TIC of -0.0s from +0.0
        parts.append(spectrum([3.0, 1.0, 2.0], _f32([0x3F800000, 0xFF812345, 0x7F800007]), level, np.ones(3) if mobility else None))
    run(concat(parts), what=f"special values mob={mobility}")


@pytest.mark.parametrize("order", ["sorted", "shuffled"])
def test_size_class_boundaries(order):
    rng = np.random.default_rng(15)
    parts = []
    for n in (0, 1, 2, 31, 32, 33, 255, 256, 257, 2048, 2049, RAW_SMEM_PEAKS - 1, RAW_SMEM_PEAKS, RAW_SMEM_PEAKS + 1, 3 * RAW_SMEM_PEAKS + 5):
        mz = rng.uniform(100.0, 1500.0, n).astype(np.float32)
        if n:
            mz[n // 3:n // 2] = mz[0]   # a run of equal masses inside
        if order == "sorted":
            mz = np.sort(mz)
        parts.append(spectrum(mz, np.exp(rng.normal(9, 1, n)), 1, rng.uniform(0.6, 1.4, n)))
    run(concat(parts), what=order)


def test_large_shuffled_spectrum():
    rng = np.random.default_rng(16)
    n = (1 << 20) + 3
    mz = rng.uniform(100.0, 1700.0, n).astype(np.float32)
    mz[rng.integers(0, n, n // 10)] = mz[rng.integers(0, n, n // 10)]   # duplicates
    it = np.exp(rng.normal(9, 2, n)).astype(np.float32)
    raw = concat([spectrum(mz, it, 1, rng.uniform(0.6, 1.4, n)), spectrum(np.sort(mz), it, 1, np.ones(n)), synth.make_raw_spectra(50, mobility=True, seed=17)])
    run(raw, what="2^20 peaks")


def test_ten_thousand_spectra():
    raw = synth.make_raw_spectra(10_000, peaks=(0, 300), levels=(0, 1, 2, 3, 4), mobility=True, seed=18)
    run(raw, what="1e4 spectra")


# ------------------------------------------------------------------------------------------------ LFQ from raw MS1
@pytest.fixture(scope="module")
def pep():
    return lfq_cases.peptides()


@pytest.fixture(scope="module")
def db(pep):
    return IndexedDatabase.build_from_peptides(pep, device=0)


def _oracle_ms1(raw):
    p = PO.so_process(raw)
    return Ms1Batch(p["peak_off"], p["masses"], p["intensities"], raw.file_id, raw.scan_start_time, p["mobilities"] if raw.mobility is not None else None)


@pytest.mark.parametrize("mobility", [False, True])
def test_lfq_add_raw_ms1(db, pep, mobility):
    runs = synth.make_ms1_runs(pep, n_ids=3000, n_files=3, spectra_per_file=400, peaks_per_spectrum=400, mobility=mobility, seed=0x51)
    settings, charges = LfqSettings(), (2, 3)
    raw = synth.ms1_to_raw(runs["batch"])
    processed = _oracle_ms1(raw)

    ref = FeatureMap.build(db, pep, settings, charges, runs["features"], runs["alignments"])
    ref.add_ms1(processed)
    orc = LO.LfqOracle(pep, settings, charges, runs["features"], runs["alignments"])
    orc.add_ms1(processed)
    want = ref.export(grids=True)
    want_q = ref.quantify()
    assert assert_map_and_grids_equal(ref, orc, settings.combine_charge_states, charges) > 0
    assert_integration_matches(ref, orc)

    for shuffle, splits in ((False, 1), (True, 1), (True, 5), (False, 7)):
        fm = FeatureMap.build(db, pep, settings, charges, runs["features"], runs["alignments"])
        r = synth.ms1_to_raw(runs["batch"], shuffle=shuffle, seed=0x52 + splits)
        cuts = np.linspace(0, len(r), splits + 1).astype(int)
        for a, z in zip(cuts[:-1], cuts[1:]):
            fm.add_raw_ms1(r.slice(a, z))
        got = fm.export(grids=True)
        assert got["touched"].tobytes() == want["touched"].tobytes(), f"shuffle={shuffle} splits={splits}: touched grids"
        assert got["grids"].tobytes() == want["grids"].tobytes(), f"shuffle={shuffle} splits={splits}: grid cells"
        q = fm.quantify()
        for k in want_q:
            assert np.asarray(q[k]).tobytes() == np.asarray(want_q[k]).tobytes(), f"shuffle={shuffle} splits={splits}: quantify {k}"


def test_lfq_add_raw_ms1_large_spectra(db, pep):
    """Spectra past the shared-memory class go through the segmented sort inside add_raw_ms1 as well."""
    runs = synth.make_ms1_runs(pep, n_ids=500, n_files=1, spectra_per_file=20, peaks_per_spectrum=3 * RAW_SMEM_PEAKS, mobility=True, seed=0x53)
    raw = synth.ms1_to_raw(runs["batch"], shuffle=True)
    settings, charges = LfqSettings(), (2, 3)
    ref = FeatureMap.build(db, pep, settings, charges, runs["features"], runs["alignments"])
    ref.add_ms1(_oracle_ms1(raw))
    fm = FeatureMap.build(db, pep, settings, charges, runs["features"], runs["alignments"])
    fm.add_raw_ms1(raw)
    assert fm.export(grids=True)["grids"].tobytes() == ref.export(grids=True)["grids"].tobytes()


# ------------------------------------------------------------------------------------------------ tmt::quantify
def _tmt_raw(seed):
    """MS2 and MS3 spectra (and MS1) holding every 18-plex reporter within a few ppm, among noise."""
    rng = np.random.default_rng(seed)
    parts = []
    for s in range(300):
        level = int(rng.choice([1, 2, 3]))
        rep = api.TMT18PLEX[rng.random(18) < 0.8]
        rep = (rep * (1.0 + rng.normal(0, 6e-6, len(rep)))).astype(np.float32)
        noise = rng.uniform(110.0, 1500.0, int(rng.integers(0, 200))).astype(np.float32)
        mz = rng.permutation(np.concatenate([rep, rep[: len(rep) // 3] + np.float32(0.001), noise]))
        parts.append(spectrum(mz, np.exp(rng.normal(9, 1, len(mz))), level, charge=int(rng.integers(0, 4))))
    return concat(parts)


@pytest.mark.parametrize("level", [1, 2, 3])
@pytest.mark.parametrize("isobaric", ["Tmt6", "Tmt10", "Tmt11", "Tmt16", "Tmt18"])
def test_tmt_quantify(isobaric, level):
    raw = _tmt_raw(19)
    mdm = api.tmt_min_deisotope_mz(isobaric, level)
    sp = SpectrumProcessor(150, level == 2, mdm)
    got = sp.process_raw(raw)
    want = PO.so_process(raw, 150, level == 2, mdm)
    assert_same(got, want, f"{isobaric} level {level}")
    rows, q = api.tmt_quantify(got, isobaric, level)
    if level == 1:
        assert len(rows) == 0 and q.shape == (0, len(api.ISOBARIC[isobaric]))
        return
    keep = np.nonzero(want["level"] == level)[0]
    assert rows.tolist() == keep.tolist() and len(rows) > 0
    off = want["peak_off"].astype(np.int64)
    take = np.concatenate([np.arange(off[r], off[r + 1]) for r in keep])
    sub_off = np.concatenate([[0], np.cumsum(off[keep + 1] - off[keep])]).astype(np.uint64)
    o = O.find_reporter_ions(sub_off, want["masses"][take], want["intensities"][take], api.ISOBARIC[isobaric], (O.PPM, -20.0, 20.0))
    assert q.tobytes() == np.asarray(o, np.float32).tobytes()
    assert (q > 0).mean() > 0.5
