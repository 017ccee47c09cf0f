"""SpectrumProcessor::process for every MS level without a GPU: the CPU oracle (oracle_process/) against the reference's own known answers
(spectrum.rs:607-650), its level-2 composition with oracle/'s process_ms2, and the x86-64 NaN rules DESIGN.md §16 defines; the argument
errors of sage_b200_process_raw and sage_b200_lfq_add_raw_ms1, reported before the device is looked at, on any machine."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as O
from oracle_process import process_oracle as PO
from sage_b200 import RawSpectra, SageB200Error, SpectrumProcessor, api, synth

EINVAL, ECUDA, ELIMIT = -1, -2, -5
PROTON = np.float32(1.0072764)


def bits(x):
    return np.atleast_1d(np.asarray(x, np.float32)).view(np.uint32).tolist()


def f32(u):
    return np.array(u, np.uint32).view(np.float32)


@pytest.mark.parametrize("mobility", [False, True])
def test_oracle_known_answers(mobility):
    # process_ms1_without_mobility_builds_empty_mobility_column / process_ms1_with_mobility_sorts_all_columns_by_mass
    m, i, mb, tic = PO.process_one([102.0, 100.0, 101.0], [30.0, 10.0, 20.0], 1, [3.0, 1.0, 2.0] if mobility else None)
    assert bits(m) == bits([np.float32(100.0) - PROTON, np.float32(101.0) - PROTON, np.float32(102.0) - PROTON])
    assert i.tolist() == [10.0, 20.0, 30.0]
    assert mb.tolist() == ([1.0, 2.0, 3.0] if mobility else [])
    assert tic == np.float32(60.0)


def test_oracle_level2_is_process_ms2():
    raw = synth.make_raw_spectra(40, peaks=(0, 300), levels=(2,), seed=3)
    for kw in (dict(take_top_n=150, deisotope=False), dict(take_top_n=50, deisotope=True, min_deisotope_mz=131.0)):
        got = PO.so_process(raw, **kw)
        for s in range(len(raw)):
            a, b = int(raw.peak_off[s]), int(raw.peak_off[s + 1])
            m, i, tic = O.process_ms2(raw.mz[a:b], raw.intensity[a:b], int(raw.precursor_charge[s]) or None, kw["take_top_n"], kw["deisotope"],
                                      kw.get("min_deisotope_mz", 0.0))
            c, d = int(got["peak_off"][s]), int(got["peak_off"][s + 1])
            assert bits(got["masses"][c:d]) == bits(m) and bits(got["intensities"][c:d]) == bits(i) and bits(got["tic"][s]) == bits(tic)
            assert np.isnan(got["mobilities"][c:d]).all() and not got["has_mobilities"][s]


def test_oracle_stable_total_cmp_order():
    mz = f32([0xFFC00005, 0x7F800000, 0x00000000, 0x80000000, 0x7FC00001, 0xFF800000]).tolist() + [5.0, 5.0]
    it = [1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0, 8.0]
    m, i, _, _ = PO.process_one(mz, it, 3)
    # -NaN < -inf < -PROTON (from +-0, +0 stays behind -0 in input order? both give -PROTON: input order) < 5 - PROTON (twice) < inf < +NaN
    assert i.tolist() == [1.0, 6.0, 3.0, 4.0, 7.0, 8.0, 2.0, 5.0]
    assert bits(m)[0] == 0xFFC00005 and bits(m)[-1] == 0x7FC00001


def test_oracle_nan_rules():
    # a NaN m/z keeps its sign and payload, quieted (subss); a signalling NaN becomes quiet
    m, _, _, _ = PO.process_one(f32([0xFF812345]), [1.0], 1)
    assert bits(m) == [0xFFC12345]
    # fold: the first NaN operand, quieted, then the accumulator's NaN wins over a later one
    _, _, _, tic = PO.process_one([1.0, 2.0, 3.0], f32([0x3F800000, 0xFF812345, 0x7F800007]), 0)
    assert bits(tic) == [0xFFC12345]
    # inf + -inf is x86's default NaN
    _, _, _, tic = PO.process_one([1.0, 2.0], f32([0x7F800000, 0xFF800000]), 4)
    assert bits(tic) == [0xFFC00000]
    # the fold starts at +0.0: -0.0 + -0.0 would stay -0.0
    _, _, _, tic = PO.process_one([1.0], f32([0x80000000]), 1)
    assert bits(tic) == [0x00000000]


def _raw(**kw):
    r = dict(peak_off=np.array([0, 3, 5], np.uint64), mz=np.float32([300.0, 200.0, 100.0, 500.0, 400.0]), intensity=np.float32([1, 2, 3, 4, 5]),
             level=np.uint8([1, 3]), precursor_charge=None, mobility=None)
    r.update(kw)
    return RawSpectra(**r)


def _process(raw, **kw):
    return SpectrumProcessor(150, False, 0.0, **kw).process_raw(raw)


def _null_params():
    api._check(api.load_library().sage_b200_process_raw(C.c_int(0), None, None, None, None, None, None, None))


def _null_mobilities_out():
    keep = []
    raw = _raw()._c(keep)
    pp = api.CProcessorParams(150, 0, 0.0)
    off, o, t = np.zeros(3, np.uint64), np.zeros(5, np.float32), np.zeros(2, np.float32)
    api._check(api.load_library().sage_b200_process_raw(C.c_int(0), C.byref(pp), C.byref(raw), api._ptr(off), api._ptr(o), api._ptr(o), None, api._ptr(t)))


def _null_level():
    keep = []
    raw = _raw()._c(keep)
    raw.level = None
    pp = api.CProcessorParams(150, 0, 0.0)
    off, o, t = np.zeros(3, np.uint64), np.zeros(5, np.float32), np.zeros(2, np.float32)
    api._check(api.load_library().sage_b200_process_raw(C.c_int(0), C.byref(pp), C.byref(raw), api._ptr(off), api._ptr(o), api._ptr(o), api._ptr(o),
                                                        api._ptr(t)))


def _big_ms2():
    n = 10_000
    return _raw(peak_off=np.array([0, 3, 3 + n], np.uint64), mz=np.linspace(100.0, 2000.0, 3 + n, dtype=np.float32), intensity=np.ones(3 + n, np.float32),
                level=np.uint8([1, 2]), precursor_charge=np.uint8([0, 2]))


BAD = {
    "null_params": (_null_params, EINVAL),
    "null_level": (_null_level, EINVAL),
    "null_mobilities_out": (_null_mobilities_out, EINVAL),
    "offsets_not_monotone": (lambda: _process(_raw(peak_off=np.array([0, 4, 3], np.uint64))), EINVAL),
    "ms2_without_charge": (lambda: _process(_raw(level=np.uint8([1, 2]))), EINVAL),
    "ms2_past_budget": (lambda: _process(_big_ms2()), ELIMIT),
    "lfq_null_handle": (lambda: api._check(api.load_library().sage_b200_lfq_add_raw_ms1(None, None)), EINVAL),
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_argument_errors_before_device(case):
    f, code = BAD[case]
    with pytest.raises(SageB200Error) as e:
        f()
    assert e.value.code == code, e.value.message


def test_empty_batch_needs_no_device():
    r = _process(_raw(peak_off=np.zeros(1, np.uint64), mz=np.zeros(0, np.float32), intensity=np.zeros(0, np.float32), level=np.zeros(0, np.uint8)))
    assert r.peak_off.tolist() == [0] and len(r.masses) == 0


def test_add_raw_ms1_takes_ms1_only():
    fm = api.FeatureMap.__new__(api.FeatureMap)
    fm._h = None
    with pytest.raises(ValueError):
        fm.add_raw_ms1(_raw())


@pytest.mark.skipif(api.device_count() > 0, reason="needs a box without GPUs")
def test_valid_input_fails_loudly():
    with pytest.raises(SageB200Error) as e:
        _process(_raw())
    assert e.value.code == ECUDA and "no CPU fallback" in e.value.message


def test_tmt_tables_and_min_deisotope_mz():
    assert [len(api.ISOBARIC[k]) for k in ("Tmt6", "Tmt10", "Tmt11", "Tmt16", "Tmt18")] == [6, 10, 11, 16, 18]
    assert bits(api.ISOBARIC["Tmt10"]) == bits(api.TMT11PLEX[:10]) and bits(api.ISOBARIC["Tmt16"]) == bits(api.TMT18PLEX[:16])
    assert bits(api.ISOBARIC["Tmt11"][-1]) == bits(np.float32(131.144499))
    want = np.float32(131.144499) * (np.float32(1.0) + np.float32(20e-6))
    assert bits(np.float32(api.tmt_min_deisotope_mz("Tmt11", 2))) == bits(want)
    assert api.tmt_min_deisotope_mz("Tmt11", 3) == 0.0
    rows, q = api.tmt_quantify(api.ProcessedBatch(np.array([0, 1], np.uint64), np.float32([125.0]), np.float32([1.0]), np.float32([np.nan]),
                                                  np.zeros(1, bool), np.float32([1.0]), np.uint8([1])), "Tmt6", 1)
    assert len(rows) == 0 and q.shape == (0, 6)
