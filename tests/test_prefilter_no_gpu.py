"""Argument errors of the prefilter (sage_b200_prefilter_create) that are reported before the device is looked at, so on any machine; and,
on a box without GPUs, a valid call failing with ECUDA (there is no CPU fallback)."""
import ctypes as C

import numpy as np
import pytest

import sage_b200
from sage_b200 import SageB200Error, SpectraBatch, Tolerance, api

EINVAL, ECUDA, ELIMIT = -1, -2, -5
FASTA = b">A\nMKWVTFISLLLLFSSAYSRGVFRRDTHKSEIAHRFK\n>B\nPEPTIDEKAAAAGGGKLLLLIIIIR\n"


def _spectra(n=3, peaks=20):
    off = np.arange(n + 1, dtype=np.uint64) * peaks
    masses = np.tile(np.linspace(200.0, 1200.0, peaks, dtype=np.float32), n)
    return SpectraBatch(peak_off=off, masses=masses, intensities=np.ones(n * peaks, np.float32), prec_mz=np.full(n, 600.0, np.float32),
                        prec_charge=np.full(n, 2, np.uint8), iso_lo=np.full(n, np.nan, np.float32), iso_hi=np.full(n, np.nan, np.float32),
                        tic=np.full(n, float(peaks), np.float32))


def _scorer(**kw):
    p = api.CScorerParams()
    p.precursor_tol, p.fragment_tol = Tolerance.ppm(-20, 20)._c(), Tolerance.ppm(-20, 20)._c()
    p.min_matched_peaks, p.min_precursor_charge, p.max_precursor_charge, p.max_fragment_charge, p.report_psms = 4, 2, 4, -1, 1
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _create(fasta=FASTA, dp="default", sp="default", pp="default", spectra="default", bucket_size=8192, kinds=(1, 4)):
    keep: list = []
    dp = api._digest_params(keep) if dp == "default" else dp
    sp = _scorer() if sp == "default" else sp
    pp = api.CPrefilterParams(0, 1, 15) if pp == "default" else pp
    cs = _spectra()._c(keep) if spectra == "default" else spectra
    k = np.array(kinds, np.uint8)
    h = C.c_void_p()
    ref = lambda x: None if x is None else C.byref(x)  # noqa: E731
    return api.load_library().sage_b200_prefilter_create(C.c_int(0), fasta, C.c_uint64(len(fasta) if fasta else 10), ref(dp), ref(sp), ref(pp), ref(cs),
                                                         C.c_uint64(bucket_size), api._ptr(k), C.c_uint64(len(k)), C.c_uint64(2), C.byref(h))


@pytest.mark.parametrize("what", ["fasta", "digest", "scorer", "params", "spectra"])
def test_null_arguments(what):
    args = {"fasta": None} if what == "fasta" else {{"digest": "dp", "scorer": "sp", "params": "pp", "spectra": "spectra"}[what]: None}
    assert _create(**args) == EINVAL
    assert "null" in api._last_error()


def test_argument_errors_before_the_device():
    keep: list = []
    assert _create(dp=api._digest_params(keep, static_mods={"C": float("inf")})) == EINVAL
    assert _create(dp=api._digest_params(keep, variable_mods={"M": [float("nan")]})) == EINVAL
    assert _create(sp=_scorer(report_psms=0)) == EINVAL
    assert _create(sp=_scorer(score_type=2)) == EINVAL
    assert _create(bucket_size=3000) == EINVAL
    assert _create(kinds=(1, 9)) == EINVAL
    assert _create(kinds=()) == EINVAL


def test_limits_before_the_device():
    keep: list = []
    assert _create(sp=_scorer(report_psms=64)) == ELIMIT
    assert "64" in api._last_error()
    assert _create(dp=api._digest_params(keep, max_len=256)) == ELIMIT
    assert _create(dp=api._digest_params(keep, max_variable_mods=9)) == ELIMIT
    with pytest.raises(SageB200Error) as e:
        sage_b200.prefilter_fasta(FASTA, _spectra(), precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), report_psms=100)
    assert e.value.code == ELIMIT


def test_python_arguments():
    with pytest.raises(ValueError):
        sage_b200.IndexedDatabase.from_fasta(FASTA, prefilter=True)
    with pytest.raises(ValueError):
        sage_b200.prefilter_fasta(FASTA, _spectra(), precursor_tol=Tolerance.ppm(-20, 20), fragment_tol=Tolerance.ppm(-20, 20), bucket_size=0)


@pytest.mark.skipif(api.device_count() > 0, reason="needs a box without GPUs")
def test_valid_call_without_gpu_is_ecuda():
    assert _create() == ECUDA
    assert "no CPU fallback" in api._last_error()
