"""Entry points that take a device index and no db handle, on a box without GPUs: valid input fails with ECUDA and says there is
no CPU fallback; an argument error that is checked before the device is still reported as EINVAL."""
import ctypes as C

import numpy as np
import pytest

from sage_b200 import SageB200Error, SpectrumProcessor, Tolerance, api

pytestmark = pytest.mark.skipif(api.device_count() > 0, reason="needs a box without GPUs")

EINVAL, ECUDA = -1, -2


def _rows(n):
    rows = np.zeros(n, api.FEATURE_DTYPE)
    rows["label"] = np.where(np.arange(n) % 3 == 0, -1, 1)
    rows["hyperscore"] = np.linspace(10.0, 40.0, n)
    rows["charge"] = 2
    return rows


PEAK_OFF = np.array([0, 3, 5], np.uint64)
MZ = np.float32([126.1277, 127.1248, 400.0, 128.1344, 500.0])
INTENS = np.float32([10.0, 20.0, 30.0, 40.0, 50.0])


def _null_processor_params():
    api._check(api.load_library().sage_b200_process_spectra(C.c_int(0), None, None, None, None, None, None))


def _null_reporter_arrays():
    api._check(api.load_library().sage_b200_find_reporter_ions(C.c_int(0), C.c_uint64(2), None, None, None, None, C.c_uint64(6),
                                                               Tolerance.ppm(-20, 20)._c(), None))


VALID = {
    "device_log": lambda: api.device_log(np.array([0.5, 2.0]), 0),
    "device_math": lambda: api.device_math("exp", np.array([0.5, 2.0])),
    "kde_build": lambda: api.kde_build(np.linspace(0.0, 1.0, 16), np.arange(16) % 2, bins=100),
    "spectrum_fdr": lambda: api.spectrum_fdr(_rows(12), Tolerance.ppm(-20, 20)),
    "find_reporter_ions": lambda: api.find_reporter_ions(PEAK_OFF, MZ, INTENS, api.TMT6PLEX, Tolerance.ppm(-20, 20)),
    "process_batch": lambda: SpectrumProcessor(150, True, 200.0).process_batch(PEAK_OFF, MZ, INTENS, np.uint8([2, 3])),
}

# one argument error of each entry point that is reported before the device is looked at
BAD_ARGUMENT = {
    "device_log": lambda: api.device_log(np.array([0.5, 2.0]), 5),
    "device_math": lambda: api.device_math("exp", np.array([0.5, 2.0]), variant=5),
    "kde_build": lambda: api.kde_build(np.linspace(0.0, 1.0, 16), np.arange(16) % 2, bins=1),
    "spectrum_fdr": lambda: api.spectrum_fdr(_rows(12), Tolerance.pct(-1, 1)),
    "find_reporter_ions": _null_reporter_arrays,
    "process_batch": _null_processor_params,
}


@pytest.mark.parametrize("entry", sorted(VALID))
def test_valid_input_fails_loudly(entry):
    with pytest.raises(SageB200Error) as e:
        VALID[entry]()
    assert e.value.code == ECUDA and "no CPU fallback" in e.value.message


@pytest.mark.parametrize("entry", sorted(BAD_ARGUMENT))
def test_argument_error_before_device_check(entry):
    with pytest.raises(SageB200Error) as e:
        BAD_ARGUMENT[entry]()
    assert e.value.code == EINVAL, e.value.message
