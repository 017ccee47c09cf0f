"""Picked FDR entry points on a box without GPUs: valid input fails with ECUDA and says there is no CPU fallback; an argument error is
reported as EINVAL before the device is looked at."""
import numpy as np
import pytest

import picked_cases as PC
import sage_b200
from sage_b200 import SageB200Error, api

pytestmark = pytest.mark.skipif(api.device_count() > 0, reason="needs a box without GPUs")

EINVAL, ECUDA = -1, -2


def _case():
    return PC.degenerate_cases()["decoy_first"]


def _fdr(case):
    return PC.device(case)


VALID = {
    "picked_fdr": lambda: _fdr(_case()),
    "picked_precursor": lambda: sage_b200.picked_precursor(np.array([1.0, 2.0]), np.array([0, 1])),
    "competition_keys": lambda: sage_b200.competition_keys(_case()["peptides"], np.array([0, 1], np.uint32)),
}

BAD_ARGUMENT = {
    "picked_fdr": lambda: _fdr(dict(_case(), pep_idx=np.array([0, 9], np.uint32), score=np.float32([1.0, 2.0]))),
    "picked_precursor": lambda: api._check(api.load_library().sage_b200_picked_precursor(0, None, None, api.C.c_uint64(2), None, None)),
    "competition_keys": lambda: sage_b200.competition_keys(_case()["peptides"], np.array([0, 1], np.uint32), hash_bits=0),
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
