"""Protein grouping entry points on a box without GPUs: valid input fails with ECUDA and says there is no CPU fallback; an argument error is
reported as EINVAL before the device is looked at."""
import numpy as np
import pytest

import protein_group_cases as G
import sage_b200
from sage_b200 import SageB200Error, api

pytestmark = pytest.mark.skipif(api.device_count() > 0, reason="needs a box without GPUs")

EINVAL, ECUDA = -1, -2


def _case():
    return G.known_cases()["expected_groups"]


def _groups(case, off=None, ids=None, n_names=None):
    o, i, names = G.name_ids(case)
    off = o if off is None else off
    ids = i if ids is None else ids
    return sage_b200.protein_groups(case["peptides"], G.rows_of(case), case["peptide_q"], case["score"], off, ids, len(names) if n_names is None else n_names)


def _bad_offsets():
    off, ids, names = G.name_ids(_case())
    off = off.copy()
    off[3], off[4] = off[4], off[3]
    return _groups(_case(), off=off)


def _bad_id():
    off, ids, names = G.name_ids(_case())
    ids = ids.copy()
    ids[2] = len(names)
    return _groups(_case(), ids=ids)


VALID = {
    "protein_groups": lambda: _groups(_case()),
    "bipartite_cover": lambda: sage_b200.bipartite_cover(np.array([0, 1], np.uint32), np.array([0, 0], np.uint32), 2, 1),
}

BAD_ARGUMENT = {
    "peptide_idx_out_of_range": lambda: _groups(dict(_case(), pep_idx=np.array([0, 10], np.uint32), label=np.ones(2, np.int32),
                                                     peptide_q=np.zeros(2, np.float32), score=np.zeros(2, np.float32))),
    "protein_offsets_decreasing": _bad_offsets,
    "protein_id_not_below_n_names": _bad_id,
    "cover_edge_out_of_range": lambda: sage_b200.bipartite_cover(np.array([0, 2], np.uint32), np.array([0, 0], np.uint32), 2, 1),
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
