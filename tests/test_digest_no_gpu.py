"""Argument errors of the digest that are reported before the device is looked at (so on any machine)."""
import ctypes as C

import pytest

import sage_b200
from sage_b200 import SageB200Error, api

EINVAL, ELIMIT = -1, -5


def _params(**kw):
    p = api.CDigestParams()
    p.min_len, p.max_len, p.cleave_at, p.restrict_, p.c_terminal = 5, 50, b"KR", b"P", 1
    p.peptide_min_mass, p.peptide_max_mass, p.max_variable_mods, p.decoy_tag, p.generate_decoys = 500.0, 5000.0, 2, b"rev_", 1
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _create(fasta, n, params):
    h = C.c_void_p()
    return api.load_library().sage_b200_digest_create(C.c_int(0), fasta, C.c_uint64(n), C.byref(params) if params is not None else None, C.byref(h))


def test_null_fasta_and_params():
    assert _create(None, 10, _params()) == EINVAL
    assert _create(b">A\nPEPTIDEK\n", 11, None) == EINVAL
    assert "null" in api._last_error()


def test_null_mod_arrays():
    assert _create(b">A\nPEPTIDEK\n", 11, _params(n_static=1)) == EINVAL
    assert _create(b">A\nPEPTIDEK\n", 11, _params(n_variable=2)) == EINVAL


def test_max_len_and_max_variable_mods_limits():
    assert _create(b">A\nPEPTIDEK\n", 11, _params(max_len=256)) == ELIMIT
    assert "255" in api._last_error()
    with pytest.raises(SageB200Error) as e:
        sage_b200.digest_fasta(">A\nPEPTIDEK\n", max_len=256)
    assert e.value.code == ELIMIT
    with pytest.raises(SageB200Error) as e:
        sage_b200.digest_fasta(">A\nPEPTIDEK\n", max_variable_mods=9)
    assert e.value.code == ELIMIT


def test_non_finite_mass():
    with pytest.raises(SageB200Error) as e:
        sage_b200.digest_fasta(">A\nPEPTIDEK\n", static_mods={"C": float("nan")})
    assert e.value.code == EINVAL


@pytest.mark.parametrize("bucket_size", [0, -4, 2.5, "8192", None, True, 1 << 31])
def test_from_fasta_bad_bucket_size(bucket_size):
    with pytest.raises(ValueError):
        sage_b200.IndexedDatabase.from_fasta(">A\nPEPTIDEK\n", bucket_size=bucket_size)
