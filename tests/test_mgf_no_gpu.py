"""The argument errors of the MGF reader's entry points (sage_b200_mgf_*, sage_b200_parse_f32), reported before any device is touched, so
they hold on any machine."""
import ctypes as C

import numpy as np
import pytest

from sage_b200 import SageB200Error, api

EINVAL, ECUDA = -1, -2


def _lib():
    return api.load_library()


def _create(text, length, out=True):
    h = C.c_void_p()
    api._check(_lib().sage_b200_mgf_create(C.c_int(0), text, C.c_uint64(length), C.c_uint64(0), C.byref(h) if out else None))


def _parse(tokens_bytes, off, n, out=True, ok=True):
    o, k = np.zeros(max(n, 1), np.float32), np.zeros(max(n, 1), np.uint8)
    api._check(_lib().sage_b200_parse_f32(C.c_int(0), tokens_bytes, api._ptr(off) if off is not None else None, C.c_uint64(n),
                                          api._ptr(o) if out else None, api._ptr(k) if ok else None))


BAD = {
    "create_null_out": lambda: _create(b"BEGIN IONS\n", 11, out=False),
    "create_null_text": lambda: _create(None, 5),
    "create_empty_file": lambda: _create(b"", 0),
    "get_info_null": lambda: api._check(_lib().sage_b200_mgf_get_info(None, None)),
    "export_null_handle": lambda: api._check(_lib().sage_b200_mgf_export(None, *([None] * 16))),
    "process_null": lambda: api._check(_lib().sage_b200_mgf_process(None, None, None, None, None, None)),
    "parse_f32_null_offsets": lambda: _parse(b"1", None, 1),
    "parse_f32_null_out": lambda: _parse(b"1", np.array([0, 1], np.uint64), 1, out=False),
    "parse_f32_null_ok": lambda: _parse(b"1", np.array([0, 1], np.uint64), 1, ok=False),
    "parse_f32_decreasing": lambda: _parse(b"12", np.array([0, 2, 1], np.uint64), 2),
    "parse_f32_null_bytes": lambda: _parse(None, np.array([0, 2], np.uint64), 1),
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_argument_errors_before_device(case):
    with pytest.raises(SageB200Error) as e:
        BAD[case]()
    assert e.value.code == EINVAL, e.value.message


def test_empty_file_message():
    with pytest.raises(SageB200Error) as e:
        api.read_mgf("")
    assert e.value.code == EINVAL and "BEGIN IONS" in e.value.message


def test_no_tokens_need_no_device():
    bits, ok = api.parse_f32([])
    assert len(bits) == 0 and len(ok) == 0


def test_text_must_be_utf8_encodable():
    with pytest.raises(UnicodeEncodeError):
        api.read_mgf("BEGIN IONS\nTITLE=\ud800\n")


@pytest.mark.skipif(api.device_count() > 0, reason="needs a box without GPUs")
def test_valid_input_fails_loudly():
    with pytest.raises(SageB200Error) as e:
        api.read_mgf("BEGIN IONS\nTITLE=a\nPEPMASS=1\n1 1\nEND IONS\n")
    assert e.value.code == ECUDA and "no CPU fallback" in e.value.message
    with pytest.raises(SageB200Error) as e:
        api.parse_f32(["1.5"])
    assert e.value.code == ECUDA
