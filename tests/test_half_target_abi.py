"""The C ABI of half-precision targets, without a GPU: the dtype enum of include/nmf_b200.h, the two dense set_target entry
points (both take the dtype) in the library and in the ctypes binding, and the host side's dtype map."""
import ctypes
import os
import re

import torch

from torchnmf_b200 import _capi
from torchnmf_b200.engine import _check_target

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_vp, _i64, _int = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int


def test_header_dtype_enum():
    header = open(os.path.join(ROOT, "include", "nmf_b200.h")).read()
    values = {k: int(v) for k, v in re.findall(r"\b(NMFB200_DTYPE_\w+)\s*=\s*(\d+)", header)}
    assert values == {"NMFB200_DTYPE_F32": 0, "NMFB200_DTYPE_F16": 1, "NMFB200_DTYPE_BF16": 2}
    assert (_capi.DTYPE_F32, _capi.DTYPE_F16, _capi.DTYPE_BF16) == (0, 1, 2)
    assert _capi.DTYPES == {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def test_set_target_symbols_and_argtypes():
    assert _capi.SIGNATURES["nmfb200_nmf_set_target"] == (_int, [_vp, _vp, _i64, _int, _vp])
    assert _capi.SIGNATURES["nmfb200_nmfd_set_target"] == (_int, [_vp, _vp, _int, _vp])
    lib = _capi.load()
    for name in ("nmfb200_nmf_set_target", "nmfb200_nmfd_set_target"):
        fn = getattr(lib, name)
        assert fn.restype is _int and fn.argtypes == _capi.SIGNATURES[name][1]
    assert lib.nmfb200_nmf_set_target(None, None, 1, 0, None) == 1
    assert b"null context" in lib.nmfb200_last_error()
    assert lib.nmfb200_nmfd_set_target(None, None, 0, None) == 1


def test_engine_target_checks():
    cpu = torch.device("cpu")
    for dtype in (torch.float32, torch.float16, torch.bfloat16):
        _check_target(torch.zeros(4, 6, dtype=dtype), cpu)
    for dtype in (torch.float64, torch.int32):
        try:
            _check_target(torch.zeros(4, 6, dtype=dtype), cpu)
        except TypeError as e:
            assert "float32, float16 or bfloat16" in str(e)
        else:
            raise AssertionError(dtype)
    rows = torch.zeros(4, 9, dtype=torch.bfloat16)[:, 2:8]          # row stride 9 > 6 columns, unit column stride
    _check_target(rows, cpu, strided_rows=True)
    for bad, strided in ((rows, False), (torch.zeros(6, 4, dtype=torch.bfloat16).t(), True)):
        try:
            _check_target(bad, cpu, strided_rows=strided)
        except ValueError:
            pass
        else:
            raise AssertionError(bad.stride())
