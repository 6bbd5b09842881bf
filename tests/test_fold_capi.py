"""The C-ABI of the north-fold halo kernel without a GPU: xg_fold_rows validates its arguments before any CUDA
call."""

import ctypes as C

import pytest

from xgcm_b200 import _build, _capi


def test_fold_rows_argument_validation_without_gpu():
    """Null pointers, fold == seam and a halo wider than the interior rows give XG_EINVAL; a mirror partner
    outside the seam dim (an `inner` seam under a center pivot: mirror 1 - 2, period n + 1) gives XG_ENOTIMPL."""
    _build.build()
    lib = _capi.load()
    i64 = _capi.i64_array
    buf = (C.c_float * 64)()
    out = (C.c_float * 64)()
    shape = i64([5, 8])
    assert lib.xg_fold_rows(0, None, out, 2, shape, 0, 1, 1, 0, 1, 0, 0, 8, 0, None, None, None) == -1
    assert "null" in _capi.last_error()
    assert lib.xg_fold_rows(0, buf, None, 2, shape, 0, 1, 1, 0, 1, 0, 0, 8, 0, None, None, None) == -1
    assert lib.xg_fold_rows(0, buf, out, 2, None, 0, 1, 1, 0, 1, 0, 0, 8, 0, None, None, None) == -1
    assert lib.xg_fold_rows(0, buf, out, 2, shape, 1, 1, 1, 0, 1, 0, 0, 8, 0, None, None, None) == -1
    assert lib.xg_fold_rows(0, buf, out, 2, shape, 0, 1, 1, 0, 0, 0, 0, 8, 0, None, None, None) == -1
    assert lib.xg_fold_rows(0, buf, out, 2, shape, 0, 1, 5, 0, 5, 1, 0, 8, 0, None, None, None) == -1
    assert "interior" in _capi.last_error()
    inner = i64([5, 7])
    assert lib.xg_fold_rows(0, buf, out, 2, inner, 0, 1, 1, 0, 1, 0, -1, 8, 0, None, None, None) == -2
    assert "incompatible" in _capi.last_error()
    with pytest.raises(NotImplementedError):
        _capi.check(-2)
