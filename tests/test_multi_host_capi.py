"""The C-ABI of the multi-axis host twins without a GPU: xg_stencil_multi_host and xg_wreduce_host_multi are
exported and check every argument before any CUDA call (a CUDA call here would fail with XG_ECUDA)."""

import ctypes as C

import pytest

from xgcm_b200 import _build, _capi

EINVAL, ENOTIMPL = -1, -2


@pytest.fixture(scope="module")
def lib():
    _build.build()
    return _capi.load()


def _ints(*v):
    return (C.c_int * len(v))(*v)


def test_both_symbols_are_exported(lib):
    for name in ("xg_stencil_multi_host", "xg_wreduce_host_multi"):
        assert hasattr(C.CDLL(str(_capi.LIB_PATH)), name)
        assert name in _capi.SIGNATURES


def test_stencil_multi_host_checks_arguments_without_gpu(lib):
    buf = (C.c_float * 64)()
    out = (C.c_float * 64)()
    shape = _capi.i64_array([4, 4, 4])
    fills = (C.c_double * 3)(0.0, 0.0, 0.0)

    def call(dtype=0, src=buf, dst=out, ndim=3, shp=shape, naxes=2, axes=_ints(2, 1), ops=_ints(1, 1),
             lo=_ints(1, 1), hi=_ints(0, 0), bc=_ints(2, 2), fill=fills):
        return lib.xg_stencil_multi_host(dtype, src, dst, ndim, shp, naxes, axes, ops, lo, hi, bc, fill, 0)

    cases = [
        (dict(src=None), EINVAL, "null pointer"),
        (dict(shp=None), EINVAL, "null pointer"),
        (dict(axes=None), EINVAL, "null pointer"),
        (dict(fill=None), EINVAL, "null pointer"),
        (dict(ndim=0), EINVAL, "bad ndim"),
        (dict(ndim=9), EINVAL, "bad ndim"),
        (dict(naxes=1), EINVAL, "2 or 3 axes"),
        (dict(naxes=4), EINVAL, "2 or 3 axes"),
        (dict(ops=_ints(7, 7)), EINVAL, "unknown op"),
        (dict(ops=_ints(0, 1)), ENOTIMPL, "ONE operator"),
        (dict(dst=buf), EINVAL, "in-place"),
        (dict(dtype=5), EINVAL, "dtype"),
        (dict(shp=_capi.i64_array([4, -4, 4])), EINVAL, "negative extent"),
        (dict(axes=_ints(2, 3)), EINVAL, "axis out of range"),
        (dict(axes=_ints(2, 2)), EINVAL, "only once"),
        (dict(lo=_ints(2, 1)), EINVAL, "halo widths"),
        (dict(bc=_ints(2, 0)), EINVAL, "periodic / fill / extend"),
        (dict(bc=_ints(2, 4)), EINVAL, "periodic / fill / extend"),
        (dict(shp=_capi.i64_array([4, 0, 4])), EINVAL, "empty operated axis"),
        # every dim of extent > 1 operated: dim 0 is cut, and the slabs have no halo planes to give it
        (dict(naxes=3, axes=_ints(2, 1, 0), ops=_ints(1, 1, 1), lo=_ints(1, 1, 1), hi=_ints(0, 0, 0),
              bc=_ints(2, 2, 1)), ENOTIMPL, "periodic boundary along the cut dim"),
        (dict(naxes=3, axes=_ints(2, 1, 0), ops=_ints(1, 1, 1), lo=_ints(1, 1, 1), hi=_ints(0, 0, 1),
              bc=_ints(2, 2, 2)), ENOTIMPL, "outer / inner shift along the cut dim"),
        (dict(naxes=3, axes=_ints(2, 1, 0), ops=_ints(1, 1, 1), lo=_ints(1, 1, 0), hi=_ints(0, 0, 0),
              bc=_ints(2, 2, 0)), ENOTIMPL, "outer / inner shift along the cut dim"),
    ]
    for kw, rc, msg in cases:
        assert call(**kw) == rc, kw
        assert msg in _capi.last_error(), (kw, _capi.last_error())
        assert _capi.last_error().startswith("xg_stencil_multi_host: ")
    # an empty result returns before the device is touched
    assert call(shp=_capi.i64_array([0, 4, 4])) == 0


def test_wreduce_host_multi_checks_arguments_without_gpu(lib):
    buf = (C.c_float * 64)()
    out = (C.c_float * 64)()
    shape = _capi.i64_array([4, 4, 4])
    w_strides = _capi.i64_array([0, 4, 1])

    def call(dtype=0, src=buf, w=None, ws=None, dst=out, ndim=3, shp=shape, naxes=2, axes=_ints(2, 1), mode=0,
             skipna=1):
        return lib.xg_wreduce_host_multi(dtype, src, w, ws, dst, ndim, shp, naxes, axes, mode, skipna, 0)

    cases = [
        (dict(src=None), EINVAL, "null pointer"),
        (dict(dst=None), EINVAL, "null pointer"),
        (dict(axes=None), EINVAL, "null pointer"),
        (dict(dtype=3), EINVAL, "dtype"),
        (dict(ndim=0, naxes=0), EINVAL, "bad ndim"),
        (dict(naxes=1), EINVAL, "between 2 and ndim axes"),
        (dict(naxes=4, axes=_ints(0, 1, 2, 0)), EINVAL, "between 2 and ndim axes"),
        (dict(mode=2), EINVAL, "mode"),
        (dict(mode=-1), EINVAL, "mode"),
        (dict(w=buf), EINVAL, "weight strides missing"),
        (dict(axes=_ints(2, 3)), EINVAL, "axis out of range"),
        (dict(axes=_ints(-1, 0)), EINVAL, "axis out of range"),
        (dict(axes=_ints(1, 1)), EINVAL, "only once"),
        (dict(shp=_capi.i64_array([4, -1, 4])), EINVAL, "negative extent"),
        (dict(w=buf, ws=_capi.i64_array([0, -4, 1])), EINVAL, "negative weight stride"),
        (dict(shp=_capi.i64_array([4, 0, 4])), ENOTIMPL, "empty reduced dim"),
        # (1, 64) reduced over both: no reduced dim of extent > 1 inside the only dim of extent > 1
        (dict(ndim=2, shp=_capi.i64_array([1, 64]), axes=_ints(0, 1)), ENOTIMPL, "inside the slab dim"),
    ]
    for kw, rc, msg in cases:
        assert call(**kw) == rc, kw
        assert msg in _capi.last_error(), (kw, _capi.last_error())
        assert _capi.last_error().startswith("xg_wreduce_host_multi: ")
    assert call(w=buf, ws=w_strides, shp=_capi.i64_array([0, 4, 4])) == 0  # empty result: nothing to do


def test_python_wrappers_map_the_status_codes():
    with pytest.raises(NotImplementedError):
        _capi.check(ENOTIMPL)
    with pytest.raises(ValueError):
        _capi.check(EINVAL)
