"""The C-ABI of the multi-result and multi-axis host twins without a GPU: xg_stencil2_host_multi,
xg_stencil_multi_host and xg_wreduce_host_multi check every argument before any CUDA call (a CUDA call here would
fail with XG_ECUDA); the two multi-axis twins are exported."""

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


def test_stencil2_host_multi_checks_arguments_without_gpu(lib):
    buf = (C.c_float * 64)()
    res = [(C.c_float * 64)() for _ in range(2)]
    outs = (C.c_void_p * 2)(*[C.addressof(r) for r in res])
    shape = _capi.i64_array([4, 4, 4])
    fills = (C.c_double * 2)(0.0, 0.0)

    def call(nout=2, ops=_ints(0, 1), dtype=0, src=buf, dst=outs, ndim=3, shp=shape, axes=_ints(2, 0),
             lo=_ints(1, 1), hi=_ints(0, 0), bc=_ints(1, 2), fill=fills):
        return lib.xg_stencil2_host_multi(nout, ops, dtype, src, dst, ndim, shp, axes, lo, hi, bc, fill, 0)

    cases = [
        (dict(src=None), EINVAL, "null pointer"),
        (dict(dst=None), EINVAL, "null pointer"),
        (dict(shp=None), EINVAL, "null pointer"),
        (dict(ops=None), EINVAL, "null pointer"),
        (dict(axes=None), EINVAL, "null pointer"),
        (dict(lo=None), EINVAL, "null pointer"),
        (dict(hi=None), EINVAL, "null pointer"),
        (dict(bc=None), EINVAL, "null pointer"),
        (dict(fill=None), EINVAL, "null pointer"),
        (dict(nout=0), EINVAL, "between 1 and 8 results per call"),
        (dict(nout=9), EINVAL, "between 1 and 8 results per call"),
        (dict(dst=(C.c_void_p * 2)(outs[0], None)), EINVAL, "null result pointer"),
        (dict(dtype=5), EINVAL, "dtype must be XG_F32 or XG_F64"),
        (dict(ndim=0), EINVAL, "bad ndim"),
        (dict(ndim=9), EINVAL, "bad ndim"),
        (dict(axes=_ints(3, 0)), EINVAL, "axis out of range"),
        (dict(axes=_ints(2, -1)), EINVAL, "axis out of range"),
        (dict(lo=_ints(2, 1)), EINVAL, "halo widths must be 0 or 1"),
        (dict(hi=_ints(0, -1)), EINVAL, "halo widths must be 0 or 1"),
        (dict(bc=_ints(0, 2)), EINVAL, "no boundary condition was specified but the operation needs to pad the axis"),
        (dict(bc=_ints(1, 5)), EINVAL, "no boundary condition was specified but the operation needs to pad the axis"),
        (dict(shp=_capi.i64_array([4, 4, 0])), EINVAL, "empty operated axis"),
        (dict(shp=_capi.i64_array([0, 4, 4])), EINVAL, "empty operated axis"),
        # dim 0 is cut into slabs: a result along it keeps its extent and pads only at the field's ends
        (dict(hi=_ints(0, 1)), ENOTIMPL, "outer / inner shifts along the outermost dimension"),
        (dict(lo=_ints(1, 0)), ENOTIMPL, "outer / inner shifts along the outermost dimension"),
        (dict(bc=_ints(1, 4)), ENOTIMPL, "extrapolate along the outermost dimension"),
    ]
    for kw, rc, msg in cases:
        assert call(**kw) == rc, kw
        assert msg in _capi.last_error(), (kw, _capi.last_error())
        assert _capi.last_error().startswith("xg_stencil2_host_multi: ")


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
