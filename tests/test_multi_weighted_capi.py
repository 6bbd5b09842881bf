"""The C-ABI of the weighted multi-axis stencils without a GPU: xg_stencil_multi_weighted and
xg_stencil_multi_weighted_host check every argument, the per-stage metric operands included, before any CUDA call
(a CUDA call here would fail with XG_ECUDA), and both are exported and declared in _capi.SIGNATURES."""

import ctypes as C

import pytest

from xgcm_b200 import _build, _capi

EINVAL, ENOTIMPL = -1, -2
NAMES = ("xg_stencil_multi_weighted", "xg_stencil_multi_weighted_host")


@pytest.fixture(scope="module")
def lib():
    _build.build()
    return _capi.load()


def _ints(*v):
    return (C.c_int * len(v))(*v)


def _ptrs(*v):
    return (C.c_void_p * len(v))(*v)


def test_both_symbols_are_exported_and_declared(lib):
    for name in NAMES:
        assert hasattr(C.CDLL(str(_capi.LIB_PATH)), name)
        assert name in _capi.SIGNATURES
    header = (_build.PKG_DIR.parent / "include" / "xgcm_b200.h").read_text()
    for name in NAMES:
        assert f"XG_API int {name}(" in header


@pytest.mark.parametrize("name", NAMES)
def test_arguments_are_checked_without_gpu(lib, name):
    buf = (C.c_float * 64)()
    out = (C.c_float * 64)()
    met = (C.c_float * 64)()
    shape = _capi.i64_array([4, 4, 4])
    fills = (C.c_double * 3)(0.0, 0.0, 0.0)
    good = _capi.i64_array([16, 4, 1] * 2)  # naxes x ndim: full 3-D metrics for both stages
    fn = getattr(lib, name)
    last = 0 if name.endswith("_host") else None  # device index / stream

    def call(dtype=0, src=buf, dst=out, ndim=3, shp=shape, naxes=2, axes=_ints(2, 1), ops=_ints(1, 1),
             lo=_ints(1, 1), hi=_ints(0, 0), bc=_ints(2, 2), fill=fills, pre=_ptrs(C.addressof(met), None),
             pre_st=good, post=None, post_st=None):
        return fn(dtype, src, dst, ndim, shp, naxes, axes, ops, lo, hi, bc, fill, pre, pre_st, post, post_st, last)

    cases = [
        (dict(src=None), EINVAL, "null pointer"),
        (dict(dst=None), EINVAL, "null pointer"),
        (dict(shp=None), EINVAL, "null pointer"),
        (dict(axes=None), EINVAL, "null pointer"),
        (dict(ops=None), EINVAL, "null pointer"),
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
        (dict(axes=_ints(-1, 1)), EINVAL, "axis out of range"),
        (dict(axes=_ints(2, 2)), EINVAL, "only once"),
        (dict(lo=_ints(2, 1)), EINVAL, "halo widths"),
        (dict(bc=_ints(2, 0)), EINVAL, "periodic / fill / extend"),
        (dict(shp=_capi.i64_array([4, 0, 4])), EINVAL, "empty operated axis"),
        # a metric without strides, or with a negative one along a dim of extent > 1: it cannot broadcast
        (dict(pre_st=None), EINVAL, "metric strides missing"),
        (dict(post=_ptrs(None, C.addressof(met)), post_st=None), EINVAL, "metric strides missing"),
        (dict(pre_st=_capi.i64_array([16, -4, 1] + [0, 0, 0])), EINVAL, "negative metric stride"),
        (dict(post=_ptrs(None, C.addressof(met)), post_st=_capi.i64_array([0, 0, 0] + [-16, 4, 1])), EINVAL,
         "negative metric stride"),
        # the last two dims not operated: the weighted kernel addresses metrics by one innermost dim
        (dict(ndim=4, shp=_capi.i64_array([4, 4, 2, 2]), axes=_ints(1, 0), pre_st=_capi.i64_array([16, 4, 2, 1] * 2)),
         ENOTIMPL, "more than one non-operated dim after the last operated one"),
    ]
    for kw, rc, msg in cases:
        assert call(**kw) == rc, kw
        assert msg in _capi.last_error(), (kw, _capi.last_error())
        assert _capi.last_error().startswith(f"{name}: ")
    # a stride along a dim of extent 1 is never read, and an empty result returns before the device is touched
    assert call(shp=_capi.i64_array([0, 4, 4]), pre_st=_capi.i64_array([-1, 4, 1, 0, 0, 0])) == 0


def test_host_twin_keeps_the_slab_refusals(lib):
    buf = (C.c_float * 64)()
    out = (C.c_float * 64)()
    met = (C.c_float * 64)()
    fills = (C.c_double * 3)(0.0, 0.0, 0.0)
    st = _capi.i64_array([16, 4, 1] * 3)
    # every dim of extent > 1 operated: dim 0 is cut, and the slabs have no halo planes to give it
    rc = lib.xg_stencil_multi_weighted_host(0, buf, out, 3, _capi.i64_array([4, 4, 4]), 3, _ints(2, 1, 0),
                                            _ints(1, 1, 1), _ints(1, 1, 1), _ints(0, 0, 0), _ints(2, 2, 1), fills,
                                            _ptrs(C.addressof(met), None, None), st, None, None, 0)
    assert rc == ENOTIMPL
    assert "periodic boundary along the cut dim" in _capi.last_error()
