"""The C-ABI of the host slab pipelines with a per-slab halo stage (xg_stencil2_host_fold /
xg_stencil2_host_connected) without a GPU: every argument is checked before any CUDA call."""

import ctypes as C

import pytest

from xgcm_b200 import _build, _capi

SHAPE = [4, 3, 6, 5]  # (batch, face, y, x): axis 3 (x) is operated, the planes are (4, 3, 6, 1)
ROW, PLANE_ROW = 3 * 6 * 5, 3 * 6


@pytest.fixture(scope="module")
def lib():
    _build.build()
    return _capi.load()


def _bufs():
    return (C.c_float * 512)(), (C.c_float * 512)()


def _fold(lib, **kw):
    a, out = _bufs()
    args = dict(op=0, dtype=0, inp=a, out=out, ndim=4, shape=_capi.i64_array(SHAPE), axis=2, lo=1, hi=1, bc=1,
                fill=0.0, pre=None, pre_st=None, post=None, post_st=None, seam=3, skip=0, mirror=0, period=5,
                negate=0, device=0)
    args.update(kw)
    return lib.xg_stencil2_host_fold(*args.values())


def _copy(side=1, source=0, doff=0, soff=0, shape=(4, 3, 6), dstr=(PLANE_ROW, 6, 1), sstr=(ROW, 30, 5), neg=0):
    return [side, source, doff, soff, list(shape), list(dstr), list(sstr), neg]


def _connected(lib, copies, partner=None, partner_shape=None, **kw):
    a, out = _bufs()
    n = len(copies)
    cndim = len(copies[0][4]) if copies else 3
    i32 = lambda v: (C.c_int * max(n, 1))(*v)  # noqa: E731
    flat = lambda k: _capi.i64_array([v for c in copies for v in c[k]] or [0])  # noqa: E731
    args = dict(op=0, dtype=0, inp=a, partner=partner, pshape=_capi.i64_array(partner_shape), out=out, ndim=4,
                shape=_capi.i64_array(SHAPE), axis=3, lo=0, hi=1, fill=0.0, post=None, post_st=None, n=n,
                cndim=cndim, side=i32([c[0] for c in copies]), source=i32([c[1] for c in copies]),
                doff=_capi.i64_array([c[2] for c in copies] or [0]), soff=_capi.i64_array([c[3] for c in copies] or [0]),
                shapes=flat(4), dstr=flat(5), sstr=flat(6), neg=i32([c[7] for c in copies]), device=0)
    args.update(kw)
    return lib.xg_stencil2_host_connected(*args.values())


def _einval(lib, rc, text):
    assert rc == -1, (rc, _capi.last_error())
    assert text in _capi.last_error(), _capi.last_error()


def test_fold_validation_without_gpu(lib):
    a, _ = _bufs()
    _einval(lib, _fold(lib, inp=None), "null pointer")
    _einval(lib, _fold(lib, axis=0, seam=3), "dim 0")          # the fold dim would be cut into slabs
    _einval(lib, _fold(lib, seam=0), "seam dim")               # ... or the seam dim
    _einval(lib, _fold(lib, seam=2), "must differ")
    _einval(lib, _fold(lib, seam=7), "seam axis out of range")
    _einval(lib, _fold(lib, hi=0), "hi must be 1")
    _einval(lib, _fold(lib, skip=2), "skip")
    _einval(lib, _fold(lib, period=0), "period")
    _einval(lib, _fold(lib, pre=a), "metric strides missing")
    _einval(lib, _fold(lib, bc=0), "no boundary condition")
    _einval(lib, _fold(lib, shape=_capi.i64_array([4, 3, 1, 5]), skip=1), "interior rows")
    # an `inner` seam (period = n + 1) under a center pivot: a mirror partner outside the seam dim
    assert _fold(lib, mirror=-1, period=6) == -2
    assert "incompatible" in _capi.last_error()


def test_connected_validation_without_gpu(lib):
    a, _ = _bufs()
    fill = _copy(source=2, sstr=(0, 0, 0))
    _einval(lib, _connected(lib, [fill], inp=None), "null pointer")
    _einval(lib, _connected(lib, [fill], axis=0), "dim 0")
    _einval(lib, _connected(lib, [fill], n=-1), "negative copy count")
    _einval(lib, _connected(lib, [fill], side=None), "null pointer in the copy list")
    _einval(lib, _connected(lib, [fill], cndim=0), "bad copy rank")
    _einval(lib, _connected(lib, [_copy(side=2)]), "side")
    _einval(lib, _connected(lib, [_copy(side=0)]), "does not pad")
    _einval(lib, _connected(lib, [_copy(source=3)]), "source must be")
    _einval(lib, _connected(lib, [_copy(source=1)]), "partner that was not given")
    # a copy list must span dim 0 in full with the contiguous dim-0 strides (so no seam maps dim 0)
    _einval(lib, _connected(lib, [_copy(shape=(3, 3, 6))]), "span dim 0")
    _einval(lib, _connected(lib, [_copy(dstr=(PLANE_ROW + 1, 6, 1))]), "span dim 0")
    _einval(lib, _connected(lib, [_copy(sstr=(30, ROW, 5))]), "span dim 0")
    _einval(lib, _connected(lib, [_copy(source=2)]), "span dim 0")
    _einval(lib, _connected(lib, [_copy(doff=1)]), "leaves the halo plane")
    _einval(lib, _connected(lib, [_copy(soff=5)]), "leaves its source array")
    _einval(lib, _connected(lib, [_copy(source=2, soff=1, sstr=(0, 0, 0))]), "fill constant")
    _einval(lib, _connected(lib, [_copy(shape=(4, 2, 6))]), "do not cover")
    _einval(lib, _connected(lib, [], n=0), "do not cover")
    # the partner component streams beside the field: same dim-0 extent
    _einval(lib, _connected(lib, [fill], partner=a, partner_shape=None), "null partner shape")
    _einval(lib, _connected(lib, [fill], partner=a, partner_shape=[3, 3, 6, 5]), "dim-0 extent")
