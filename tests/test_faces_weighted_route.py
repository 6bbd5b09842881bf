"""Metric-weighted operators across face connections without a GPU: the C-ABI of xg_stencil2_host_connected_weighted
checks every argument before any CUDA call; the weighted copy list (``connected_halo_program`` with a metric layout)
replayed in numpy gives the halo of x * pre; the Grid sends a weighted numpy field to the streamed entry point exactly
where it should (with the kernels replaced by the oracle), with the values of the device route and of the reference's
pad(x * m) -> stencil -> / m_new; and a weighted cumint of a numpy field on a plain grid takes the whole-field route."""

import ctypes as C
import itertools

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from _mock_backend import install
from oracle import stencil as S
from oracle.faces import pad_face_connections
from xgcm_b200 import _build, _capi, device, ops
from xgcm_b200.padding import broadcast_strides, connected_halo_program

SHAPE = [4, 3, 6, 5]  # (batch, face, y, x): axis 3 (x) is operated, the planes are (4, 3, 6, 1)
ROW, PLANE_ROW = 3 * 6 * 5, 3 * 6
PRE_STRIDES = [0, 30, 5, 1]  # a (face, y, x) metric broadcast over the batch dim


@pytest.fixture(scope="module")
def lib():
    _build.build()
    return _capi.load()


def _copy(side=1, source=0, doff=0, soff=0, shape=(4, 3, 6), dstr=(PLANE_ROW, 6, 1), sstr=(ROW, 30, 5), neg=0,
          poff=0, pstr=(0, 30, 5)):
    return [side, source, doff, soff, list(shape), list(dstr), list(sstr), neg, poff, list(pstr)]


FILL = _copy(source=2, sstr=(0, 0, 0), pstr=(0, 0, 0))


def _weighted(lib, copies, **kw):
    a, out, m = (C.c_float * 512)(), (C.c_float * 512)(), (C.c_float * 128)()
    n = len(copies)
    cndim = len(copies[0][4]) if copies else 3
    i32 = lambda v: (C.c_int * max(n, 1))(*v)  # noqa: E731
    flat = lambda k: _capi.i64_array([v for c in copies for v in c[k]] or [0])  # noqa: E731
    one = lambda k: _capi.i64_array([c[k] for c in copies] or [0])  # noqa: E731
    args = dict(op=0, dtype=0, inp=a, out=out, ndim=4, shape=_capi.i64_array(SHAPE), axis=3, lo=0, hi=1, fill=0.0,
                pre=m, pre_st=_capi.i64_array(PRE_STRIDES), post=None, post_st=None, n=n, cndim=cndim,
                side=i32([c[0] for c in copies]), source=i32([c[1] for c in copies]), doff=one(2), soff=one(3),
                poff=one(8), shapes=flat(4), dstr=flat(5), sstr=flat(6), pstr=flat(9),
                neg=i32([c[7] for c in copies]), device=0)
    args.update(kw)
    return lib.xg_stencil2_host_connected_weighted(*args.values())


def _einval(rc, text):
    assert rc == -1, (rc, _capi.last_error())
    assert text in _capi.last_error(), _capi.last_error()


def test_symbol_exported(lib):
    assert hasattr(lib, "xg_stencil2_host_connected_weighted")
    assert "xg_stencil2_host_connected_weighted" in _capi.SIGNATURES


def test_weighted_validation_without_gpu(lib):
    _einval(_weighted(lib, [FILL], inp=None), "null pointer")
    _einval(_weighted(lib, [FILL], axis=0), "dim 0")
    _einval(_weighted(lib, [FILL], lo=2), "halo widths")
    _einval(_weighted(lib, [FILL], pre=None), "null pre-metric")
    _einval(_weighted(lib, [FILL], pre_st=None), "metric strides missing")
    _einval(_weighted(lib, [FILL], side=None), "null pointer in the copy list")
    _einval(_weighted(lib, [FILL], poff=None), "null pointer in the copy list")
    _einval(_weighted(lib, [FILL], pstr=None), "null pointer in the copy list")
    # no partner: a copy that reads one is refused
    _einval(_weighted(lib, [_copy(source=1)]), "partner that was not given")
    # the field copies are checked as in xg_stencil2_host_connected
    _einval(_weighted(lib, [_copy(soff=5)]), "leaves its source array")
    _einval(_weighted(lib, [_copy(shape=(4, 2, 6))]), "do not cover")
    # the metric copies: the pre-metric's dim-0 stride, inside the pre-metric, the constant 1 for a fill copy
    _einval(_weighted(lib, [_copy(pstr=(30, 30, 5))]), "dim-0 stride")
    _einval(_weighted(lib, [_copy(poff=5)]), "leaves the pre-metric")
    _einval(_weighted(lib, [_copy(pstr=(0, 30, -5))]), "leaves the pre-metric")
    _einval(_weighted(lib, [_copy(source=2, sstr=(0, 0, 0), poff=1, pstr=(0, 0, 0))]), "constant 1")
    _einval(_weighted(lib, [_copy(source=2, sstr=(0, 0, 0), pstr=(0, 0, 1))]), "constant 1")
    # an unknown host device group: before any CUDA call too
    _einval(_weighted(lib, [FILL], device=_capi.XG_HOST_GROUP_BASE + 999), "group")


N = 6
COORDS = {"X": {"center": "x", "left": "xl", "outer": "xo"}, "Y": {"center": "y", "left": "yl"},
          "Z": {"center": "k", "left": "kl"}}
AXES = {"X": ("x", "xl", "xo"), "Y": ("y", "yl"), "Z": ("k", "kl")}
CUBED_SPHERE = {
    "face": {
        0: {"X": ((3, "X", False), (1, "X", False)), "Y": ((4, "Y", False), (5, "Y", False))},
        1: {"X": ((0, "X", False), (2, "X", False)), "Y": ((4, "X", False), (5, "X", True))},
        2: {"X": ((1, "X", False), (3, "X", False)), "Y": ((4, "Y", True), (5, "Y", True))},
        3: {"X": ((2, "X", False), (0, "X", False)), "Y": ((4, "X", True), (5, "X", False))},
        4: {"X": ((3, "Y", True), (1, "Y", False)), "Y": ((2, "Y", True), (0, "Y", False))},
        5: {"X": ((3, "Y", False), (1, "Y", True)), "Y": ((0, "Y", False), (2, "Y", True))},
    }
}
STRIP = {"face": {0: {"X": (None, (1, "X", False))}, 1: {"X": ((0, "X", False), None)}}}


def _dataset(fc, lead=(2, 3), seed=0):
    rng = np.random.default_rng(seed)
    nf = len(fc["face"])
    coords = {"x": np.arange(N) + 0.0, "xl": np.arange(N) - 0.5, "xo": np.arange(N + 1) - 0.5,
              "y": np.arange(N) + 0.0, "yl": np.arange(N) - 0.5, "face": np.arange(nf),
              "k": np.arange(lead[1]) + 0.0, "kl": np.arange(lead[1]) - 0.5}
    return xg.Dataset(data_vars={
        "c": (("t", "k", "face", "y", "x"), rng.standard_normal(lead + (nf, N, N))),
        "u": (("t", "k", "face", "y", "xl"), rng.standard_normal(lead + (nf, N, N))),
        "v": (("t", "k", "face", "yl", "x"), rng.standard_normal(lead + (nf, N, N))),
        "dx_c": (("k", "face", "y", "x"), 0.5 + rng.random((lead[1], nf, N, N))),
        "dx_l": (("k", "face", "y", "xl"), 0.5 + rng.random((lead[1], nf, N, N))),
        "dx_o": (("k", "face", "y", "xo"), 0.5 + rng.random((lead[1], nf, N, N + 1))),
        "dy_c": (("face", "y", "x"), 0.5 + rng.random((nf, N, N))),
        "dy_l": (("face", "yl", "x"), 0.5 + rng.random((nf, N, N))),
        "dz_c": (("k",), 0.5 + rng.random(lead[1])),
        "dz_l": (("kl",), 0.5 + rng.random(lead[1]))}, coords=coords)


def _grid(ds, fc):
    return xg.Grid(ds, coords=COORDS, face_connections=fc, autoparse_metadata=False,
                   metrics={("X",): ["dx_c", "dx_l", "dx_o"], ("Y",): ["dy_c", "dy_l"], ("Z",): ["dz_c", "dz_l"]})


def _replay(program, x, pre, fill, p_shape):
    """The weighted copy list: planes of x (fill constant), weight planes of pre (1), multiplied."""
    planes = [np.full(p_shape, np.inf, x.dtype), np.full(p_shape, np.inf, x.dtype)]
    weights = [np.full(p_shape, np.inf, x.dtype), np.full(p_shape, np.inf, x.dtype)]
    xs = {"self": x.ravel(), "fill": np.array([fill], x.dtype)}
    ms = {"self": np.ascontiguousarray(pre, x.dtype).ravel(), "fill": np.array([1.0], x.dtype)}
    for side, doff, dstr, src, soff, sstr, shp, neg, poff, pstr in program:
        assert src != "partner" and not neg and shp[0] == x.shape[0]
        idx = np.indices(shp).reshape(len(shp), -1)
        di = doff + (np.asarray(dstr)[:, None] * idx).sum(0)
        planes[side].reshape(-1)[di] = xs[src][soff + (np.asarray(sstr)[:, None] * idx).sum(0)]
        weights[side].reshape(-1)[di] = ms[src][poff + (np.asarray(pstr)[:, None] * idx).sum(0)]
    return [p * w for p, w in zip(planes, weights)]


def _connected_weighted(x, axis, op, lo, hi, fill_value, program, pre, post=None, out=None, device=None):
    """The definition of xg_stencil2_host_connected_weighted (include/xgcm_b200.h) on the oracle-backed stencil."""
    x = np.asarray(x)
    p_shape = list(x.shape)
    p_shape[axis] = 1
    hl, hh = _replay(program, x, pre, fill_value, p_shape)
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, x.dtype))  # noqa: E731
    return ops.stencil2(t(x), axis, op, lo, hi, "fill" if (lo or hi) else None, fill_value, pre=t(pre), post=t(post),
                        halo_lo=t(hl) if lo else None, halo_hi=t(hh) if hi else None).numpy()


@pytest.fixture
def spy(monkeypatch):
    """Oracle-backed ops on a grid device of type cuda (the whole-field route's upload stays on the CPU), with the
    names of the streamed entry points each call ran."""
    install(monkeypatch)
    monkeypatch.setattr(device, "default_device", lambda: torch.device("cuda"))
    monkeypatch.setattr(xg.DataArray, "to_device", lambda self, dev=None: self._replace(
        data=torch.from_numpy(np.ascontiguousarray(self.data))))
    ran = []

    def weighted(*a, **kw):
        ran.append("stencil2_host_connected_weighted")
        return _connected_weighted(*a, **kw)

    def unweighted(*a, **kw):
        ran.append("stencil2_host_connected")

    monkeypatch.setattr(ops, "stencil2_host_connected_weighted", weighted)
    monkeypatch.setattr(ops, "stencil2_host_connected", unweighted)
    return ran


def _dev(da):
    return xg.DataArray(torch.from_numpy(np.ascontiguousarray(da.values)), dims=da.dims)


def _vals(x):
    return x.data.numpy() if isinstance(x.data, torch.Tensor) else np.asarray(x.data)


def _bcast(da, dims):
    v = np.transpose(da.values, [da.dims.index(d) for d in dims if d in da.dims])
    return v.reshape([da.values.shape[da.dims.index(d)] if d in da.dims else 1 for d in dims])


@pytest.mark.parametrize("mode", ["fill", "extend", "periodic"])
def test_weighted_program_is_the_halo_of_x_times_pre(mode):
    ds = _dataset(STRIP)
    grid = _grid(ds, STRIP)
    c = ds["c"]
    for ax, (lo, hi), metric in itertools.product(["X", "Y"], [(1, 0), (0, 1), (1, 1)], ["dx_c", "dy_c"]):
        dims, shape = c.dims, list(c.shape)
        pre = _bcast(ds[metric], dims)
        program = connected_halo_program(grid, ax, lo, hi, dims, shape, mode,
                                         pre_strides=broadcast_strides(pre.shape, shape))
        assert all(len(p) == 10 for p in program)
        t = dims.index([d for d in dims if d in AXES[ax]][0])
        p_shape = list(shape)
        p_shape[t] = 1
        planes = _replay(program, c.values, pre, 1.5, p_shape)
        want = pad_face_connections(c.values * pre, dims, AXES, "face", STRIP["face"], {ax: (lo, hi)},
                                    {a: mode for a in AXES}, {a: 1.5 for a in AXES})
        for side, w, row in ((0, lo, 0), (1, hi, want.shape[t] - 1)):
            if w:
                np.testing.assert_array_equal(planes[side], np.take(want, [row], axis=t), err_msg=f"{ax} {metric}")


def _oracle(op, da, fc, ax, lo, hi, padding, fill, pre, post):
    padded = pad_face_connections(da.values * pre, da.dims, AXES, "face", fc["face"], {ax: (lo, hi)},
                                  {a: padding for a in AXES}, {a: fill for a in AXES})
    return S.stencil2(op, padded, da.dims.index([d for d in da.dims if d in AXES[ax]][0]), 0, 0, None) / post


@pytest.mark.parametrize("name", ["cubed_sphere", "strip"])
def test_weighted_numpy_field_streams(name, spy):
    fc = {"cubed_sphere": CUBED_SPHERE, "strip": STRIP}[name]
    ds = _dataset(fc)
    grid = _grid(ds, fc)
    c = ds["c"]
    cases = [("X", "left", "X", "dx_c", "dx_l"), ("X", "outer", "X", "dx_c", "dx_o"),
             ("Y", "left", "Y", "dy_c", "dy_l"), ("Z", "left", "Z", "dz_c", "dz_l")]
    for (ax, to, weighted, m_in, m_out), (padding, fill), op in itertools.product(
            cases, [("fill", 1.5), ("extend", 0.0), ("periodic", 0.0)], ["diff", "interp", "min", "max"]):
        kw = dict(to=to, padding=padding, fill_value=fill, metric_weighted=weighted)
        spy.clear()
        got = getattr(grid, op)(c, ax, **kw)
        assert spy == ["stencil2_host_connected_weighted"], (ax, to, spy)
        dev = getattr(grid, op)(_dev(c), ax, **kw)
        assert spy == ["stencil2_host_connected_weighted"]
        np.testing.assert_array_equal(_vals(got), _vals(dev), err_msg=f"{op} {ax} {padding}")
        lo, hi = S.PADDING_WIDTH[("center", to)]
        want = _oracle(op, c, fc, ax, lo, hi, padding, fill, _bcast(ds[m_in], c.dims), _bcast(ds[m_out], got.dims))
        np.testing.assert_array_equal(_vals(got), want, err_msg=f"{op} {ax} {padding}")


def test_whole_field_layouts_and_vectors(spy):
    ds = _dataset(CUBED_SPHERE)
    grid = _grid(ds, CUBED_SPHERE)
    # (face, k, j, i): no batch dim in front of the face dim -> the fused device route
    a = np.ascontiguousarray(ds["c"].values[0].transpose(1, 0, 2, 3))
    da = xg.DataArray(a, dims=("face", "k", "y", "x"))
    spy.clear()
    got = grid.interp(da, "X", metric_weighted="X")
    assert spy == []
    np.testing.assert_array_equal(_vals(got), _vals(grid.interp(_dev(da), "X", metric_weighted="X")))
    want = _oracle("interp", da, CUBED_SPHERE, "X", 1, 0, None, 0.0, _bcast(ds["dx_c"], da.dims),
                   _bcast(ds["dx_l"], got.dims))
    np.testing.assert_array_equal(_vals(got), want)
    # device tensors never stream
    grid.interp(_dev(ds["c"]), "X", metric_weighted="X")
    assert spy == []
    # vector components with a pre-metric: not implemented, on either route
    u, v = ds["u"], ds["v"]
    for arg, other in ((u, v), (_dev(u), _dev(v))):
        with pytest.raises(NotImplementedError, match="vector components"):
            grid.interp({"X": arg}, "X", other_component={"Y": other}, metric_weighted="X")
    assert spy == []


def test_plain_grid_weighted_cumint_of_numpy_field(spy):
    rng = np.random.default_rng(5)
    ds = xg.Dataset(data_vars={"a": (("t", "y", "x"), rng.standard_normal((3, 5, 7))),
                               "dx": (("y", "x"), 0.5 + rng.random((5, 7))),
                               "dxl": (("y", "xl"), 0.5 + rng.random((5, 7)))},
                    coords={"x": np.arange(7.0), "xl": np.arange(7.0) - 0.5, "y": np.arange(5.0)})
    grid = xg.Grid(ds, coords={"X": {"center": "x", "left": "xl"}, "Y": {"center": "y"}}, autoparse_metadata=False,
                   metrics={("X",): ["dx", "dxl"]}, padding="fill")
    got = grid.cumint(ds["a"], "X", metric_weighted="X")
    want = grid.cumint(_dev(ds["a"]), "X", metric_weighted="X")
    assert isinstance(got.data, np.ndarray)
    np.testing.assert_array_equal(_vals(got), _vals(want))
