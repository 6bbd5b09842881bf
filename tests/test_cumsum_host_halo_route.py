"""Grid.cumsum / cumint of numpy fields on face-connected and north-fold grids without a GPU: the C-ABI of
xg_cumscan_host_fold / xg_cumscan_host_connected checks every argument before any CUDA call, and the Grid picks
the streamed route (xg_cumscan_host, or its _fold / _connected twin) with the kernels replaced by the oracle, giving
the values and errors of the whole-field route."""

import ctypes as C
import itertools
import warnings

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from _mock_fold import fold_rows
from _mock_fold import install as install_fold
from oracle import stencil as S
from xgcm_b200 import _build, _capi, ops

SHAPE = [4, 3, 6, 5]  # (batch, face, y, x), scanned along x (axis 3) and trimmed: the scanned field is (4, 3, 6, 4)
ROW, PLANE_ROW = 3 * 6 * 4, 3 * 6


@pytest.fixture(scope="module")
def lib():
    _build.build()
    return _capi.load()


def _bufs():
    return (C.c_float * 512)(), (C.c_float * 512)()


def _fold(lib, **kw):
    a, out = _bufs()
    args = dict(dtype=0, inp=a, out=out, ndim=4, shape=_capi.i64_array(SHAPE), axis=2, reverse=1, trim=2, lo=0, hi=1,
                pre=None, pre_st=None, post=None, post_st=None, skipna=1, seam=3, skip=0, mirror=0, period=5,
                device=0)
    args.update(kw)
    return lib.xg_cumscan_host_fold(*args.values())


def _copy(side=1, source=0, doff=0, soff=0, shape=(4, 3, 6), dstr=(PLANE_ROW, 6, 1), sstr=(ROW, 24, 4), neg=0):
    return [side, source, doff, soff, list(shape), list(dstr), list(sstr), neg]


def _connected(lib, copies, **kw):
    a, out = _bufs()
    n = len(copies)
    cndim = len(copies[0][4]) if copies else 3
    i32 = lambda v: (C.c_int * max(n, 1))(*v)  # noqa: E731
    flat = lambda k: _capi.i64_array([v for c in copies for v in c[k]] or [0])  # noqa: E731
    args = dict(dtype=0, inp=a, out=out, ndim=4, shape=_capi.i64_array(SHAPE), axis=3, reverse=1, trim=2, lo=0, hi=1,
                fill=0.0, pre=None, pre_st=None, post=None, post_st=None, skipna=1, n=n, cndim=cndim,
                side=i32([c[0] for c in copies]), source=i32([c[1] for c in copies]),
                doff=_capi.i64_array([c[2] for c in copies] or [0]), soff=_capi.i64_array([c[3] for c in copies] or [0]),
                shapes=flat(4), dstr=flat(5), sstr=flat(6), neg=i32([c[7] for c in copies]), device=0)
    args.update(kw)
    return lib.xg_cumscan_host_connected(*args.values())


def _einval(rc, text):
    assert rc == -1, (rc, _capi.last_error())
    assert text in _capi.last_error(), _capi.last_error()


def test_symbols_exported(lib):
    for name in ("xg_cumscan_host_fold", "xg_cumscan_host_connected"):
        assert hasattr(lib, name) and name in _capi.SIGNATURES


def test_fold_validation_without_gpu(lib):
    a, _ = _bufs()
    _einval(_fold(lib, inp=None), "null pointer")
    _einval(_fold(lib, dtype=7), "dtype")
    _einval(_fold(lib, ndim=0), "bad ndim")
    _einval(_fold(lib, axis=4), "axis out of range")
    _einval(_fold(lib, axis=0, seam=3), "dim 0")                  # the scanned dim would be cut into slabs
    _einval(_fold(lib, shape=_capi.i64_array([4, 3, -6, 5])), "negative extent")
    _einval(_fold(lib, trim=3), "unknown trim")
    _einval(_fold(lib, hi=2), "pad widths")
    _einval(_fold(lib, hi=0), "pad_lo must be 0, pad_hi 1")
    _einval(_fold(lib, lo=1), "pad_lo must be 0, pad_hi 1")
    _einval(_fold(lib, pre=a), "metric strides missing")
    _einval(_fold(lib, post=a), "metric strides missing")
    _einval(_fold(lib, shape=_capi.i64_array([4, 3, 1, 5])), "no scanned row")
    _einval(_fold(lib, seam=0), "seam dim")                       # the seam dim would be cut into slabs
    _einval(_fold(lib, seam=2), "must differ")
    _einval(_fold(lib, seam=7), "seam axis out of range")
    _einval(_fold(lib, skip=2), "skip")
    _einval(_fold(lib, period=0), "period")
    # the fold row is planned for the SCANNED field: 2 rows, trimmed to 1, leave no interior row past the pole
    _einval(_fold(lib, shape=_capi.i64_array([4, 3, 2, 5]), skip=1), "interior rows")
    _einval(_fold(lib, device=_capi.XG_HOST_GROUP_BASE + 63), "unknown host device group")
    assert _fold(lib, mirror=-1, period=6) == -2  # an `inner` seam under a center pivot
    assert "incompatible" in _capi.last_error()


def test_connected_validation_without_gpu(lib):
    a, _ = _bufs()
    fill = _copy(source=2, sstr=(0, 0, 0))
    _einval(_connected(lib, [fill], inp=None), "null pointer")
    _einval(_connected(lib, [fill], axis=0), "dim 0")
    _einval(_connected(lib, [fill], trim=-1), "unknown trim")
    _einval(_connected(lib, [fill], lo=2), "pad widths")
    _einval(_connected(lib, [fill], pre=a), "metric strides missing")
    _einval(_connected(lib, [fill], n=-1), "negative copy count")
    _einval(_connected(lib, [fill], side=None), "null pointer in the copy list")
    _einval(_connected(lib, [fill], cndim=0), "bad copy rank")
    _einval(_connected(lib, [_copy(side=2)]), "side")
    _einval(_connected(lib, [_copy(side=0)]), "does not pad")
    _einval(_connected(lib, [_copy(source=3)]), "source must be")
    _einval(_connected(lib, [_copy(source=1)]), "partner that was not given")  # a scalar field has none
    # the copies read the scanned field: its dim-0 stride is the trimmed row, not the input's
    _einval(_connected(lib, [_copy(sstr=(3 * 6 * 5, 30, 5))]), "span dim 0")
    _einval(_connected(lib, [_copy(shape=(3, 3, 6))]), "span dim 0")
    _einval(_connected(lib, [_copy(dstr=(PLANE_ROW + 1, 6, 1))]), "span dim 0")
    _einval(_connected(lib, [_copy(doff=1)]), "leaves the halo plane")
    _einval(_connected(lib, [_copy(soff=4)]), "leaves its source array")  # past the 4 scanned columns
    _einval(_connected(lib, [_copy(source=2, soff=1, sstr=(0, 0, 0))]), "fill constant")
    _einval(_connected(lib, [_copy(shape=(4, 2, 6))]), "do not cover")
    _einval(_connected(lib, [], n=0), "do not cover")
    _einval(_connected(lib, [fill], device=_capi.XG_HOST_GROUP_BASE + 63), "unknown host device group")


# ---------------------------------------------------------------------------------------------- Grid routing
def _scan(x, axis, reverse, trim, pre, skipna):
    return np.ascontiguousarray(S.cumscan(x, axis, reverse, trim, 0, 0, None, 0.0, pre, None, skipna))


def _host_fold(x, axis, reverse, trim, seam_axis, skip, mirror, period, pre=None, post=None, skipna=True,
               device=None):
    """The definition of xg_cumscan_host_fold (include/xgcm_b200.h)."""
    c = _scan(x, axis, reverse, trim, pre, skipna)
    out = np.concatenate([c, fold_rows(torch.from_numpy(c), axis, seam_axis, 1, skip, mirror, period).numpy()], axis)
    return out if post is None else out / post


def _host_connected(x, axis, reverse, trim, pad_lo, pad_hi, fill_value, program, pre=None, post=None, skipna=True,
                    device=None):
    """The definition of xg_cumscan_host_connected: the copy list replayed on the scanned field."""
    c = _scan(x, axis, reverse, trim, pre, skipna)
    p_shape = list(c.shape)
    p_shape[axis] = 1
    planes = [np.full(p_shape, np.inf, c.dtype), np.full(p_shape, np.inf, c.dtype)]
    srcs = {"self": c.ravel(), "fill": np.array([fill_value], c.dtype)}
    for side, doff, dstr, src, soff, sstr, shp, neg in program:
        assert shp[0] == c.shape[0] and src != "partner"
        idx = np.indices(shp).reshape(len(shp), -1)
        v = srcs[src][soff + (np.asarray(sstr)[:, None] * idx).sum(0)]
        planes[side].reshape(-1)[doff + (np.asarray(dstr)[:, None] * idx).sum(0)] = -v if neg else v
    out = np.concatenate(([planes[0]] if pad_lo else []) + [c] + ([planes[1]] if pad_hi else []), axis)
    return out if post is None else out / post


@pytest.fixture
def spy(monkeypatch):
    install_fold(monkeypatch)
    ran = []
    for name, fn in (("cumscan_host", ops.cumscan_host), ("cumscan_host_fold", _host_fold),
                     ("cumscan_host_connected", _host_connected)):
        def wrapped(*a, _fn=fn, _name=name, **kw):
            ran.append(_name)
            return _fn(*a, **kw)

        monkeypatch.setattr(ops, name, wrapped)
    return ran


def _dev(da):
    return xg.DataArray(torch.from_numpy(np.ascontiguousarray(da.values)), dims=da.dims)


def _vals(x):
    return x.data.numpy() if isinstance(x.data, torch.Tensor) else np.asarray(x.data)


N = 6
COORDS = {"X": {"center": "x", "left": "xl", "outer": "xo"}, "Y": {"center": "y", "left": "yl", "outer": "yo"},
          "Z": {"center": "k", "left": "kl"}}
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


def _faces(fc):
    rng = np.random.default_rng(0)
    nf = len(fc["face"])
    shape = (2, 3, nf, N, N)
    c = rng.standard_normal(shape)
    c[rng.random(shape) < 0.1] = np.nan
    ds = xg.Dataset(
        data_vars={"c": (("t", "k", "face", "y", "x"), c), "u": (("t", "k", "face", "y", "xl"), rng.random(shape))},
        coords={"x": np.arange(N), "xl": np.arange(N), "xo": np.arange(N + 1), "y": np.arange(N),
                "yl": np.arange(N), "yo": np.arange(N + 1), "k": np.arange(3), "kl": np.arange(3),
                "face": np.arange(nf), "dx_c": (("face", "y", "x"), 1 + rng.random((nf, N, N))),
                "dx_o": (("face", "y", "xo"), 1 + rng.random((nf, N, N + 1)))})
    return ds, xg.Grid(ds, coords=COORDS, face_connections=fc, metrics={("X",): ["dx_c", "dx_o"]})


def _same_as_device(grid, da, ax, spy, ran, **kw):
    spy.clear()
    got = grid.cumsum(da, ax, **kw)
    assert spy == ran, (ax, kw, spy)
    dev = grid.cumsum(_dev(da), ax, **kw)
    np.testing.assert_array_equal(_vals(got), _vals(dev), err_msg=f"{ax} {kw}")


@pytest.mark.parametrize("fc", [CUBED_SPHERE, STRIP], ids=["cubed_sphere", "strip"])
def test_faces_route_and_values(fc, spy):
    ds, grid = _faces(fc)
    c, u = ds["c"], ds["u"]
    entries = [(c, "outer", False), (c, "outer", True)]
    if fc is STRIP:  # no seam swaps axes: the trimmed entries pad too
        entries += [(c, "left", False), (u, "center", True)]
    for (da, to, reverse), (padding, fill), ax in itertools.product(
            entries, [("fill", 1.5), ("extend", 0.0), ("periodic", 0.0)], ("X", "Y")):
        if ax == "Y" and da is u:
            continue
        want = "cumscan_host_connected" if ax in fc["face"][0] else "cumscan_host"
        _same_as_device(grid, da, ax, spy, [want], to=to, reverse=reverse, padding=padding, fill_value=fill)
    # the pre weight and the post divide
    _same_as_device(grid, c, "X", spy, ["cumscan_host_connected"], to="outer", reverse=True, metric_weighted="X",
                    padding="fill")
    spy.clear()
    got = grid.cumint(c, "X", to="outer", reverse=True, padding="extend")
    assert spy == ["cumscan_host_connected"]
    np.testing.assert_array_equal(_vals(got), _vals(grid.cumint(_dev(c), "X", to="outer", reverse=True,
                                                                padding="extend")))
    # Z and a shift that pads nothing need no seam
    _same_as_device(grid, c, "Z", spy, ["cumscan_host"], to="left", padding="extend")
    _same_as_device(grid, u, "X", spy, ["cumscan_host"], to="center")


def test_faces_errors_and_whole_field_routes(spy):
    ds, grid = _faces(CUBED_SPHERE)
    c = ds["c"]
    for arg in (c, _dev(c)):
        with pytest.raises(ValueError, match="equal size"):
            grid.cumsum(arg, "X", to="left", padding="fill")
        with pytest.raises(ValueError, match="No boundary condition"):
            grid.cumsum(arg, "Z", to="left")
    ds2, strip = _faces(STRIP)
    for arg in (ds2["c"], _dev(ds2["c"])):
        with pytest.raises(ValueError, match="No boundary condition"):
            strip.cumsum(arg, "X", to="outer")
    assert spy == []
    # no batch dim in front of the face dim, and cumint + metric_weighted: the whole-field route
    t = xg.DataArray(np.ascontiguousarray(np.moveaxis(c.values, 2, 0)), dims=("face", "t", "k", "y", "x"))
    got = grid.cumsum(t, "Y", to="outer", padding="extend")
    np.testing.assert_array_equal(_vals(got), _vals(grid.cumsum(_dev(t), "Y", to="outer", padding="extend")))
    got = grid.cumint(c, "X", to="outer", metric_weighted="X")
    np.testing.assert_array_equal(_vals(got), _vals(grid.cumint(_dev(c), "X", to="outer", metric_weighted="X")))
    assert spy == []


NX, NY = 8, 7
POS = ("center", "left", "right", "outer")
EXTRA = {"center": 0, "left": 0, "right": 0, "outer": 1}


def _fold_grid(pivot, south):
    coords = {"x" + p: np.arange(NX + EXTRA[p]) for p in POS}
    coords.update({"y" + p: np.arange(NY + EXTRA[p]) for p in POS})
    rng = np.random.default_rng(1)
    ds = xg.Dataset(data_vars={f"dy_{p}": (("y" + p, "xcenter"), 0.5 + rng.random((NY + EXTRA[p], NX)))
                               for p in POS}, coords=coords)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        grid = xg.Grid(ds, coords={"X": {p: "x" + p for p in POS}, "Y": {p: "y" + p for p in POS}},
                       padding={"X": "periodic", "Y": {"fold": pivot, "south": south}}, autoparse_metadata=False)
    grid.set_metrics("Y", [f"dy_{p}" for p in POS])
    return grid


@pytest.mark.parametrize("pivot", ["T", "F", "U", "V"])
def test_fold_route_and_values(pivot, spy):
    rng = np.random.default_rng(2)
    for south in ("fill", "periodic"):
        grid = _fold_grid(pivot, south)
        for src, to, reverse in [("center", "right", True), ("center", "outer", True), ("left", "center", True),
                                 ("center", "left", False), ("center", "outer", False)]:
            a = rng.standard_normal((2, 3, NY, NX))
            a[rng.random(a.shape) < 0.1] = np.nan
            da = xg.DataArray(a, dims=("t", "z", "y" + src, "xcenter"))
            folds = reverse  # a reverse scan pads the north edge: across the fold
            _same_as_device(grid, da, "Y", spy, ["cumscan_host_fold" if folds else "cumscan_host"], to=to,
                            reverse=reverse)
        _same_as_device(grid, da, "Y", spy, ["cumscan_host_fold"], to="right", reverse=True, metric_weighted="Y")
    spy.clear()
    got = grid.cumint(da, "Y", to="right", reverse=True)
    assert spy == ["cumscan_host_fold"]
    np.testing.assert_array_equal(_vals(got), _vals(grid.cumint(_dev(da), "Y", to="right", reverse=True)))
    # a 2-D field and cumint + metric_weighted keep the whole-field route
    spy.clear()
    flat = xg.DataArray(rng.standard_normal((NY, NX)), dims=("ycenter", "xcenter"))
    np.testing.assert_array_equal(_vals(grid.cumsum(flat, "Y", to="outer", reverse=True)),
                                  _vals(grid.cumsum(_dev(flat), "Y", to="outer", reverse=True)))
    got = grid.cumint(da, "Y", to="right", reverse=True, metric_weighted="Y")
    np.testing.assert_array_equal(
        _vals(got), _vals(grid.cumint(_dev(da), "Y", to="right", reverse=True, metric_weighted="Y")))
    assert spy == []
