"""Multi-axis Grid.diff / interp / min / max of numpy fields on face-connected and north-fold grids without a GPU: the
C-ABI of xg_stencil_chain_host_fold / xg_stencil_chain_host_connected checks every argument before any CUDA call, and
the Grid picks the streamed chain (with the kernels replaced by the oracle) exactly where it should, giving the values
and errors of the whole-field route."""

import ctypes as C
import itertools
import warnings

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from _mock_fold import fold_rows
from _mock_fold import install as install_fold
from xgcm_b200 import _build, _capi, device, ops

SHAPE = [4, 3, 6, 5]  # (batch, face / z, y, x)


@pytest.fixture(scope="module")
def lib():
    _build.build()
    return _capi.load()


def _i32(v):
    return (C.c_int * max(len(v), 1))(*v)


def _fold(lib, **kw):
    a, out = (C.c_float * 512)(), (C.c_float * 512)()
    # stage 0: X center -> left, periodic; stage 1: Y center -> right across the fold, seam X
    args = dict(dtype=0, inp=a, out=out, ndim=4, shape=SHAPE, nstage=2, axis=[3, 2], op=[0, 1], lo=[1, 0],
                hi=[0, 1], bc=[1, 2], fill=[0.0, 0.0], fold=[0, 1], seam=[0, 3], skip=[0, 0], mirror=[0, 0],
                period=[1, 5], device=0)
    args.update(kw)
    for k in ("axis", "op", "lo", "hi", "bc", "fold", "seam", "skip"):
        if args[k] is not None:
            args[k] = _i32(args[k])
    for k in ("shape", "mirror", "period"):
        args[k] = _capi.i64_array(args[k])
    if args["fill"] is not None:
        args["fill"] = (C.c_double * len(args["fill"]))(*args["fill"])
    return lib.xg_stencil_chain_host_fold(*args.values())


# stage 0: X center -> outer (lo = hi = 1, x becomes 6), stage 1: Y center -> right (hi = 1) of the (4, 3, 6, 6) result
ROW0, PLANE0, ROW1, PLANE1 = 90, 18, 108, 18


def _copy(side, source=2, doff=0, soff=0, shape=(4, 3, 6), dstr=(18, 6, 1), sstr=(0, 0, 0), neg=0):
    return [side, source, doff, soff, list(shape), list(dstr), list(sstr), neg]


STAGE0 = [_copy(0), _copy(1)]
STAGE1 = [_copy(1, source=0, soff=5 * 6, sstr=(ROW1, 36, 1))]  # the last y row of stage 0's result


def _connected(lib, programs=(STAGE0, STAGE1), **kw):
    a, out = (C.c_float * 512)(), (C.c_float * 512)()
    copies = [c for p in programs for c in p]
    cndim = len(copies[0][4]) if copies else 3
    flat = lambda k: _capi.i64_array([v for c in copies for v in c[k]] or [0])  # noqa: E731
    args = dict(dtype=0, inp=a, out=out, ndim=4, shape=_capi.i64_array(SHAPE), nstage=2, axis=_i32([3, 2]),
                op=_i32([0, 1]), lo=_i32([1, 0]), hi=_i32([1, 1]), fill=(C.c_double * 3)(0.0, 1.5, 0.0),
                ncopies=_i32([len(p) for p in programs]), cndim=cndim, side=_i32([c[0] for c in copies]),
                source=_i32([c[1] for c in copies]), doff=_capi.i64_array([c[2] for c in copies] or [0]),
                soff=_capi.i64_array([c[3] for c in copies] or [0]), shapes=flat(4), dstr=flat(5), sstr=flat(6),
                neg=_i32([c[7] for c in copies]), device=0)
    args.update(kw)
    return lib.xg_stencil_chain_host_connected(*args.values())


def _einval(rc, text):
    assert rc == -1, (rc, _capi.last_error())
    assert text in _capi.last_error(), _capi.last_error()


def test_symbols_exported(lib):
    for name in ("xg_stencil_chain_host_fold", "xg_stencil_chain_host_connected"):
        assert hasattr(lib, name) and name in _capi.SIGNATURES


def test_fold_validation_without_gpu(lib):
    a = (C.c_float * 512)()
    _einval(_fold(lib, inp=None), "null pointer")
    _einval(_fold(lib, fill=None), "null pointer")
    _einval(_fold(lib, fold=None), "null pointer")
    _einval(_fold(lib, dtype=7), "dtype")
    _einval(_fold(lib, ndim=0), "bad ndim")
    _einval(_fold(lib, out=a, inp=a), "in-place")
    _einval(_fold(lib, nstage=1, axis=[3], op=[0], lo=[1], hi=[0]), "2 or 3 stages")
    _einval(_fold(lib, nstage=4, axis=[3, 2, 1, 0], op=[0] * 4, lo=[0] * 4, hi=[1] * 4, bc=[2] * 4, fill=[0.0] * 4,
                  fold=[0] * 4, seam=[0] * 4, skip=[0] * 4, mirror=[0] * 4, period=[1] * 4), "2 or 3 stages")
    _einval(_fold(lib, axis=[3, 4]), "axis out of range")
    _einval(_fold(lib, axis=[0, 2]), "dim 0")  # a stage along the slab dim
    _einval(_fold(lib, axis=[2, 2], fold=[0, 0]), "only once")
    _einval(_fold(lib, op=[0, 9]), "unknown op")
    _einval(_fold(lib, hi=[0, 2]), "halo widths")
    _einval(_fold(lib, bc=[0, 2]), "no boundary condition")  # stage 0 pads X
    _einval(_fold(lib, shape=[4, 3, -6, 5]), "negative extent")
    _einval(_fold(lib, fold=[0, 2]), "fold must be 0 or 1")
    _einval(_fold(lib, seam=[0, 0]), "seam dim")  # the seam would be cut into slabs
    _einval(_fold(lib, seam=[0, 2]), "must differ")
    _einval(_fold(lib, seam=[0, 7]), "seam axis out of range")
    _einval(_fold(lib, skip=[0, 2]), "skip")
    _einval(_fold(lib, period=[1, 0]), "period")
    _einval(_fold(lib, lo=[1, 1], hi=[0, 0]), "hi must be 1")
    _einval(_fold(lib, device=_capi.XG_HOST_GROUP_BASE + 63), "unknown host device group")
    # the fold of stage 1 is checked against ITS input: X inner (5 -> 4 columns) leaves the mirror partner of seam
    # index 1 (column 4) outside; against the field's 5 columns it would pass
    rc = _fold(lib, lo=[0, 0], hi=[0, 1], bc=[0, 2])
    assert rc == -2 and "incompatible" in _capi.last_error(), (rc, _capi.last_error())


def test_connected_validation_without_gpu(lib):
    a = (C.c_float * 512)()
    _einval(_connected(lib, inp=None), "null pointer")
    _einval(_connected(lib, ncopies=None), "null pointer")
    _einval(_connected(lib, out=a, inp=a), "in-place")
    _einval(_connected(lib, nstage=1), "2 or 3 stages")
    _einval(_connected(lib, nstage=4), "2 or 3 stages")
    _einval(_connected(lib, axis=_i32([0, 2])), "dim 0")
    _einval(_connected(lib, axis=_i32([3, 3])), "only once")
    _einval(_connected(lib, lo=_i32([2, 0])), "halo widths")
    _einval(_connected(lib, programs=(STAGE0, STAGE1), ncopies=_i32([2, -1])), "negative copy count")
    _einval(_connected(lib, side=None), "null pointer in the copy list")
    _einval(_connected(lib, programs=(STAGE0, [_copy(0)])), "stage 1: copy 0: writes a halo plane the call does not")
    # the copies of stage 1 are described for ITS input, (4, 3, 6, 6): rows of 108, planes of 18
    _einval(_connected(lib, programs=(STAGE0, [_copy(1, source=0, soff=30, sstr=(ROW0, 30, 1))])), "span dim 0")
    _einval(_connected(lib, programs=(STAGE0, [_copy(1, source=0, soff=31, sstr=(ROW1, 36, 1))])),
            "leaves its source array")
    _einval(_connected(lib, programs=(STAGE0, [_copy(1, shape=(4, 3, 5))])), "stage 1: the copies do not cover")
    _einval(_connected(lib, programs=(STAGE0[:1], STAGE1)), "stage 0: the copies do not cover")
    _einval(_connected(lib, programs=(STAGE0, [])), "do not cover")
    _einval(_connected(lib, programs=(STAGE0, [_copy(1, source=1)])), "partner that was not given")
    _einval(_connected(lib, device=_capi.XG_HOST_GROUP_BASE + 63), "unknown host device group")


# ---------------------------------------------------------------------------------------------- Grid routing
def _stencil(x, axis, op, lo, hi, padding, fill, halo_lo=None, halo_hi=None):
    return ops.stencil2(torch.from_numpy(np.ascontiguousarray(x)), axis, op, lo, hi, padding, fill, halo_lo=halo_lo,
                        halo_hi=halo_hi).numpy()


def _chain_fold(x, stages, device=None):
    """The definition of xg_stencil_chain_host_fold (include/xgcm_b200.h), stage by stage."""
    a = np.asarray(x)
    for axis, op, lo, hi, padding, fill, plan in stages:
        hl = hh = None
        if plan is not None:
            hh = fold_rows(torch.from_numpy(np.ascontiguousarray(a)), axis, plan[0], 1, *plan[1:])
            hl = hh if lo and padding == "periodic" else None
        a = _stencil(a, axis, op, lo, hi, padding, fill, hl, hh)
    return a


def _chain_connected(x, stages, programs, device=None):
    """The definition of xg_stencil_chain_host_connected: each stage's copy list replayed on its input."""
    a = np.asarray(x)
    for (axis, op, lo, hi, fill), program in zip(stages, programs):
        p_shape = list(a.shape)
        p_shape[axis] = 1
        planes = [np.full(p_shape, np.inf, a.dtype), np.full(p_shape, np.inf, a.dtype)]
        srcs = {"self": a.ravel(), "fill": np.array([fill], a.dtype)}
        for side, doff, dstr, src, soff, sstr, shp, neg in program:
            assert shp[0] == a.shape[0] and src != "partner"
            idx = np.indices(shp).reshape(len(shp), -1)
            v = srcs[src][soff + (np.asarray(sstr)[:, None] * idx).sum(0)]
            planes[side].reshape(-1)[doff + (np.asarray(dstr)[:, None] * idx).sum(0)] = -v if neg else v
        hl, hh = (torch.from_numpy(planes[0]) if lo else None), (torch.from_numpy(planes[1]) if hi else None)
        a = _stencil(a, axis, op, lo, hi, "fill" if (lo or hi) else None, fill, hl, hh)
    return a


@pytest.fixture
def spy(monkeypatch):
    """Oracle-backed ops on a grid device of type cuda (the whole-field route's upload stays on the CPU), with the
    names of the chain entry points each call ran."""
    install_fold(monkeypatch)
    monkeypatch.setattr(device, "default_device", lambda: torch.device("cuda"))
    monkeypatch.setattr(xg.DataArray, "to_device", lambda self, dev=None: self._replace(
        data=torch.from_numpy(np.ascontiguousarray(self.data))))
    ran = []
    for name, fn in (("stencil_chain_host_fold", _chain_fold), ("stencil_chain_host_connected", _chain_connected)):
        def wrapped(*a, _fn=fn, _name=name, **kw):
            ran.append(_name)
            return _fn(*a, **kw)

        monkeypatch.setattr(ops, name, wrapped)
    return ran


def _dev(da):
    return xg.DataArray(torch.from_numpy(np.ascontiguousarray(da.values)), dims=da.dims)


def _vals(x):
    return x.data.numpy() if isinstance(x.data, torch.Tensor) else np.asarray(x.data)


def _same_as_device(grid, op, da, axes, spy, ran, **kw):
    spy.clear()
    got = getattr(grid, op)(da, axes, **kw)
    assert spy == ran, (op, axes, kw, spy)
    want = getattr(grid, op)(_dev(da), axes, **kw)
    assert got.dims == want.dims, (got.dims, want.dims)
    np.testing.assert_array_equal(_vals(got), _vals(want), err_msg=f"{op} {axes} {kw}")


def _same_error(call, da, exc, match, spy):
    spy.clear()
    for arg in (da, _dev(da)):
        with pytest.raises(exc, match=match):
            call(arg)
    assert spy == []


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
    ds = xg.Dataset(data_vars={"c": (("t", "k", "face", "y", "x"), c)},
                    coords={"x": np.arange(N), "xl": np.arange(N), "xo": np.arange(N + 1), "y": np.arange(N),
                            "yl": np.arange(N), "yo": np.arange(N + 1), "k": np.arange(3), "kl": np.arange(3),
                            "face": np.arange(nf)})
    return ds, xg.Grid(ds, coords=COORDS, face_connections=fc)


@pytest.mark.parametrize("fc", [CUBED_SPHERE, STRIP], ids=["cubed_sphere", "strip"])
def test_faces_route_and_values(fc, spy):
    ds, grid = _faces(fc)
    c = ds["c"]
    for op, axes, (padding, fill) in itertools.product(
            ("diff", "interp", "min", "max"), (["X", "Y"], ["Y", "X"], ["X", "Y", "Z"]),
            [("fill", 1.5), ("extend", 0.0), ("periodic", 0.0)]):
        _same_as_device(grid, op, c, axes, spy, ["stencil_chain_host_connected"], padding=padding, fill_value=fill)
    # per-axis boundaries and fills, and a shift that changes the X extent on the strip (no seam swaps axes)
    _same_as_device(grid, "interp", c, ["Z", "X"], spy, ["stencil_chain_host_connected"],
                    padding={"X": "fill", "Y": "extend", "Z": "fill"}, fill_value={"X": 2.5, "Z": -1.0})
    if fc is STRIP:
        _same_as_device(grid, "diff", c, ["X", "Y"], spy, ["stencil_chain_host_connected"], to={"X": "outer"},
                        padding="periodic")


def test_faces_errors_and_whole_field_routes(spy):
    ds, grid = _faces(CUBED_SPHERE)
    c = ds["c"]
    # X outer makes the faces 7 x 6: the Y seams that swap axes need faces of equal size
    _same_error(lambda a: grid.diff(a, ["X", "Y"], to={"X": "outer"}, padding="fill"), c, ValueError, "equal size",
                spy)
    _same_error(lambda a: grid.interp(a, ["X", "Z"]), c, ValueError, "No boundary condition", spy)
    _same_error(lambda a: grid.interp(a, ["X", "Y"], to={"Y": "right"}), c, ValueError, "does not exist", spy)
    ds2, strip = _faces(STRIP)
    _same_error(lambda a: strip.interp(a, ["Y", "X"]), ds2["c"], ValueError, "No boundary condition", spy)
    _same_error(lambda a: grid.interp(a, ["X", "Y"], padding="extrapolate"), c, NotImplementedError, "extrapolate",
                spy)
    # no batch dim in front of the face dim: the whole-field route
    t = xg.DataArray(np.ascontiguousarray(np.moveaxis(c.values, 2, 0)), dims=("face", "t", "k", "y", "x"))
    _same_as_device(grid, "interp", t, ["X", "Y"], spy, [], padding="extend")
    # a device tensor keeps the per-axis launches, and so does a vector component
    assert grid._multi_axis_halo_host("interp", _dev(c), ["X", "Y"], {}, {}) is None
    _same_error(lambda a: grid.interp(a, ["X", "Y"], padding="extend", other_component={"Y": c}), c, ValueError,
                "unambiguously", spy)
    assert spy == []


NX, NY = 8, 7
POS = ("center", "left", "right", "outer", "inner")
EXTRA = {"center": 0, "left": 0, "right": 0, "outer": 1, "inner": -1}


def _fold_grid(pivot, south):
    coords = {"x" + p: np.arange(NX + EXTRA[p]) for p in POS}
    coords.update({"y" + p: np.arange(NY + EXTRA[p]) for p in POS})
    coords.update({"zcenter": np.arange(3), "zleft": np.arange(3)})
    ds = xg.Dataset(data_vars={}, coords=coords)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        return xg.Grid(ds, coords={"X": {p: "x" + p for p in POS}, "Y": {p: "y" + p for p in POS},
                                   "Z": {"center": "zcenter", "left": "zleft"}},
                       padding={"X": "periodic", "Y": {"fold": pivot, "south": south}, "Z": "extend"},
                       autoparse_metadata=False)


def _fold_field(ysrc, xsrc, lead=(2, 3), seed=2):
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(lead + (NY + EXTRA[ysrc], NX + EXTRA[xsrc]))
    a[rng.random(a.shape) < 0.1] = np.nan
    return xg.DataArray(a, dims=("t", "zcenter")[2 - len(lead):] + ("y" + ysrc, "x" + xsrc))


@pytest.mark.parametrize("pivot", ["T", "F", "U", "V"])
def test_fold_route_and_values(pivot, spy):
    for south in ("fill", "periodic", "extend"):
        grid = _fold_grid(pivot, south)
        for (ysrc, yto), xto, axes, op in itertools.product(
                [("center", "right"), ("left", "center"), ("center", "outer")], ("left", "right"),
                (["X", "Y"], ["Y", "X"], ["X", "Y", "Z"]), ("diff", "interp", "min", "max")):
            da = _fold_field(ysrc, "center")
            _same_as_device(grid, op, da, axes, spy, ["stencil_chain_host_fold"], to={"X": xto, "Y": yto})
        # a fill per axis; Y center -> left pads the south edge alone: no fold, the fused route
        da = _fold_field("center", "center")
        _same_as_device(grid, "interp", da, ["Y", "X"], spy, ["stencil_chain_host_fold"], to={"Y": "right"},
                        padding={"X": "fill", "Y": "fill"}, fill_value={"X": 1.5, "Y": -2.0})


def test_fold_errors_and_whole_field_routes(spy):
    grid = _fold_grid("T", "fill")
    da = _fold_field("center", "center")
    _same_error(lambda a: grid.interp(a, ["Y", "Z"], to={"Y": "right", "Z": "right"}), da, ValueError, "does not exist", spy)
    # no batch dim in front: a 2-D field, and (1, Z, Y, X) with Z operated
    flat = _fold_field("center", "center", lead=())
    _same_as_device(grid, "interp", flat, ["X", "Y"], spy, [], to={"Y": "right"})
    one = _fold_field("center", "center", lead=(1, 3))
    _same_as_device(grid, "interp", one, ["X", "Y", "Z"], spy, [], to={"Y": "right"})
    # extrapolate along X, and a fold the plan cannot mirror (an inner seam under a center-type pivot)
    assert grid._multi_axis_halo_host("interp", da, ["X", "Y"], {"Y": "right"}, {"padding": {"X": "extrapolate"}}) \
        is None
    with pytest.raises(NotImplementedError):
        grid.interp(_dev(da), ["X", "Y"], to={"X": "inner", "Y": "right"})
    spy.clear()
    with pytest.raises(NotImplementedError):
        grid.interp(da, ["X", "Y"], to={"X": "inner", "Y": "right"})
    assert spy == []
