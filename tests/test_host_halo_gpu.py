"""Numpy fields on face-connected and north-fold grids stream through the host slab pipelines
(xg_stencil2_host_connected / xg_stencil2_host_fold): bit for bit equal to the same call on device tensors
and to the oracles, with device memory bounded by the slab size.  XG_HOST_SLAB_MB=1 forces at least four
slabs with a ragged last one."""

import itertools
import warnings

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from oracle import fold as F
from oracle import stencil as S
from oracle.faces import pad_face_connections
from xgcm_b200 import _capi

pytestmark = pytest.mark.gpu

N = 48
LEAD = (3, 5)  # (time, k): 15 slab rows of 6 x 48 x 48 cells -> slabs of 4, 4, 4, 3 at 1 MiB
COORDS = {"X": {"center": "x", "left": "xl"}, "Y": {"center": "y", "left": "yl"}}
AXES = {"X": ("x", "xl"), "Y": ("y", "yl")}
# xgcm/test/test_faceconnections.py:99-127: same-axis, swapped and reversed seams
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
# two faces side by side along X: the outer X edges and both Y edges are unconnected
STRIP = {"face": {0: {"X": (None, (1, "X", False))}, 1: {"X": ((0, "X", False), None)}}}


@pytest.fixture(autouse=True)
def slab(monkeypatch):
    monkeypatch.setenv("XG_HOST_SLAB_MB", "1")


def _launches():
    return _capi.load().xg_launch_count()


def _workspace_bytes():
    v = _capi.i64_array([0])
    _capi.check(_capi.load().xg_host_workspace_bytes(0, v))
    return int(v[0])


def _on_device(da):
    return xg.DataArray(torch.from_numpy(np.ascontiguousarray(da.values)).to("cuda:0"), dims=da.dims)


def _host(x):
    return x.data.cpu().numpy() if isinstance(x.data, torch.Tensor) else np.asarray(x.data)


def _faces_grid(dtype, lead=LEAD, lead_dims=("time", "k"), fc=CUBED_SPHERE, seed=0):
    rng = np.random.default_rng(seed)
    nf = len(fc["face"])
    shape = lead + (nf, N, N)
    coords = {"x": np.arange(N) + 0.0, "xl": np.arange(N) - 0.5, "y": np.arange(N) + 0.0,
              "yl": np.arange(N) - 0.5, "face": np.arange(nf),
              "dx_l": (("face", "y", "xl"), 1.0 + rng.random((nf, N, N))),
              "dx_c": (("face", "y", "x"), 1.0 + rng.random((nf, N, N)))}
    ds = xg.Dataset(data_vars={
        "c": (lead_dims + ("face", "y", "x"), rng.standard_normal(shape).astype(dtype)),
        "u": (lead_dims + ("face", "y", "xl"), rng.standard_normal(shape).astype(dtype)),
        "v": (lead_dims + ("face", "yl", "x"), rng.standard_normal(shape).astype(dtype))}, coords=coords)
    return ds, xg.Grid(ds, coords=COORDS, face_connections=fc, metrics={("X",): ["dx_c", "dx_l"]})


def _faces_oracle(op, da, fc, ax, lo, hi, padding, fill, vector_axis=None, partner=None, post=None):
    padded = pad_face_connections(
        da.values, da.dims, AXES, "face", fc["face"], {ax: (lo, hi)}, {a: padding for a in AXES},
        {a: fill for a in AXES}, vector_axis=vector_axis, partner=None if partner is None else partner.values,
        partner_dims=None if partner is None else partner.dims)
    k = [d for d in da.dims if d in AXES[ax]][0]
    r = S.stencil2(op, padded, da.dims.index(k), 0, 0, None)
    return r if post is None else r / post


def _same(got, dev, want, msg):
    got = _host(got)
    assert isinstance(got, np.ndarray) and got.dtype == want.dtype
    np.testing.assert_array_equal(got, _host(dev), err_msg=msg)
    np.testing.assert_array_equal(got, want.astype(got.dtype), err_msg=msg)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_faces_every_op_shift_and_padding(dtype):
    ds, grid = _faces_grid(dtype)
    c, u, v = ds["c"], ds["u"], ds["v"]
    checked = 0
    for (padding, fill), ax in itertools.product(
            [("fill", 0.0), ("fill", 1.5), ("fill", np.nan), ("extend", 0.0), ("periodic", 0.0)], ("X", "Y")):
        kw = dict(padding=padding, fill_value=fill)
        left = {"X": "xl", "Y": "yl"}[ax]
        for op in ("diff", "interp", "min", "max"):
            # center -> left (lower halo) on the scalar, left -> center (upper halo) on a vector component
            got = getattr(grid, op)(c, ax, **kw)
            dev = getattr(grid, op)(_on_device(c), ax, **kw)
            _same(got, dev, _faces_oracle(op, c, CUBED_SPHERE, ax, 1, 0, padding, fill), f"{op} {ax} {padding}")
            comp, other = (u, v) if ax == "X" else (v, u)
            oax = "Y" if ax == "X" else "X"
            got = getattr(grid, op)({ax: comp}, ax, other_component={oax: other}, **kw)
            dev = getattr(grid, op)({ax: _on_device(comp)}, ax, other_component={oax: _on_device(other)}, **kw)
            assert left in comp.dims
            _same(got, dev, _faces_oracle(op, comp, CUBED_SPHERE, ax, 0, 1, padding, fill, ax, other),
                  f"vector {op} {ax} {padding}")
            checked += 2
        # a bare component with other_component (its axis inferred from its position)
        comp, other, oax = (u, v, "Y") if ax == "X" else (v, u, "X")
        got = grid.diff(comp, ax, other_component={oax: other}, **kw)
        _same(got, grid.diff(_on_device(comp), ax, other_component={oax: _on_device(other)}, **kw),
              _faces_oracle("diff", comp, CUBED_SPHERE, ax, 0, 1, padding, fill, ax, other), f"bare {ax}")
    assert checked == 80
    # derivative: the post metric divides each slab
    dx_l = ds["dx_l"].values.astype(dtype)  # metrics are rounded to the field's dtype
    got = grid.derivative(c, "X")
    _same(got, grid.derivative(_on_device(c), "X"),
          _faces_oracle("diff", c, CUBED_SPHERE, "X", 1, 0, None, 0.0, post=dx_l), "derivative")


@pytest.mark.parametrize("padding", ["fill", "extend", "periodic"])
def test_faces_unconnected_edges(padding):
    ds, grid = _faces_grid(np.float32, fc=STRIP)
    c = ds["c"]
    for ax, (lo, hi) in itertools.product(("X", "Y"), ((1, 0),)):
        got = grid.interp(c, ax, padding=padding, fill_value=1.5)
        _same(got, grid.interp(_on_device(c), ax, padding=padding, fill_value=1.5),
              _faces_oracle("interp", c, STRIP, ax, lo, hi, padding, 1.5), f"{ax} {padding}")


def test_faces_streaming_happened():
    ds, grid = _faces_grid(np.float32, lead=(1, 30), lead_dims=("one", "k"))  # (1, k, face, j, i)
    c = ds["c"].values
    field = xg.DataArray(c, dims=ds["c"].dims)
    _capi.check(_capi.load().xg_host_workspace_release())
    grid.diff(field, "X", padding="fill")  # warm-up: workspace and plan
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    n0 = _launches()
    got = grid.diff(field, "X", padding="fill")
    n_slabs = -(-30 // 8)  # 30 rows of 6 x 48 x 48 fp32 (55 KiB): min(18, ceil(30 / 4)) = 8 rows per slab
    assert _launches() - n0 >= 2 * n_slabs  # halo copies + stencil per slab
    assert torch.cuda.max_memory_allocated() - base < c.nbytes // 4
    row = 6 * N * N * 4
    assert _workspace_bytes() <= 3 * 2 * 8 * row + 2 * 8 * 6 * N * 4 + 8  # slots + planes + fill constant
    want = _faces_oracle("diff", ds["c"], CUBED_SPHERE, "X", 1, 0, "fill", 0.0)
    np.testing.assert_array_equal(_host(got), want)


def test_faces_fallback_layouts_unchanged():
    """(face, k, j, i) and metric_weighted keep the whole-field device path and its values."""
    ds, grid = _faces_grid(np.float64, lead=(4,), lead_dims=("k",))
    c = ds["c"].transpose("face", "k", "y", "x")
    got = grid.diff(c, "X", padding="extend")
    dev = grid.diff(_on_device(c), "X", padding="extend")
    np.testing.assert_array_equal(_host(got), _host(dev))
    c = ds["c"]
    got = grid.interp(c, "X", metric_weighted="X")
    dev = grid.interp(_on_device(c), "X", metric_weighted="X")
    np.testing.assert_array_equal(_host(got), _host(dev))
    weighted = xg.DataArray(c.values * ds["dx_c"].values, dims=c.dims)
    np.testing.assert_array_equal(
        _host(got), _faces_oracle("interp", weighted, CUBED_SPHERE, "X", 1, 0, None, 0.0, post=ds["dx_l"].values))


# ------------------------------------------------------------------ north fold
NX, NY = 40, 33
POS = ("center", "left", "right", "outer", "inner")
EXTRA = {"center": 0, "left": 0, "right": 0, "outer": 1, "inner": -1}
XD = {p: "x" + p for p in POS}
YD = {p: "y" + p for p in POS}
PIVOTS = ["center", "corner", "U", "V", {"X": "right", "Y": "center"}]
FLEAD = (5, 6)  # (time, z): 30 rows of ~5 KiB -> ceil(30 / 8) = 4 slabs, the last ragged


def _fold_grid(south, pivot, dtype, seed=0):
    rng = np.random.default_rng(seed)
    coords = {XD[p]: np.arange(NX + EXTRA[p]) for p in POS}
    coords.update({YD[p]: np.arange(NY + EXTRA[p]) for p in POS})
    data = {f"dy_{p}": ((YD[p], "xcenter"), 0.5 + rng.random((NY + EXTRA[p], NX)).astype(dtype)) for p in POS}
    data.update({f"area_{p}": ((YD[p], "xcenter"), 0.5 + rng.random((NY + EXTRA[p], NX)).astype(dtype))
                 for p in POS})
    ds = xg.Dataset(data_vars=data, coords=coords)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        grid = xg.Grid(ds, coords={"X": dict(XD), "Y": dict(YD)},
                       padding={"X": "periodic", "Y": {"fold": pivot, "south": south}}, autoparse_metadata=False)
    grid.set_metrics("Y", [f"dy_{p}" for p in POS])
    grid.set_metrics(("X", "Y"), [f"area_{p}" for p in POS])
    return ds, grid


def _fold_oracle(op, a, ypos, xpos, pivot, lo, hi, south, vector=False, pre=None, post=None):
    x = a if pre is None else a * pre
    fa = a.ndim - 2
    padded = F.pad_fold(x, fa, fa + 1, ypos, xpos, F.resolve_pivot(pivot, "Y", "X"), {fa: (lo, hi)}, {fa: south},
                        vector=vector)
    r = S.stencil2(op, padded, fa, 0, 0, None)
    return r if post is None else r / post


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_fold_every_pivot_op_and_south_edge(dtype):
    rng = np.random.default_rng(1)
    checked = 0
    for pivot, south in itertools.product(PIVOTS, ("fill", "periodic", "extend")):
        ds, grid = _fold_grid(south, pivot, dtype)
        roles = F.resolve_pivot(pivot, "Y", "X")
        for xpos, (src, dst) in itertools.product(("center", "left", "outer", "inner"),
                                                  [("left", "center"), ("center", "right"), ("inner", "center"),
                                                   ("center", "outer")]):
            if xpos == "inner" and roles["seam"] == "center":
                continue
            lo, hi = S.PADDING_WIDTH[(src, dst)]
            if not hi:
                continue
            a = rng.standard_normal(FLEAD + (NY + EXTRA[src], NX + EXTRA[xpos])).astype(dtype)
            da = xg.DataArray(a, dims=("time", "z", YD[src], XD[xpos]))
            for op, vector in itertools.product(("diff", "interp", "min", "max"), (False, True)):
                arg = {"Y": da} if vector else da
                got = getattr(grid, op)(arg, "Y", to=dst)
                dev_arg = {"Y": _on_device(da)} if vector else _on_device(da)
                dev = getattr(grid, op)(dev_arg, "Y", to=dst)
                want = _fold_oracle(op, a, src, xpos, pivot, lo, hi, south, vector)
                _same(got, dev, want, f"{pivot} {south} {op} {src}->{dst} x{xpos} {vector}")
                checked += 1
    assert checked > 300


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_fold_metrics(dtype):
    rng = np.random.default_rng(2)
    for pivot, south in (("corner", "periodic"), ("U", "fill"), ("center", "extend")):
        ds, grid = _fold_grid(south, pivot, dtype)
        for src, dst in (("left", "center"), ("center", "right")):
            lo, hi = S.PADDING_WIDTH[(src, dst)]
            a = rng.standard_normal(FLEAD + (NY + EXTRA[src], NX)).astype(dtype)
            da = xg.DataArray(a, dims=("time", "z", YD[src], "xcenter"))
            got = grid.derivative(da, "Y", to=dst)
            _same(got, grid.derivative(_on_device(da), "Y", to=dst),
                  _fold_oracle("diff", a, src, "center", pivot, lo, hi, south, post=ds[f"dy_{dst}"].values), "der")
            got = grid.interp(da, "Y", to=dst, metric_weighted=["X", "Y"])
            dev = grid.interp(_on_device(da), "Y", to=dst, metric_weighted=["X", "Y"])
            want = _fold_oracle("interp", a, src, "center", pivot, lo, hi, south, pre=ds[f"area_{src}"].values,
                                post=ds[f"area_{dst}"].values)
            _same(got, dev, want, f"metric_weighted {pivot} {src}->{dst}")


def test_fold_streaming_happened():
    ds, grid = _fold_grid("periodic", "corner", np.float32)
    a = np.random.default_rng(3).standard_normal((12, 20, NY, NX)).astype(np.float32)
    da = xg.DataArray(a, dims=("time", "z", "yleft", "xcenter"))
    _capi.check(_capi.load().xg_host_workspace_release())
    grid.diff(da, "Y", to="center")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    n0 = _launches()
    got = grid.diff(da, "Y", to="center")
    rows = min((1 << 20) // (NY * NX * 4), -(-240 // 4))
    n_slabs = -(-240 // rows)
    assert n_slabs >= 4
    assert _launches() - n0 >= 2 * n_slabs  # fold row + stencil per slab
    assert torch.cuda.max_memory_allocated() - base < a.nbytes // 4
    plane = rows * NX * 4
    assert _workspace_bytes() <= 3 * 2 * rows * NY * NX * 4 + 2 * plane  # slots + planes
    np.testing.assert_array_equal(_host(got), _fold_oracle("diff", a, "left", "center", "corner", 0, 1, "periodic"))


def test_plain_grid_drops_leading_size_one_dims():
    """(1, Z, Y, X) on a plain grid is cut along Z, not sent whole as one slab."""
    ds, grid = _fold_grid("periodic", "corner", np.float64)
    a = np.random.default_rng(4).standard_normal((1, 64, NY, NX))
    da = xg.DataArray(a, dims=("one", "z", "ycenter", "xcenter"))
    grid.diff(da, "X")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    n0 = _launches()
    got = grid.diff(da, "X")
    assert _launches() - n0 >= 4
    assert torch.cuda.max_memory_allocated() - base < a.nbytes // 4
    np.testing.assert_array_equal(_host(got), S.stencil2("diff", a, 3, 1, 0, "periodic"))
