"""Multi-axis Grid.diff / interp / min / max of numpy fields on face-connected and north-fold grids stream through the
host slab pipelines (xg_stencil_chain_host_connected / xg_stencil_chain_host_fold): bit for bit equal to the same
call on device tensors and to the oracle's per-axis composition (pad across the faces or the fold, then the stencil,
one axis after another), with device memory bounded by the slab size.  XG_HOST_SLAB_MB=1 forces at least four slabs
with a ragged last one."""

import itertools
import warnings

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from oracle import fold as F
from oracle import stencil as S
from oracle.faces import pad_face_connections
from xgcm_b200 import _capi, ops

pytestmark = pytest.mark.gpu

OPS = ("diff", "interp", "min", "max")
ORDERS = (["X", "Y"], ["Y", "X"], ["X", "Y", "Z"])


@pytest.fixture(autouse=True)
def slab(monkeypatch):
    monkeypatch.setenv("XG_HOST_SLAB_MB", "1")


@pytest.fixture
def spy(monkeypatch):
    """Names of the streamed chain entry points each call ran."""
    ran = []
    for name in ("stencil_chain_host_fold", "stencil_chain_host_connected"):
        fn = getattr(ops, name)

        def wrapped(*a, _fn=fn, _name=name, **kw):
            ran.append(_name)
            return _fn(*a, **kw)

        monkeypatch.setattr(ops, name, wrapped)
    return ran


def _workspace_bytes():
    v = _capi.i64_array([0])
    _capi.check(_capi.load().xg_host_workspace_bytes(0, v))
    return int(v[0])


def _on_device(da):
    return xg.DataArray(torch.from_numpy(np.ascontiguousarray(da.values)).to("cuda:0"), dims=da.dims)


def _host(x):
    return x.data.cpu().numpy() if isinstance(x.data, torch.Tensor) else np.asarray(x.data)


def _same(got, dev, want, msg):
    got = _host(got)
    assert isinstance(got, np.ndarray) and got.dtype == want.dtype, msg
    np.testing.assert_array_equal(got, _host(dev), err_msg=msg)
    np.testing.assert_array_equal(got, want, err_msg=msg)


# ------------------------------------------------------------------ face connections
N = 48
LEAD = (3, 5)  # (time, k): 15 slab rows of 6 x 48 x 48 cells -> slabs of 4, 4, 4, 3 at 1 MiB
COORDS = {"X": {"center": "x", "left": "xl"}, "Y": {"center": "y", "left": "yl"}, "Z": {"center": "k", "left": "kl"}}
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
PADDINGS = [("fill", 0.0), ("fill", 1.5), ("fill", np.nan), ("extend", 0.0), ("periodic", 0.0)]


def _faces_grid(dtype, fc=CUBED_SPHERE, lead=LEAD, lead_dims=("time", "k"), seed=0, nan=True):
    rng = np.random.default_rng(seed)
    nf = len(fc["face"])
    shape = lead + (nf, N, N)
    c = rng.standard_normal(shape).astype(dtype)
    if nan:
        c[rng.random(shape) < 0.05] = np.nan
    coords = {"x": np.arange(N) + 0.0, "xl": np.arange(N) - 0.5, "y": np.arange(N) + 0.0, "yl": np.arange(N) - 0.5,
              "face": np.arange(nf), "k": np.arange(lead[-1]) + 0.0, "kl": np.arange(lead[-1]) - 0.5}
    ds = xg.Dataset(data_vars={"c": (lead_dims + ("face", "y", "x"), c)}, coords=coords)
    return ds, xg.Grid(ds, coords=COORDS, face_connections=fc)


def _faces_oracle(op, da, fc, axes, paddings, fills):
    """Each axis in turn, center -> left: pad (across the faces for X / Y, the basic boundary for Z), then the
    stencil."""
    a, dims = da.values, list(da.dims)
    for ax in axes:
        if ax == "Z":
            a = S.stencil2(op, a, dims.index("k"), 1, 0, paddings["Z"], fills.get("Z", 0.0))
            dims[dims.index("k")] = "kl"
            continue
        a = pad_face_connections(a, tuple(dims), AXES, "face", fc["face"], {ax: (1, 0)},
                                 {k: paddings[k] for k in AXES}, {k: fills.get(k, 0.0) for k in AXES})
        d = dims.index(AXES[ax][0])
        a = S.stencil2(op, a, d, 0, 0, None)
        dims[d] = AXES[ax][1]
    return a


@pytest.mark.parametrize("fc", [CUBED_SPHERE, STRIP], ids=["cubed_sphere", "strip"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_faces_every_op_order_and_padding(fc, dtype, spy):
    ds, grid = _faces_grid(dtype, fc=fc)
    c = ds["c"]
    checked = 0
    for op, axes, (padding, fill) in itertools.product(OPS, ORDERS, PADDINGS):
        kw = dict(padding=padding, fill_value=fill)
        spy.clear()
        got = getattr(grid, op)(c, axes, **kw)
        assert spy == ["stencil_chain_host_connected"], (op, axes, padding)
        dev = getattr(grid, op)(_on_device(c), axes, **kw)
        want = _faces_oracle(op, c, fc, axes, {a: padding for a in "XYZ"}, {a: fill for a in "XYZ"})
        _same(got, dev, want, f"{op} {axes} {padding} {fill}")
        checked += 1
    assert checked == len(OPS) * len(ORDERS) * len(PADDINGS)


@pytest.mark.parametrize("fc", [CUBED_SPHERE, STRIP], ids=["cubed_sphere", "strip"])
def test_faces_fill_per_axis(fc, spy):
    ds, grid = _faces_grid(np.float32, fc=fc)
    c = ds["c"]
    paddings, fills = {"X": "fill", "Y": "fill", "Z": "fill"}, {"X": 2.5, "Y": np.nan, "Z": -1.0}
    for axes in (["Z", "X", "Y"], ["Y", "Z"]):
        spy.clear()
        got = grid.interp(c, axes, padding=paddings, fill_value=fills)
        assert spy == ["stencil_chain_host_connected"]
        _same(got, grid.interp(_on_device(c), axes, padding=paddings, fill_value=fills),
              _faces_oracle("interp", c, fc, axes, paddings, fills), f"{axes}")


def test_faces_errors_and_whole_field_layouts(spy):
    ds, grid = _faces_grid(np.float64)
    c = ds["c"]
    for arg in (c, _on_device(c)):
        with pytest.raises(ValueError, match="No boundary condition"):
            grid.interp(arg, ["X", "Z"])
    ds2, strip = _faces_grid(np.float64, fc=STRIP)
    for arg in (ds2["c"], _on_device(ds2["c"])):
        with pytest.raises(ValueError, match="No boundary condition"):
            strip.diff(arg, ["Y", "X"])
    assert spy == []
    # no batch dim in front of the face dim: the whole-field route, same values
    t = c.transpose("face", "time", "k", "y", "x")
    t = xg.DataArray(np.ascontiguousarray(t.values), dims=t.dims)
    got = grid.diff(t, ["X", "Y"], padding="extend")
    assert spy == []
    np.testing.assert_array_equal(_host(got), _host(grid.diff(_on_device(t), ["X", "Y"], padding="extend")))


def test_faces_streaming_is_bounded_by_the_slab():
    ds, grid = _faces_grid(np.float32, lead=(1, 30), lead_dims=("one", "k"), nan=False)  # (1, k, face, j, i)
    c = ds["c"]
    _capi.check(_capi.load().xg_host_workspace_release())
    grid.interp(c, ["X", "Y"])  # warm-up: workspace and plan
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    got = grid.interp(c, ["X", "Y"])
    assert torch.cuda.max_memory_allocated() - base < c.values.nbytes // 4
    row, plane = 6 * N * N * 4, 6 * N * 4
    rows = min((1 << 20) // (3 * row), -(-30 // 4))  # a slab row moves the input, the intermediate and the result
    assert -(-30 // rows) >= 4
    assert _workspace_bytes() <= rows * (3 * 2 * row + row + 2 * plane) + 16  # slots, intermediate, planes, fills
    want = _faces_oracle("interp", c, CUBED_SPHERE, ["X", "Y"], {"X": "fill", "Y": "fill"}, {})
    np.testing.assert_array_equal(_host(got), want)


# ------------------------------------------------------------------ north fold
NX, NY = 40, 33
POS = ("center", "left", "right", "outer")
EXTRA = {"center": 0, "left": 0, "right": 0, "outer": 1}
XD = {p: "x" + p for p in POS}
YD = {p: "y" + p for p in POS}
PIVOTS = ["T", "F", "U", "V"]
FLEAD = (5, 6)  # (time, z): 30 rows of ~5 KiB each -> at least 4 slabs, the last ragged
DEFAULT = {"center": "left", "left": "center", "right": "center", "outer": "center"}


def _fold_grid(south, pivot, dtype, host_devices=None, seed=0):
    rng = np.random.default_rng(seed)
    coords = {XD[p]: np.arange(NX + EXTRA[p]) for p in POS}
    coords.update({YD[p]: np.arange(NY + EXTRA[p]) for p in POS})
    coords.update({"zc": np.arange(FLEAD[1]) + 0.5, "zl": np.arange(FLEAD[1]) + 0.0})
    data = {f"dy_{p}": ((YD[p], "xcenter"), 0.5 + rng.random((NY + EXTRA[p], NX)).astype(dtype)) for p in POS}
    ds = xg.Dataset(data_vars=data, coords=coords)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        grid = xg.Grid(ds, coords={"X": dict(XD), "Y": dict(YD), "Z": {"center": "zc", "left": "zl"}},
                       padding={"X": "periodic", "Y": {"fold": pivot, "south": south}, "Z": "extend"},
                       autoparse_metadata=False, host_devices=host_devices)
    grid.set_metrics("Y", [f"dy_{p}" for p in POS])
    return ds, grid


def _fold_field(ysrc, dtype, seed=1, lead=FLEAD, nan=True):
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(lead + (NY + EXTRA[ysrc], NX)).astype(dtype)
    if nan:
        a[rng.random(a.shape) < 0.05] = np.nan
    return xg.DataArray(a, dims=("time", "zc")[2 - len(lead):] + (YD[ysrc], "xcenter"))


def _fold_oracle(op, da, axes, to, pivot, south, fills=None):
    """Each axis in turn: X periodic, Y across the fold (its south edge ``south``), Z extend."""
    fills = fills or {}
    a = da.values
    ya, xa = a.ndim - 2, a.ndim - 1
    pos = {"Y": da.dims[ya][1:], "X": da.dims[xa][1:]}
    roles = F.resolve_pivot(pivot, "Y", "X")
    for ax in axes:
        if ax == "Z":
            a = S.stencil2(op, a, ya - 1, 1, 0, "extend")
            continue
        dst = to.get(ax) or DEFAULT[pos[ax]]
        lo, hi = S.PADDING_WIDTH[(pos[ax], dst)]
        if ax == "X":
            a = S.stencil2(op, a, xa, lo, hi, "periodic")
        else:
            padded = F.pad_fold(a, ya, xa, pos["Y"], pos["X"], roles, {ya: (lo, hi)}, {ya: south},
                                {ya: fills.get("Y", 0.0)})
            a = S.stencil2(op, padded, ya, 0, 0, None)
        pos[ax] = dst
    return a


# (Y from, Y to, X to): every Y entry that pads the north edge, with X shifts that move the seam position before the
# fold stage (X first) or after it (Y first)
FOLD_CASES = [("center", "right", "left"), ("left", "center", "right"), ("center", "outer", "left"),
              ("center", "right", "right")]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_fold_every_pivot_op_order_and_shift(dtype, spy):
    checked = 0
    for pivot, south in itertools.product(PIVOTS, ("fill", "periodic", "extend")):
        ds, grid = _fold_grid(south, pivot, dtype)
        for (ysrc, yto, xto), axes, op in itertools.product(FOLD_CASES, ORDERS, OPS):
            da = _fold_field(ysrc, dtype)
            to = {"X": xto, "Y": yto}
            spy.clear()
            got = getattr(grid, op)(da, axes, to=to)
            assert spy == ["stencil_chain_host_fold"], (pivot, ysrc, yto, axes)
            dev = getattr(grid, op)(_on_device(da), axes, to=to)
            _same(got, dev, _fold_oracle(op, da, axes, to, pivot, south), f"{pivot} {south} {op} {axes} {to}")
            checked += 1
    assert checked == len(PIVOTS) * 3 * len(FOLD_CASES) * len(ORDERS) * len(OPS)


@pytest.mark.parametrize("fill", [0.0, 1.5, np.nan])
def test_fold_south_fill_values(fill, spy):
    ds, grid = _fold_grid("fill", "F", np.float32)
    da = _fold_field("center", np.float32)  # center -> outer pads the south edge with the fill, the north one folds
    for axes, to in ((["X", "Y"], {"Y": "outer"}), (["Y", "X"], {"Y": "outer", "X": "right"})):
        for kw in (dict(fill_value=fill), dict(fill_value={"Y": fill, "X": 7.0})):
            spy.clear()
            got = grid.interp(da, axes, to=to, padding={"Y": "fill"}, **kw)
            assert spy == ["stencil_chain_host_fold"]
            dev = grid.interp(_on_device(da), axes, to=to, padding={"Y": "fill"}, **kw)
            _same(got, dev, _fold_oracle("interp", da, axes, to, "F", "fill", {"Y": fill}), f"{axes} {kw}")


def test_fold_whole_field_routes(spy):
    ds, grid = _fold_grid("fill", "T", np.float64)
    da = _fold_field("center", np.float64)
    to = {"Y": "right"}
    # metric weighting, a 2-D field, and (1, Z, Y, X) with Z operated: the whole-field route, same values
    for arg, axes, kw in ((da, ["Y", "X"], dict(metric_weighted={"Y": ("Y",)})),
                          (_fold_field("center", np.float64, lead=()), ["X", "Y"], {}),
                          (_fold_field("center", np.float64, lead=(1, FLEAD[1])), ["X", "Y", "Z"], {})):
        spy.clear()
        got = grid.interp(arg, axes, to=to, **kw)
        assert spy == []
        np.testing.assert_array_equal(_host(got), _host(grid.interp(_on_device(arg), axes, to=to, **kw)))
    flat = _fold_field("center", np.float64, lead=())
    np.testing.assert_array_equal(_host(grid.interp(flat, ["X", "Y"], to=to)),
                                  _fold_oracle("interp", flat, ["X", "Y"], to, "T", "fill"))


def test_fold_streaming_is_bounded_by_the_slab():
    ds, grid = _fold_grid("periodic", "F", np.float32)
    a = _fold_field("center", np.float32, lead=(12, 20), nan=False).values
    da = xg.DataArray(a, dims=("time", "lev", "ycenter", "xcenter"))  # 20 levels: not the grid's Z
    to = {"Y": "right"}
    _capi.check(_capi.load().xg_host_workspace_release())
    grid.interp(da, ["X", "Y"], to=to)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    got = grid.interp(da, ["X", "Y"], to=to)
    assert torch.cuda.max_memory_allocated() - base < da.values.nbytes // 4
    row = NY * NX * 4
    rows = min((1 << 20) // (3 * row), -(-240 // 4))  # input, intermediate and result per slab row
    assert -(-240 // rows) >= 4
    assert _workspace_bytes() <= rows * (3 * 2 * row + row + 2 * NX * 4)  # slots, intermediate, planes
    np.testing.assert_array_equal(_host(got), _fold_oracle("interp", da, ["X", "Y"], to, "F", "periodic"))


# ------------------------------------------------------------------ host device groups
def _group_cases(host_devices):
    ds, grid = _faces_grid(np.float32, fc=CUBED_SPHERE)
    gds, group = ds, xg.Grid(ds, coords=COORDS, face_connections=CUBED_SPHERE, host_devices=host_devices)
    yield grid, group, ds["c"], ["X", "Y", "Z"], dict(padding="extend")
    _, fgrid = _fold_grid("fill", "T", np.float64)
    _, fgroup = _fold_grid("fill", "T", np.float64, host_devices=host_devices)
    yield fgrid, fgroup, _fold_field("center", np.float64), ["Y", "X"], dict(to={"Y": "outer"})


def test_host_group_of_one_matches_one_device(spy):
    for grid, group, da, axes, kw in _group_cases([0]):
        spy.clear()
        got = group.diff(da, axes, **kw)
        assert len(spy) == 1
        np.testing.assert_array_equal(_host(got), _host(grid.diff(da, axes, **kw)))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_host_group_of_two_matches_one_device(spy):
    for grid, group, da, axes, kw in _group_cases([0, 1]):
        np.testing.assert_array_equal(_host(group.diff(da, axes, **kw)), _host(grid.diff(da, axes, **kw)))
