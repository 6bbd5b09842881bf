"""Metric-weighted diff / interp / min / max across face connections: the fused device route (halo planes of
x * pre, one xg_stencil2 with the pre- and post-metric) and the streamed numpy route
(xg_stencil2_host_connected_weighted), bit for bit equal to each other and to the reference's composition:
pad(x * m) -> stencil -> / m_new (oracle/faces.py).  XG_HOST_SLAB_MB=1 forces several slabs."""

import itertools

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from oracle import stencil as S
from oracle.faces import pad_face_connections
from xgcm_b200 import _capi, ops

pytestmark = pytest.mark.gpu

N = 8
LEAD = (3, 4)  # (time, k): 12 slab rows -> 4 slabs of 3
POS = {"center": "", "left": "l", "right": "r", "outer": "o"}
COORDS = {"X": {p: "x" + s for p, s in POS.items()}, "Y": {p: "y" + s for p, s in POS.items()},
          "Z": {"center": "k", "left": "kl"}}
AXES = {"X": tuple(COORDS["X"].values()), "Y": tuple(COORDS["Y"].values()), "Z": ("k", "kl")}

X_TO_X = {"face": {0: {"X": (None, (1, "X", False))}, 1: {"X": ((0, "X", False), None)}}}
X_TO_X_REV = {"face": {0: {"X": (None, (1, "X", True))}, 1: {"X": (None, (0, "X", True))}}}
X_TO_Y = {"face": {0: {"X": (None, (1, "Y", False))}, 1: {"Y": ((0, "X", False), None)}}}
X_TO_Y_REV = {"face": {0: {"X": (None, (1, "Y", True))}, 1: {"Y": (None, (0, "X", True))}}}
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
GRIDS = {"cubed_sphere": CUBED_SPHERE, "x_to_x": X_TO_X, "x_to_x_rev": X_TO_X_REV, "x_to_y": X_TO_Y,
         "x_to_y_rev": X_TO_Y_REV}
SHIFTS = [("center", "left"), ("center", "right"), ("center", "outer"), ("left", "center"), ("right", "center")]
PADDINGS = [("fill", 1.5), ("extend", 0.0), ("periodic", 0.0)]


@pytest.fixture(autouse=True)
def slab(monkeypatch):
    monkeypatch.setenv("XG_HOST_SLAB_MB", "1")


@pytest.fixture
def streamed(monkeypatch):
    """The number of calls that reached xg_stencil2_host_connected_weighted."""
    count = [0]
    real = ops.stencil2_host_connected_weighted

    def counted(*a, **kw):
        count[0] += 1
        return real(*a, **kw)

    monkeypatch.setattr(ops, "stencil2_host_connected_weighted", counted)
    return count


def _dataset(fc, dtype, lead=LEAD, seed=0, n=N):
    """A field at every X / Y position of (time, k, face, y, x), and metrics: dx (face, y, x*) and dy at the same
    X positions (so that the X, Y product has no interpolation), dxk (k, face, y, x*), dz (k) / (kl)."""
    rng = np.random.default_rng(seed)
    nf = len(fc["face"])

    def _n(pos):
        return n + 1 if pos == "outer" else n

    coords = {d: np.arange(_n(p)) + 0.0 for ax in ("X", "Y") for p, d in COORDS[ax].items()}
    coords.update({"face": np.arange(nf), "k": np.arange(lead[1]) + 0.0, "kl": np.arange(lead[1]) - 0.5,
                   "time": np.arange(lead[0]) + 0.0})
    data = {}
    for py, px in itertools.product(POS, POS):
        dims = ("time", "k", "face", COORDS["Y"][py], COORDS["X"][px])
        a = rng.standard_normal(lead + (nf, _n(py), _n(px))).astype(dtype)
        a.ravel()[rng.choice(a.size, 3, replace=False)] = np.nan
        data[f"f_{py}_{px}"] = (dims, a)
    for p in POS:
        data[f"dx_{p}"] = (("face", "y", COORDS["X"][p]), 0.5 + rng.random((nf, n, _n(p))))
        data[f"dyx_{p}"] = (("face", "y", COORDS["X"][p]), 0.5 + rng.random((nf, n, _n(p))))
        data[f"dy_{p}"] = (("face", COORDS["Y"][p], "x"), 0.5 + rng.random((nf, _n(p), n)))
        data[f"dxk_{p}"] = (("k", "face", "y", COORDS["X"][p]), 0.5 + rng.random((lead[1], nf, n, _n(p))))
    data["dz_c"] = (("k",), 0.5 + rng.random(lead[1]))
    data["dz_l"] = (("kl",), 0.5 + rng.random(lead[1]))
    return xg.Dataset(data_vars=data, coords=coords)


# metric kind -> ({axes: metric names}, metric_weighted, operated axis)
KINDS = {
    "face": ({("X",): [f"dx_{p}" for p in POS], ("Y",): [f"dy_{p}" for p in POS]}, None, None),
    "level": ({("X",): [f"dxk_{p}" for p in POS]}, "X", "X"),
    "dz": ({("Z",): ["dz_c", "dz_l"]}, "Z", "Z"),
    "product": ({("X",): [f"dx_{p}" for p in POS], ("Y",): [f"dyx_{p}" for p in POS]}, ["X", "Y"], "X"),
}


def _grid(ds, fc, kind, **kw):
    return xg.Grid(ds, coords=COORDS, face_connections=fc, metrics=KINDS[kind][0], autoparse_metadata=False, **kw)


def _bcast(values, mdims, dims, dtype):
    """A metric's values (dims ``mdims``) rounded to the field's dtype and shaped to broadcast against ``dims``."""
    mdims = tuple(mdims)
    v = np.transpose(values, [mdims.index(d) for d in dims if d in mdims])
    return v.reshape([values.shape[mdims.index(d)] if d in mdims else 1 for d in dims]).astype(dtype)


def _metric(ds, kind, ax, dims, dtype):
    """The weight the reference applies at ``dims``: the registered metric(s) of ``kind`` there."""
    if kind == "dz":
        name = "dz_c" if "k" in dims else "dz_l"
        return _bcast(ds[name].values, ds[name].dims, dims, dtype)
    prefix = {"face": "dx" if ax == "X" else "dy", "level": "dxk", "product": "dx"}[kind]
    pos_dim = [d for d in dims if d in AXES[ax]][0]
    p = [p for p, d in COORDS[ax].items() if d == pos_dim][0]
    m = ds[f"{prefix}_{p}"]
    if kind == "product":
        other = ds[f"dyx_{p}"]
        return _bcast(m.values * other.values, m.dims, dims, dtype)
    return _bcast(m.values, m.dims, dims, dtype)


def _oracle(op, a, dims, fc, ax, lo, hi, padding, fill, pre, post):
    padded = pad_face_connections(
        (a * pre).astype(a.dtype), dims, AXES, "face", fc["face"], {ax: (lo, hi)}, {x: padding for x in AXES},
        {x: fill for x in AXES})
    axis = dims.index([d for d in dims if d in AXES[ax]][0])
    return S.stencil2(op, padded, axis, 0, 0, None) / post


def _dev(da):
    return xg.DataArray(torch.from_numpy(np.ascontiguousarray(da.values)).to("cuda:0"), dims=da.dims)


def _host(x):
    return x.data.cpu().numpy() if isinstance(x.data, torch.Tensor) else np.asarray(x.data)


def _field(ds, ax, src):
    py, px = (src, "center") if ax == "Y" else ("center", src) if ax == "X" else ("center", "center")
    return ds[f"f_{py}_{px}"]


def _check(grid, ds, fc, kind, op, ax, src, dst, padding, fill, streamed, da=None, dtype=np.float32):
    weighted = KINDS[kind][1] or ax
    da = _field(ds, ax, src) if da is None else da
    lo, hi = S.PADDING_WIDTH[(src, dst)]
    kw = dict(to=dst, padding=padding, fill_value=fill, metric_weighted=weighted)
    n0 = streamed[0]
    got = getattr(grid, op)(da, ax, **kw)
    assert streamed[0] == n0 + 1, "the numpy field did not stream"
    dev = getattr(grid, op)(_dev(da), ax, **kw)
    assert streamed[0] == n0 + 1
    out_dims = got.dims
    pre = _metric(ds, kind, ax, da.dims, dtype)
    post = _metric(ds, kind, ax, out_dims, dtype)
    want = _oracle(op, da.values, da.dims, fc, ax, lo, hi, padding, fill, pre, post)
    msg = f"{kind} {op} {ax} {src}->{dst} {padding}"
    g = _host(got)
    assert isinstance(got.data, np.ndarray) and g.dtype == dtype, msg
    np.testing.assert_array_equal(g, _host(dev), err_msg=msg)
    np.testing.assert_array_equal(g, want.astype(dtype), err_msg=msg)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", list(GRIDS))
def test_every_grid_op_shift_and_padding(name, dtype, streamed):
    fc = GRIDS[name]
    ds = _dataset(fc, dtype)
    grid = _grid(ds, fc, "face")
    axes = ("X", "Y") if name == "cubed_sphere" else ("X",)
    checked = 0
    for ax, (src, dst), (padding, fill), op in itertools.product(axes, SHIFTS, PADDINGS,
                                                                  ("diff", "interp", "min", "max")):
        if name.startswith("x_to_y") and "outer" in (src, dst):
            continue  # a seam that swaps axes needs square faces (ValueError on every route, as in the reference)
        _check(grid, ds, fc, "face", op, ax, src, dst, padding, fill, streamed, dtype=dtype)
        checked += 1
    assert checked >= 3 * 4 * 4


def _drop_time(da):
    """(k, face, j, i): the slab dim is k, which a (k, face, j, i) metric spans."""
    return xg.DataArray(np.ascontiguousarray(da.values[0]), dims=da.dims[1:])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("kind", ["level", "dz", "product"])
def test_metric_layouts(kind, dtype, streamed):
    """(k, face, j, i) spanning the slab dim, a 1-D dz along Z (no connection there) and a metric product."""
    checked = 0
    for name in ("cubed_sphere", "x_to_y_rev", "x_to_x"):
        fc = GRIDS[name]
        ds = _dataset(fc, dtype, seed=1)
        grid = _grid(ds, fc, kind)
        ax = KINDS[kind][2]
        shifts = [("center", "left")] if ax == "Z" else [s for s in SHIFTS if "outer" not in s]
        for (src, dst), (padding, fill), op in itertools.product(shifts, PADDINGS, ("diff", "interp", "min", "max")):
            for da in ((_field(ds, ax, src), _drop_time(_field(ds, ax, src))) if kind == "level" else (None,)):
                _check(grid, ds, fc, kind, op, ax, src, dst, padding, fill, streamed, da=da, dtype=dtype)
                checked += 1
    assert checked >= 3 * 3 * 4


def test_vector_components_still_raise():
    ds = _dataset(CUBED_SPHERE, np.float32)
    grid = _grid(ds, CUBED_SPHERE, "face")
    u, v = ds["f_center_left"], ds["f_left_center"]
    for arg, other in ((u, v), (_dev(u), _dev(v))):
        with pytest.raises(NotImplementedError, match="vector components"):
            grid.interp({"X": arg}, "X", other_component={"Y": other}, metric_weighted="X")


def test_face_first_layout_takes_the_device_route(streamed):
    ds = _dataset(CUBED_SPHERE, np.float64)
    grid = _grid(ds, CUBED_SPHERE, "face")
    da = xg.DataArray(np.ascontiguousarray(ds["f_center_center"].values[0].transpose(1, 0, 2, 3)),
                      dims=("face", "k", "y", "x"))
    got = grid.interp(da, "X", metric_weighted="X")
    assert streamed[0] == 0
    np.testing.assert_array_equal(_host(got), _host(grid.interp(_dev(da), "X", metric_weighted="X")))
    pre = _metric(ds, "face", "X", da.dims, np.float64)
    post = _metric(ds, "face", "X", got.dims, np.float64)
    np.testing.assert_array_equal(_host(got), _oracle("interp", da.values, da.dims, CUBED_SPHERE, "X", 1, 0, None,
                                                      0.0, pre, post))


def _workspace_bytes():
    v = _capi.i64_array([0])
    _capi.check(_capi.load().xg_host_workspace_bytes(0, v))
    return int(v[0])


def test_device_route_memory():
    """No padded or weighted copy of the field: the peak over the call stays below the result plus field / 8."""
    ds = _dataset(CUBED_SPHERE, np.float32, lead=(4, 12), n=48)
    grid = _grid(ds, CUBED_SPHERE, "face")
    x = _dev(ds["f_center_center"])
    grid.interp(x, "X", metric_weighted="X")  # warm-up: metric uploads and plans
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    got = grid.interp(x, "X", metric_weighted="X")
    torch.cuda.synchronize()
    field = x.data.numel() * 4
    assert torch.cuda.max_memory_allocated() - base < got.data.numel() * 4 + field // 8


def test_host_route_memory(streamed):
    """The numpy field streams: nothing field-sized on the torch side, a workspace bounded by the slab size."""
    ds = _dataset(CUBED_SPHERE, np.float32, lead=(1, 40))
    grid = _grid(ds, CUBED_SPHERE, "face")
    a = ds["f_center_center"]
    _capi.check(_capi.load().xg_host_workspace_release())
    grid.diff(a, "X", metric_weighted="X")  # warm-up
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    got = grid.diff(a, "X", metric_weighted="X")
    assert streamed[0] == 2
    assert torch.cuda.max_memory_allocated() - base < a.values.nbytes // 4
    row = 6 * N * N * 4
    rows = -(-40 // 4)  # 1 MiB holds more: at least four slabs
    plane = 6 * N * 4
    metrics = 2 * 6 * N * N * 4
    # slots (input + result) + planes + weight planes + metrics + fill constants
    assert _workspace_bytes() <= 3 * 2 * rows * row + 4 * rows * plane + metrics + 8
    pre = _metric(ds, "face", "X", a.dims, np.float32)
    post = _metric(ds, "face", "X", got.dims, np.float32)
    np.testing.assert_array_equal(_host(got), _oracle("diff", a.values, a.dims, CUBED_SPHERE, "X", 1, 0, None, 0.0,
                                                      pre, post))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_host_device_group_matches_one_gpu(streamed):
    ds = _dataset(CUBED_SPHERE, np.float64, lead=(5, 6))
    one = _grid(ds, CUBED_SPHERE, "level")
    two = _grid(ds, CUBED_SPHERE, "level", host_devices=[0, 1])
    a = ds["f_center_center"]
    for op, to in (("interp", "left"), ("diff", "outer"), ("max", "right")):
        np.testing.assert_array_equal(_host(getattr(two, op)(a, "X", to=to, metric_weighted="X")),
                                      _host(getattr(one, op)(a, "X", to=to, metric_weighted="X")))
    assert streamed[0] == 6
