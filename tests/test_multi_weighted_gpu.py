"""Multi-axis Grid.diff / interp / min / max with ``metric_weighted`` in ONE fused launch
(xg_stencil_multi_weighted), and numpy fields streamed in slabs (xg_stencil_multi_weighted_host).

Every result equals, bit for bit, the per-axis route — the single-axis weighted calls in series — and the
oracle's stencil2 with pre / post metrics applied stage by stage; the launch label is asserted beside the values,
so a silent fallback to the per-axis launches cannot pass."""

import ctypes as C
import itertools
import warnings

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from oracle import stencil as oracle
from xgcm_b200 import _capi, ops

pytestmark = pytest.mark.gpu

SHIFTS = {"left": (1, 0), "right": (0, 1), "outer": (1, 1), "inner": (0, 0), "center": (0, 0)}
SUFFIX = {"center": "C", "left": "G", "right": "R", "outer": "O", "inner": "I"}
POSITIONS = list(SUFFIX)


def _extent(n, pos):
    return n + 1 if pos == "outer" else n - 1 if pos == "inner" else n


def _grid(sizes, padding, fill_value, metric_kind, dtype, rng, host_devices=None):
    """Plain grid over `sizes` ({"Z": nz, "Y": ny, "X": nx}) with the five positions per axis (dims ZC, YG, XO ...).

    metric_kind: "registered" — dz, 2-D areas and 3-D volumes at every position the calls need, so get_metric finds
    each one as registered; "product" — only dx, dy, dz (the areas are their products); "interpolated" — dx, dy, dz
    and areas / volumes at the cell centre only (get_metric interpolates them to the other positions)."""
    coords, ds_coords, metrics, data_vars = {}, {}, {}, {}
    for ax, n in sizes.items():
        coords[ax] = {p: ax + s for p, s in SUFFIX.items()}
        for p, s in SUFFIX.items():
            ds_coords[ax + s] = np.arange(_extent(n, p)) + (0.5 if p == "center" else 0.0)

    def add(key, dims):
        name = "m_" + "_".join(dims)
        if name in data_vars:
            return
        shape = tuple(len(ds_coords[d]) for d in dims)
        data_vars[name] = (dims, (rng.random(shape) + 0.5).astype(np.float64))
        metrics.setdefault(key, []).append(name)

    hz = [a for a in ("Y", "X") if a in sizes]
    for ax in sizes:  # 1-D metrics along each axis at every position
        for p in POSITIONS:
            add((ax,), (ax + SUFFIX[p],))
    if metric_kind == "registered":
        for py, px in itertools.product(POSITIONS, POSITIONS):
            add(tuple(hz), ("Y" + SUFFIX[py], "X" + SUFFIX[px]))
        if "Z" in sizes:
            for pz, py, px in itertools.product(POSITIONS, POSITIONS, POSITIONS):
                add(("X", "Y", "Z"), ("Z" + SUFFIX[pz], "Y" + SUFFIX[py], "X" + SUFFIX[px]))
    elif metric_kind == "interpolated":
        add(tuple(hz), ("YC", "XC"))
        if "Z" in sizes:
            add(("X", "Y", "Z"), ("ZC", "YC", "XC"))
    ds = xg.Dataset(data_vars=data_vars, coords=ds_coords)
    return xg.Grid(ds, coords=coords, padding=padding, fill_value=fill_value, metrics=metrics,
                   autoparse_metadata=False, host_devices=host_devices)


def _field(shape, dtype, seed, nan_frac=0.02):
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(shape).astype(dtype)
    a[rng.random(shape) < nan_frac] = np.nan
    return a


def _label():
    return _capi.last_launch()


def _per_axis(grid, op, da, axes, to, weighted):
    """The per-axis route: the single-axis weighted calls in series."""
    cur = da
    for ax in axes:
        w = weighted.get(ax) if isinstance(weighted, dict) else weighted
        cur = getattr(grid, op)(cur, ax, to={ax: to}, metric_weighted=w)
    return cur


def _chain(grid, dims, shape, axes, to, weighted, paddings, fills, dtype):
    """Per stage: the stencil spec (axis, op-less) and the pre / post metrics get_metric gives the stage, as host
    arrays shaped against the stage's input / output."""
    stages = []
    dims, shape = tuple(dims), list(shape)
    for ax in axes:
        w = weighted.get(ax) if isinstance(weighted, dict) else weighted
        lo, hi = SHIFTS[to]
        d_in = [d for d in dims if d[0] == ax][0]
        num = dims.index(d_in)
        out_dims = tuple(ax + SUFFIX[to] if d == d_in else d for d in dims)
        out_shape = list(shape)
        out_shape[num] += lo + hi - 1
        pre = post = None
        if w:
            pre = grid._metric_host(grid.get_metric(xg.DataArray(np.empty(shape, dtype), dims=dims), w), dims, dtype)
            post = grid._metric_host(grid.get_metric(xg.DataArray(np.empty(out_shape, dtype), dims=out_dims), w),
                                     out_dims, dtype)
        pad = paddings[ax] if (lo or hi) else None
        stages.append(((num, lo, hi, pad, fills[ax]), pre, post, shape, out_shape))
        dims, shape = out_dims, out_shape
    return stages


def _oracle(op, a, stages):
    """oracle.stencil2 stage by stage, with each stage's pre / post metrics."""
    cur = a
    for (num, lo, hi, pad, fill), pre, post, _, _ in stages:
        cur = oracle.stencil2(op, cur, num, lo, hi, pad, fill, pre, post).astype(a.dtype)
    return cur


def _ops_call(op, x, stages):
    """ops.stencil_multi with the chain's metrics as device tensors: the fused kernel whatever the metric shapes."""
    specs = [(num, op, lo, hi, pad, fill) for (num, lo, hi, pad, fill), *_ in stages]
    pre = [None if m is None else torch.from_numpy(m).to(x.device) for _, m, _, _, _ in stages]
    post = [None if m is None else torch.from_numpy(m).to(x.device) for _, _, m, _, _ in stages]
    return ops.stencil_multi(x, specs, pre=pre, post=post)


WEIGHTS = ["X", ("X", "Y"), {"X": ("X", "Y"), "Y": None, "Z": "Z"}, {"Y": "Y", "Z": ("X", "Y", "Z")},
           ("X", "Y", "Z")]
ORDERS = [["X", "Y"], ["Y", "X"], ["X", "Y", "Z"], ["Z", "Y", "X"], ["Y", "Z"], ["X", "Z"]]
PADS = [{"X": "periodic", "Y": "fill", "Z": "extend"}, {"X": "fill", "Y": "extend", "Z": "periodic"},
        {"X": "extend", "Y": "periodic", "Z": "fill"}]
FILLS = [{"X": 1.5, "Y": -2.0, "Z": 0.0}, {"X": np.nan, "Y": 3.0, "Z": -1.0}]


def _weights_for(w, axes):
    """`w` as metric_weighted for `axes`: None when no operated axis would be weighted (the case is skipped)."""
    if isinstance(w, dict):
        w = {k: v for k, v in w.items() if k in axes}
        return w if any(w.values()) else None
    return w


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("metric_kind", ["registered", "product", "interpolated"])
@pytest.mark.parametrize("shape", [(5, 9, 67), (6, 10, 64)])
def test_fused_weighted_equals_per_axis_route_and_oracle(shape, metric_kind, dtype):
    sizes = dict(zip("ZYX", shape))
    grids = {}
    a = _field(shape, dtype, seed=shape[0])
    dev = xg.DataArray(torch.from_numpy(a).cuda(), dims=("ZC", "YC", "XC"))
    lib = _capi.load()
    cases = itertools.product(range(len(ORDERS)), ("diff", "interp", "min", "max"), POSITIONS[1:])
    for i, (k, op, to) in enumerate(cases):
        axes = ORDERS[k]
        w = _weights_for(WEIGHTS[(i + k) % len(WEIGHTS)], axes)
        # get_metric interpolates a metric to the axis's default position only (the reference's interp_like)
        if w is None or (metric_kind == "interpolated" and to != "left"):
            continue
        pads, fills = PADS[i % len(PADS)], FILLS[(i // 3) % len(FILLS)]
        key = (i % len(PADS), (i // 3) % len(FILLS))
        if key not in grids:
            grids[key] = _grid(sizes, pads, fills, metric_kind, dtype, np.random.default_rng(1))
        grid = grids[key]
        msg = f"{op} {axes} to={to} w={w} pads={pads} fills={fills}"
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = _per_axis(grid, op, dev, axes, to, w)
            n0 = lib.xg_launch_count()
            got = getattr(grid, op)(dev, axes, to={ax: to for ax in axes}, metric_weighted=w)
            launches = lib.xg_launch_count() - n0
            label = _label()
            stages = _chain(grid, dev.dims, shape, axes, to, w, pads, fills, dtype)
        ref = _oracle(op, a, stages)
        assert got.dims == want.dims, msg
        np.testing.assert_array_equal(got.data.cpu().numpy(), want.data.cpu().numpy(), err_msg=msg)
        np.testing.assert_array_equal(got.data.cpu().numpy(), ref, err_msg=msg)
        assert label == "xg_stencil_multi(weighted)", msg
        if metric_kind == "registered":
            assert launches == 1, (msg, launches)
        # the fused kernel itself, whatever the metric shapes
        direct = _ops_call(op, dev.data, stages)
        assert _label() == "xg_stencil_multi(weighted)", msg
        np.testing.assert_array_equal(direct.cpu().numpy(), ref, err_msg=msg)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_large_fields_misaligned_slices_and_time_dims(dtype):
    """Fields the metric-free chain would hand to the TMA tile kernel (several tiles per CTA, x not a tile
    multiple), a time dim in front, and a slice at a storage offset that rules out 16-byte vectors: one weighted
    launch each, equal to the per-axis route and the oracle."""
    rng = np.random.default_rng(2)
    pads, fills = {"X": "periodic", "Y": "fill", "Z": "extend"}, {"X": 0.0, "Y": 2.5, "Z": 0.0}
    for shape, axes, w in [((12, 260, 520), ["X", "Y"], ("X", "Y", "Z")),
                           ((12, 260, 520), ["X", "Y"], ("X", "Y")),
                           ((9, 130, 452), ["X", "Y", "Z"], {"X": "X", "Y": "Y"}),
                           ((3, 5, 40, 96), ["Y", "X"], ("X", "Y"))]:
        sizes = dict(zip("ZYX", shape[-3:]))
        grid = _grid(sizes, pads, fills, "registered", dtype, rng)
        dims = ("T", "ZC", "YC", "XC")[-len(shape):]
        a = torch.from_numpy(_field(shape, dtype, seed=shape[-1])).cuda()
        views = [a]
        if len(shape) == 4:  # the same values one element into an allocation: no 16-byte vectors
            flat = torch.empty(a.numel() + 1, dtype=a.dtype, device=a.device)
            views.append(flat[1:].view(shape))
            views[1].copy_(a)
            assert views[1].data_ptr() % 16 != 0
        for x in views:
            da = xg.DataArray(x, dims=dims)
            want = _per_axis(grid, "interp", da, axes, "left", w)
            got = grid.interp(da, axes, to="left", metric_weighted=w)
            assert _label() == "xg_stencil_multi(weighted)", (shape, axes)
            np.testing.assert_array_equal(got.data.cpu().numpy(), want.data.cpu().numpy())
            stages = _chain(grid, dims, x.shape, axes, "left", w, pads, fills, dtype)
            direct = _ops_call("interp", x, stages)
            assert _label() == "xg_stencil_multi(weighted)", (shape, axes)
            np.testing.assert_array_equal(direct.cpu().numpy(), want.data.cpu().numpy())
            np.testing.assert_array_equal(direct.cpu().numpy(), _oracle("interp", x.cpu().numpy(), stages))
            # the same call without metrics keeps its metric-free route
            grid.interp(da, axes, to="left")
            assert _label() != "xg_stencil_multi(weighted)"


def _spy(monkeypatch, name):
    calls = []
    real = getattr(ops, name)

    def wrapped(*a, **k):
        calls.append(name)
        return real(*a, **k)

    monkeypatch.setattr(ops, name, wrapped)
    return calls


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("dims,shape,axes", [
    (("T", "ZC", "YC", "XC"), (4, 6, 30, 64), ["X", "Y"]),
    (("T", "ZC", "YC", "XC"), (4, 6, 30, 64), ["Z", "Y", "X"]),
    (("ZC", "YC", "XC"), (13, 30, 64), ["X", "Y", "Z"]),
    (("ZC", "YC", "XC"), (13, 30, 64), ["Y", "X"]),
])
def test_numpy_fields_stream_and_equal_the_device_call(monkeypatch, dims, shape, axes, dtype):
    monkeypatch.setenv("XG_HOST_SLAB_MB", "1")
    rng = np.random.default_rng(3)
    sizes = {d[0]: n for d, n in zip(dims, shape) if d != "T"}
    pads = {"X": "periodic", "Y": "fill", "Z": "extend"}
    grid = _grid(sizes, pads, {"X": 0.0, "Y": -1.0, "Z": 0.0}, "registered", dtype, rng)
    a = _field(shape, dtype, seed=5)
    da = xg.DataArray(a, dims=dims)
    dev = xg.DataArray(torch.from_numpy(a).cuda(), dims=dims)
    host_route = _spy(monkeypatch, "stencil_multi_host")
    device_route = _spy(monkeypatch, "stencil_multi")
    upload = _spy(monkeypatch, "stencil2")
    for op, to, w in [("interp", "left", ("X", "Y")), ("diff", "right", {"X": "X", "Y": "Y"}),
                      ("max", "left", ("X", "Y"))]:
        host_route.clear()
        device_route.clear()
        upload.clear()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            got = getattr(grid, op)(da, axes, to={ax: to for ax in axes}, metric_weighted=w)
            assert host_route == ["stencil_multi_host"] and not device_route and not upload, (op, axes)
            assert not got.is_device
            want = getattr(grid, op)(dev, axes, to={ax: to for ax in axes}, metric_weighted=w)
        np.testing.assert_array_equal(np.asarray(got.data), want.data.cpu().numpy(), err_msg=f"{op} {axes}")


def _workspace_bytes():
    v = C.c_int64(-1)
    _capi.check(_capi.load().xg_host_workspace_bytes(torch.cuda.current_device(), C.byref(v)))
    return v.value


def test_weighted_calls_of_a_large_numpy_field_keep_a_small_device_footprint(monkeypatch):
    """interp(["X", "Y"]) with 2-D areas of a 384 MiB field with 8 MiB slabs: the workspace (the areas uploaded
    whole, plus the slabs) and torch's allocations stay far below the field's size."""
    monkeypatch.setenv("XG_HOST_SLAB_MB", "8")
    nz, ny, nx = 96, 1024, 1024
    rng = np.random.default_rng(7)
    a = rng.random((nz, ny, nx), dtype=np.float32)
    coords = {ax: {"center": ax + "C", "left": ax + "G"} for ax in "ZYX"}
    ds_coords = {ax + s: np.arange(n) + off for ax, n in zip("ZYX", (nz, ny, nx)) for s, off in (("C", 0.5), ("G", 0.0))}
    areas = {f"area_{py}{px}": (("Y" + py, "X" + px), rng.random((ny, nx), dtype=np.float32) + 0.5)
             for py in "CG" for px in "CG"}
    ds = xg.Dataset(data_vars=areas, coords=ds_coords)
    grid = xg.Grid(ds, coords=coords, padding={"X": "periodic", "Y": "fill", "Z": "extend"},
                   metrics={("X", "Y"): list(areas)}, autoparse_metadata=False)
    da = xg.DataArray(a, dims=("ZC", "YC", "XC"))
    lib = _capi.load()
    _capi.check(lib.xg_host_workspace_release())
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    n0 = lib.xg_launch_count()
    got = grid.interp(da, ["X", "Y"], to="left", metric_weighted=("X", "Y"))
    n1 = lib.xg_launch_count()
    torch.cuda.synchronize()
    workspace, peak = _workspace_bytes(), torch.cuda.max_memory_allocated() - base
    assert 0 < workspace < a.nbytes / 4, workspace
    assert peak < a.nbytes / 4, peak
    assert n1 - n0 >= 8, n1 - n0  # several slabs, one fused launch each
    dev = da.to_device()
    want = grid.interp(dev, ["X", "Y"], to="left", metric_weighted=("X", "Y"))
    np.testing.assert_array_equal(np.asarray(got.data), want.data.cpu().numpy())


def test_host_device_group_of_every_gpu_gives_the_one_gpu_bits(monkeypatch):
    monkeypatch.setenv("XG_HOST_SLAB_MB", "1")
    shape = (6, 8, 40, 128)
    sizes = dict(zip("ZYX", shape[1:]))
    pads, fills = {"X": "periodic", "Y": "fill", "Z": "extend"}, {"X": 0.0, "Y": 1.0, "Z": 0.0}
    one = _grid(sizes, pads, fills, "registered", np.float32, np.random.default_rng(4))
    group = _grid(sizes, pads, fills, "registered", np.float32, np.random.default_rng(4), host_devices="all")
    a = _field(shape, np.float32, seed=9)
    da = xg.DataArray(a, dims=("T", "ZC", "YC", "XC"))
    for axes in (["X", "Y"], ["X", "Y", "Z"]):
        want = one.interp(da, axes, to="left", metric_weighted={"X": "X", "Y": ("X", "Y")})
        got = group.interp(da, axes, to="left", metric_weighted={"X": "X", "Y": ("X", "Y")})
        np.testing.assert_array_equal(np.asarray(got.data), np.asarray(want.data))
