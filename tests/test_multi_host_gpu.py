"""Multi-axis Grid.diff / interp / min / max and Grid.integrate / average of numpy fields stream through the GPU in
slabs (xg_stencil_multi_host, xg_wreduce_host_multi).  Every result equals the same Grid call on the
device-resident field bit for bit.  Slabs of 1 MiB cut each call into several slabs with a ragged last one; the
cases the slabs cannot pad still give the device result, through the whole-field route."""

import ctypes as C

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from xgcm_b200 import _capi, ops

pytestmark = pytest.mark.gpu

SHIFTS = {"left": (1, 0), "right": (0, 1), "outer": (1, 1), "inner": (0, 0)}


def _grid(sizes, padding="fill", fill_value=0.0, metrics=None, data_vars=None):
    """A plain grid with the five positions on every axis of `sizes` ({"X": nx, ...}): dims XC, XG, XR, XO, XI."""
    coords, ds_coords = {}, {}
    for ax, n in sizes.items():
        pos = {"center": (ax + "C", np.arange(n) + 0.5), "left": (ax + "G", np.arange(n) + 0.0),
               "right": (ax + "R", np.arange(n) + 1.0), "outer": (ax + "O", np.arange(n + 1) + 0.0),
               "inner": (ax + "I", np.arange(n - 1) + 1.0)}
        coords[ax] = {p: name for p, (name, _) in pos.items()}
        ds_coords.update({name: values for name, values in pos.values()})
    ds = xg.Dataset(data_vars=data_vars or {}, coords=ds_coords)
    return xg.Grid(ds, coords=coords, padding=padding, fill_value=fill_value, metrics=metrics,
                   autoparse_metadata=False)


def _field(shape, dtype, seed, nan_frac=0.01):
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(shape).astype(dtype)
    a[rng.random(shape) < nan_frac] = np.nan
    return a


def _host(res):
    assert not res.is_device
    return np.asarray(res.data)


def _spy(monkeypatch, name):
    """Count the calls of ops.<name> (the whole-field device route of a Grid call)."""
    calls = []
    real = getattr(ops, name)

    def wrapped(*a, **k):
        calls.append(name)
        return real(*a, **k)

    monkeypatch.setattr(ops, name, wrapped)
    return calls


@pytest.fixture(autouse=True)
def small_slabs(monkeypatch):
    monkeypatch.setenv("XG_HOST_SLAB_MB", "1")


# ------------------------------------------------------------------------------------------------- stencils
# (dims, shape, axes, cut): the slab dim is a batch dim, an un-operated middle dim, or operated dim 0
LAYOUTS = {
    "batch_xy": (("T", "ZC", "YC", "XC"), (7, 6, 20, 64), ["X", "Y"], "batch"),
    "batch_xyz": (("T", "ZC", "YC", "XC"), (7, 6, 20, 64), ["X", "Y", "Z"], "batch"),
    "batch_zyx": (("T", "ZC", "YC", "XC"), (7, 6, 20, 64), ["Z", "Y", "X"], "batch"),
    "middle_xz": (("ZC", "YC", "XC"), (9, 37, 96), ["X", "Z"], "middle"),
    "middle_zx": (("ZC", "YC", "XC"), (9, 37, 96), ["Z", "X"], "middle"),
    "unit_t_yx": (("T", "ZC", "YC", "XC"), (1, 13, 24, 64), ["Y", "X"], "middle"),
    "dim0_xyz": (("ZC", "YC", "XC"), (23, 30, 64), ["X", "Y", "Z"], "dim0"),
    "dim0_yzx": (("ZC", "YC", "XC"), (23, 30, 64), ["Y", "Z", "X"], "dim0"),
    "dim0_zy": (("ZC", "YC"), (45, 1000), ["Z", "Y"], "dim0"),
}
# each op meets each target position once, the paddings (fill with NaN and with a number) rotating under them
COMBOS = [(op, to, ("periodic", "fill", "extend", "fill_nan")[(i + j) % 4])
          for i, op in enumerate(("diff", "interp", "min", "max"))
          for j, to in enumerate(("left", "right", "outer", "inner"))]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_multi_axis_stencils_of_numpy_fields_equal_the_device_call(monkeypatch, layout, dtype):
    dims, shape, axes, cut = LAYOUTS[layout]
    sizes = {d[0]: n for d, n in zip(dims, shape) if d != "T"}
    a = _field(shape, dtype, seed=len(layout))
    da = xg.DataArray(a, dims=dims)
    dev = da.to_device()
    device_route = _spy(monkeypatch, "stencil_multi")
    host_route = _spy(monkeypatch, "stencil_multi_host")
    lib = _capi.load()
    for op, to, pad in COMBOS:
        grid = _grid(sizes, padding="fill" if pad == "fill_nan" else pad, fill_value=np.nan if pad == "fill_nan" else 1.5)
        kw = dict(to={ax: to for ax in axes})
        device_route.clear()
        host_route.clear()
        n0 = lib.xg_launch_count()
        got = getattr(grid, op)(da, axes, **kw)
        launches = lib.xg_launch_count() - n0
        want = getattr(grid, op)(dev, axes, **kw)
        assert got.dims == want.dims
        np.testing.assert_array_equal(_host(got), want.data.cpu().numpy(), err_msg=f"{op} to={to} {pad}")
        # the slabs cannot pad a cut operated dim across its ends: outer / inner shifts and periodic
        refused = cut == "dim0" and (to in ("outer", "inner") or pad == "periodic")
        assert host_route == ["stencil_multi_host"], (op, to, pad)
        assert device_route == (["stencil_multi"] * 2 if refused else ["stencil_multi"]), (op, to, pad)
        if not refused:
            assert launches >= 4, (op, to, pad, launches)  # one fused launch per slab, several slabs


def test_refused_cases_fall_back_to_the_device_route(monkeypatch):
    """A periodic Z or an outer Z of a (Z, Y, X) field operated along all three dims: the twin refuses (XG_ENOTIMPL),
    and the Grid call gives the device result."""
    a = _field((23, 30, 64), np.float32, seed=5)
    da = xg.DataArray(a, dims=("ZC", "YC", "XC"))
    with pytest.raises(NotImplementedError):
        ops.stencil_multi_host(a, [(2, "diff", 1, 0, "fill", 0.0), (1, "diff", 1, 0, "fill", 0.0),
                                   (0, "diff", 1, 0, "periodic", 0.0)])
    with pytest.raises(NotImplementedError):
        ops.stencil_multi_host(a, [(2, "interp", 1, 0, "fill", 0.0), (1, "interp", 1, 0, "fill", 0.0),
                                   (0, "interp", 1, 1, "extend", 0.0)])
    grid = _grid({"X": 64, "Y": 30, "Z": 23}, padding={"X": "fill", "Y": "extend", "Z": "periodic"})
    for kw in (dict(), dict(to={"X": "left", "Y": "right", "Z": "outer"}, padding="extend")):
        got = grid.interp(da, ["X", "Y", "Z"], **kw)
        want = grid.interp(da.to_device(), ["X", "Y", "Z"], **kw)
        np.testing.assert_array_equal(_host(got), want.data.cpu().numpy())


# ------------------------------------------------------------------------------------------------- reductions
def _reduce_case(name, dtype):
    """(grid, DataArray, axes) of one reduction case; the weight is the metric the Grid selects."""
    rng = np.random.default_rng(11)
    w = lambda *shape: (rng.random(shape) + 0.25).astype(np.float64)  # noqa: E731
    if name == "batch_bcast":  # slab dim T, not reduced; area (Y, X) broadcast along it: uploaded whole
        shape, dims, axes = (9, 6, 30, 70), ("T", "ZC", "YC", "XC"), ["X", "Y"]
        metrics, data = {("X", "Y"): ["area"]}, {"area": (("YC", "XC"), w(30, 70))}
    elif name == "batch_span":  # slab dim Z, not reduced; a (Z, Y, X) area spans it: streamed beside the field
        shape, dims, axes = (13, 30, 70), ("ZC", "YC", "XC"), ["X", "Y"]
        metrics, data = {("X", "Y"): ["area"]}, {"area": (("ZC", "YC", "XC"), w(13, 30, 70))}
    elif name == "middle_span":  # slab dim Y between the reduced Z and X; the (Z, Y, X) weight spans it
        shape, dims, axes = (11, 40, 70), ("ZC", "YC", "XC"), ["Z", "X"]
        metrics, data = {("X", "Z"): ["dxdz"]}, {"dxdz": (("ZC", "YC", "XC"), w(11, 40, 70))}
    elif name == "whole_span":  # every dim reduced: slabs of Z, the (Z, Y, X) volume streamed beside them
        shape, dims, axes = (31, 40, 70), ("ZC", "YC", "XC"), ["X", "Y", "Z"]
        metrics, data = {("X", "Y", "Z"): ["vol"]}, {"vol": (("ZC", "YC", "XC"), w(31, 40, 70))}
    elif name == "whole_bcast":  # every dim reduced, the weight broadcast along the slab dim Z
        shape, dims, axes = (31, 40, 70), ("ZC", "YC", "XC"), ["Z", "Y", "X"]
        metrics, data = {("X", "Y", "Z"): ["wxy"]}, {"wxy": (("YC", "XC"), w(40, 70))}
    elif name == "whole_unit_t":  # (1, Z, Y, X): the slab dim is Z, behind a non-reduced dim of extent 1
        shape, dims, axes = (1, 31, 40, 70), ("T", "ZC", "YC", "XC"), ["X", "Y", "Z"]
        metrics, data = {("X", "Y", "Z"): ["vol"]}, {"vol": (("ZC", "YC", "XC"), w(31, 40, 70))}
    elif name == "whole_2d":  # (Y, X) over both, area spanning Y
        shape, dims, axes = (300, 280), ("YC", "XC"), ["Y", "X"]
        metrics, data = {("X", "Y"): ["area"]}, {"area": (("YC", "XC"), w(300, 280))}
    elif name == "whole_product":  # dx (X) * dy (Y) * dz (Z), multiplied on the device by the Grid
        shape, dims, axes = (31, 40, 70), ("ZC", "YC", "XC"), ["X", "Y", "Z"]
        metrics = {("X",): ["dx"], ("Y",): ["dy"], ("Z",): ["dz"]}
        data = {"dx": (("XC",), w(70)), "dy": (("YC",), w(40)), "dz": (("ZC",), w(31))}
    else:
        raise KeyError(name)
    sizes = {d[0]: n for d, n in zip(dims, shape) if d != "T"}
    grid = _grid(sizes, metrics=metrics, data_vars=data)
    a = _field(shape, dtype, seed=len(name), nan_frac=0.02)
    a[(slice(None),) * (len(shape) - 2) + (3,)] = np.nan  # whole NaN rows: lines with no valid weight
    if dims[0] == "T" and shape[0] > 2:
        a[2] = np.nan  # a whole step: its mean has no valid weight at all (NaN)
    return grid, xg.DataArray(a, dims=dims), axes


REDUCE_CASES = ["batch_bcast", "batch_span", "middle_span", "whole_span", "whole_bcast", "whole_unit_t", "whole_2d",
                "whole_product"]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("case", REDUCE_CASES)
def test_multi_axis_reductions_of_numpy_fields_equal_the_device_call(monkeypatch, case, dtype):
    grid, da, axes = _reduce_case(case, dtype)
    dev = da.to_device()
    device_route = _spy(monkeypatch, "wreduce")
    lib = _capi.load()
    for method in ("integrate", "average"):
        for skipna in (True, False):
            device_route.clear()
            n0 = lib.xg_launch_count()
            got = getattr(grid, method)(da, axes, skipna=skipna)
            launches = lib.xg_launch_count() - n0
            assert device_route == [], (method, skipna)  # streamed, not the whole-field chain
            assert launches >= 4 * (len(axes) - 1)
            want = getattr(grid, method)(dev, axes, skipna=skipna)
            assert got.dims == want.dims
            np.testing.assert_array_equal(_host(got), want.data.cpu().numpy(), err_msg=f"{method} skipna={skipna}")


def test_wreduce_host_multi_matches_the_device_chain_for_any_axis_order():
    """The ops-level twin against the launch sequence of Grid._weighted_reduce written out with ops.wreduce."""
    rng = np.random.default_rng(2)
    a = _field((5, 17, 33, 40), np.float64, seed=2)
    w = (rng.random((1, 17, 1, 40)) + 0.5)
    x, wt = torch.from_numpy(a).cuda(), torch.from_numpy(w).cuda()
    for axes in ([3, 1], [1, 3], [0, 2], [0, 1, 2, 3], [2, 0, 3]):
        order = sorted(axes, reverse=True)
        for mode in ("sum", "mean"):
            num, den = x, None
            for k, axis in enumerate(order):
                if mode == "mean":
                    den = ops.wreduce(num, axis, wt, "wvalid", True) if k == 0 else ops.wreduce(den, axis, None, "sum", False)
                num = ops.wreduce(num, axis, wt if k == 0 else None, "sum", True)
            want = ops.binary("divnz", num, den) if mode == "mean" else num
            got = ops.wreduce_host_multi(a, axes, w, mode, True)
            np.testing.assert_array_equal(got, want.cpu().numpy(), err_msg=f"{axes} {mode}")


# ------------------------------------------------------------------------------------------------- footprint
def _workspace_bytes():
    v = C.c_int64(-1)
    _capi.check(_capi.load().xg_host_workspace_bytes(torch.cuda.current_device(), C.byref(v)))
    return v.value


def test_multi_axis_calls_of_a_large_numpy_field_keep_a_small_device_footprint(monkeypatch):
    """interp(["X", "Y", "Z"]) and average(["X", "Y", "Z"]) of a 384 MiB field with 8 MiB slabs: the workspace and
    torch's allocations stay far below the field's size.  The volume weight is one registered host metric (a product
    of separate metrics would be formed on the device, as large as the field)."""
    monkeypatch.setenv("XG_HOST_SLAB_MB", "8")
    nz, ny, nx = 96, 1024, 1024
    rng = np.random.default_rng(7)
    a = rng.random((nz, ny, nx), dtype=np.float32)
    vol = (rng.random((nz, ny, nx), dtype=np.float32) + 0.5)
    grid = _grid({"X": nx, "Y": ny, "Z": nz}, padding={"X": "periodic", "Y": "fill", "Z": "extend"},
                 metrics={("X", "Y", "Z"): ["vol"]}, data_vars={"vol": (("ZC", "YC", "XC"), vol)})
    da = xg.DataArray(a, dims=("ZC", "YC", "XC"))
    lib = _capi.load()
    _capi.check(lib.xg_host_workspace_release())
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    n0 = lib.xg_launch_count()
    corner = grid.interp(da, ["X", "Y", "Z"], to="left")
    n1 = lib.xg_launch_count()
    mean = grid.average(da, ["X", "Y", "Z"])
    n2 = lib.xg_launch_count()
    torch.cuda.synchronize()
    workspace, peak = _workspace_bytes(), torch.cuda.max_memory_allocated() - base
    assert 0 < workspace < a.nbytes / 4, workspace
    assert peak < a.nbytes / 4, peak
    assert n1 - n0 >= nz  # one fused launch per plane of Z (8 MiB slabs hold one input and one result plane)
    assert n2 - n1 >= 4 * nz  # per slab: two launches along X, two along Y (sum and valid weights)
    # and the values are the device call's
    dev = da.to_device()
    np.testing.assert_array_equal(_host(corner), grid.interp(dev, ["X", "Y", "Z"], to="left").data.cpu().numpy())
    np.testing.assert_array_equal(_host(mean), grid.average(dev, ["X", "Y", "Z"]).data.cpu().numpy())
