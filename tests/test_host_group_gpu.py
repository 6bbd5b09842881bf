"""Host device groups on the H100: every slab-streaming host entry point spread over a group gives the bits of the
same call on device 0.  Groups (0, 0) and (0, 0, 0) run on one GPU (the blocks take turns on its workspace), so
every block boundary, ragged block and per-member upload is exercised here; (0, 1) and "all" need two GPUs.
XG_HOST_SLAB_MB=1, so every member streams several slabs.  Every host result buffer starts poisoned with a byte
pattern that differs between the calls compared, so rows a group never writes cannot pass."""

import ctypes as C
import warnings

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from xgcm_b200 import _capi, ops

pytestmark = pytest.mark.gpu

GROUPS = [(0, 0), (0, 0, 0)]


@pytest.fixture(autouse=True)
def slab(monkeypatch):
    monkeypatch.setenv("XG_HOST_SLAB_MB", "1")


def _bits(a):
    return np.ascontiguousarray(np.asarray(a)).view(np.uint8)


def _as_list(r):
    return list(r) if isinstance(r, (list, tuple)) else [r]


_POISON = [0xA5]  # the byte every host result buffer starts as (ops.pinned_empty, below)


@pytest.fixture(autouse=True)
def poisoned_results(monkeypatch):
    """Every result buffer of an ops.*_host call is filled with the byte _POISON[0] before the call writes it."""
    real = ops.pinned_empty

    def poisoned(shape, dtype=np.float32):
        a = real(shape, dtype)
        a.reshape(-1).view(np.uint8).fill(_POISON[0])
        return a

    monkeypatch.setattr(ops, "pinned_empty", poisoned)


def _same(call, groups=GROUPS):
    """call(device) on device 0 and on every group in `groups`: bit for bit the same results.

    Each call's result buffers start as a byte pattern of their own, and every result stays referenced until all
    comparisons are done (so no buffer is handed back to the next call holding the answer already): a row that one
    call never writes differs from the other call's row."""
    runs = []
    for k, d in enumerate([0] + list(groups)):
        _POISON[0] = (0xA5, 0x5A, 0xC3, 0x3C)[k % 4]
        runs.append(_as_list(call(d)))
    want = runs[0]
    for g, got in zip(groups, runs[1:]):
        assert len(got) == len(want)
        for k, (w, x) in enumerate(zip(want, got)):
            assert x.shape == w.shape and x.dtype == w.dtype, (g, k)
            np.testing.assert_array_equal(_bits(x), _bits(w), err_msg=f"group {g}, result {k}")
    return want


def _rand(shape, dtype=np.float32, seed=0, nan=True):
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(shape).astype(dtype)
    if nan:
        a.reshape(-1)[rng.choice(a.size, size=min(a.size, 16), replace=False)] = np.nan
    return a


def _workspace_bytes(device):
    v = _capi.i64_array([0])
    _capi.check(_capi.load().xg_host_workspace_bytes(device, v))
    return int(v[0])


# ------------------------------------------------------------------------------------------------ the stencils
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("op, lo, hi, pad", [("diff", 1, 0, "periodic"), ("interp", 0, 1, "periodic"),
                                             ("diff", 1, 1, "extrapolate"), ("interp", 1, 0, "extrapolate"),
                                             ("diff", 0, 0, None), ("min", 1, 0, "fill"), ("max", 0, 1, "extend")])
def test_stencil2_along_dim_0(op, lo, hi, pad, dtype):
    """Dim 0 operated: blocks read the row next to them, the wrap planes go up once per member, extrapolate keeps
    two rows in the blocks at the field's edges.  37 rows: ragged blocks of 19 / 18 and 13 / 12 / 12."""
    x = _rand((37, 48, 96), dtype)
    post = (0.5 + np.random.default_rng(1).random((1, 48, 96))).astype(dtype)
    _same(lambda d: ops.stencil2_host(x, 0, op, lo, hi, pad, 1.5, device=d))
    if pad != "periodic":  # a pre-metric along dim 0 (periodic: the device entry point's case)
        pre = (0.5 + np.random.default_rng(2).random((37, 1, 96))).astype(dtype)
        _same(lambda d: ops.stencil2_host(x, 0, op, lo, hi, pad, 1.5, pre=pre, post=post, device=d))


@pytest.mark.parametrize("axis", [1, 2])
def test_stencil2_along_a_batch_dim(axis):
    x = _rand((29, 40, 72))
    _same(lambda d: ops.stencil2_host(x, axis, "diff", 1, 0, "periodic", device=d))


def test_stencil2_host_multi():
    x = _rand((31, 40, 96))
    specs = [(0, "diff", 1, 0, "periodic", 0.0), (0, "interp", 0, 1, "fill", 2.0), (1, "interp", 1, 0, "fill", 0.0),
             (2, "diff", 0, 1, "extend", 0.0), (2, "min", 1, 1, "periodic", 0.0)]
    _same(lambda d: ops.stencil2_host_multi(x, specs, device=d))


@pytest.mark.parametrize("specs", [
    [(2, "interp", 1, 0, "periodic", 0.0), (1, "interp", 1, 0, "fill", 0.0)],    # slab dim 0 not operated
    [(2, "diff", 1, 0, "periodic", 0.0), (0, "diff", 0, 1, "fill", 0.0)],        # slab dim 1, a middle dim
    [(2, "max", 0, 1, "periodic", 0.0), (1, "max", 1, 0, "fill", 0.0), (0, "max", 1, 0, "extend", 0.0)],  # all
])
def test_stencil_multi_host(specs):
    x = _rand((33, 40, 64))
    _same(lambda d: ops.stencil_multi_host(x, specs, device=d))


# --------------------------------------------------------------------------------- fold and face-connected halos
POS = ("center", "left", "right")


def _fold_grid(pivot, host_devices, ny=33, nx=40, dtype=np.float32):
    rng = np.random.default_rng(5)
    coords = {"x" + p: np.arange(nx) for p in POS}
    coords.update({"y" + p: np.arange(ny) for p in POS})
    data, reg = {}, {("X",): [], ("Y",): [], ("X", "Y"): []}
    for yp in POS:
        for xp in POS:
            for name, key in (("dx", ("X",)), ("dy", ("Y",)), ("area", ("X", "Y"))):
                data[f"{name}_{yp}_{xp}"] = (("y" + yp, "x" + xp), (0.5 + rng.random((ny, nx))).astype(dtype))
                reg[key].append(f"{name}_{yp}_{xp}")
    ds = xg.Dataset(data_vars=data, coords=coords)
    padding = {"X": "periodic", "Y": {"fold": pivot, "south": "fill"} if pivot else "fill"}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        return xg.Grid(ds, coords={"X": {p: "x" + p for p in POS}, "Y": {p: "y" + p for p in POS}}, padding=padding,
                       autoparse_metadata=False, metrics=reg, host_devices=host_devices)


def _grid_same(make_grid, call, groups=GROUPS):
    _same(lambda d: call(make_grid(None if d == 0 else d)), groups)


@pytest.mark.parametrize("pivot", ["T", "corner", None])
def test_fold_stencil_and_pair(pivot):
    """xg_stencil2_host_fold (interp to the right across the fold), xg_stencil_pair_host[_fold] (divergence and
    vorticity): 2 x 31 batch rows of (33, 40)."""
    u = xg.DataArray(_rand((2, 31, 33, 40), seed=3), dims=("t", "z", "ycenter", "xleft"))
    v = xg.DataArray(_rand((2, 31, 33, 40), seed=4), dims=("t", "z", "yleft", "xcenter"))
    c = xg.DataArray(_rand((2, 31, 33, 40), seed=6), dims=("t", "z", "ycenter", "xcenter"))
    to = {"X": "center", "Y": "center"}
    _grid_same(lambda h: _fold_grid(pivot, h), lambda g: g.interp(c, "Y", to="right").data)
    _grid_same(lambda h: _fold_grid(pivot, h), lambda g: g.diff(c, "Y", to="left").data)
    _grid_same(lambda h: _fold_grid(pivot, h), lambda g: g.divergence(u, v, to=to).data)
    _grid_same(lambda h: _fold_grid(pivot, h), lambda g: g.vorticity(v, u, to=to).data)


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


def test_face_connected_halos():
    n = 40
    coords = {"x": np.arange(n) + 0.0, "xl": np.arange(n) - 0.5, "y": np.arange(n) + 0.0, "yl": np.arange(n) - 0.5,
              "face": np.arange(6)}
    ds = xg.Dataset(data_vars={"c": (("t", "k", "face", "y", "x"), _rand((3, 5, 6, n, n), seed=7)),
                               "u": (("t", "k", "face", "y", "xl"), _rand((3, 5, 6, n, n), seed=8)),
                               "v": (("t", "k", "face", "yl", "x"), _rand((3, 5, 6, n, n), seed=9))}, coords=coords)

    def grid(h):
        return xg.Grid(ds, coords={"X": {"center": "x", "left": "xl"}, "Y": {"center": "y", "left": "yl"}},
                       face_connections=CUBED_SPHERE, host_devices=h)

    _grid_same(grid, lambda g: g.diff(ds["c"], "X").data)
    _grid_same(grid, lambda g: g.interp(ds["c"], "Y").data)
    _grid_same(grid, lambda g: g.diff({"X": ds["u"]}, "X", other_component={"Y": ds["v"]}).data)


def test_pair_host_with_metrics():
    a, b = _rand((23, 40, 64), seed=10), _rand((23, 40, 64), seed=11)
    pre_a = (0.5 + np.random.default_rng(12).random((1, 40, 64))).astype(np.float32)
    post = (0.5 + np.random.default_rng(13).random((23, 40, 64))).astype(np.float32)
    _same(lambda d: ops.stencil_pair_host(a, b, ("diff", 1, 0, "periodic", 0.0), (1, "diff", 0, 1, "fill", 0.0), 2,
                                          pre_a=pre_a, post=post, device=d))


# ------------------------------------------------------------------------------------ scans, reductions, transforms
@pytest.mark.parametrize("axis", [0, 2])  # axis 0: the slabs cut dim 1, a non-leading dim
def test_cumscan(axis):
    x = _rand((27, 35, 64))
    post = (0.5 + np.random.default_rng(14).random((27, 35, 64))).astype(np.float32)
    _same(lambda d: ops.cumscan_host(x, axis, reverse=True, device=d))
    _same(lambda d: ops.cumscan_host(x, axis, trim="drop_last", pad_lo=1, padding="fill", fill_value=0.0, post=post,
                                     device=d))


def test_wreduce_forms():
    x = _rand((26, 36, 64), np.float64)
    w = (0.5 + np.random.default_rng(15).random((26, 36, 64))).astype(np.float64)
    w2 = (0.5 + np.random.default_rng(16).random((1, 36, 64))).astype(np.float64)
    for mode in ("sum", "mean"):
        _same(lambda d: ops.wreduce_host(x, 1, w, mode, device=d))                 # one dim
        _same(lambda d: ops.wreduce_host_multi(x, [1, 2], w, mode, device=d))      # slab dim 0, weight streamed
        _same(lambda d: ops.wreduce_host_multi(x, [0, 2], w2, mode, device=d))     # slab dim 1, weight whole
        _same(lambda d: ops.wreduce_host_multi(x, [0, 1, 2], w, mode, device=d))  # every dim: first member alone


def test_transforms():
    rng = np.random.default_rng(17)
    nt, nz, ny, nx = 3, 12, 40, 64
    phi = _rand((nt, nz, ny, nx), seed=18)
    bounds = np.cumsum(0.5 + rng.random((nt, nz + 1, ny, nx)), axis=1).astype(np.float32)
    centres = np.cumsum(0.5 + rng.random((nt, nz, ny, nx)), axis=1).astype(np.float32)
    centres_1d = np.cumsum(0.5 + rng.random((1, nz, 1, 1)), axis=1).astype(np.float32)
    bins = np.linspace(0.0, float(bounds.max()) + 1, 15).astype(np.float32)
    levels = np.linspace(1.0, float(centres.max()), 20).astype(np.float32)
    _same(lambda d: ops.vinterp_conservative_host(phi, bounds, bins, 1, device=d))
    _same(lambda d: ops.vinterp_conservative_host(phi, centres, bins, 1, theta_at_centers=True, device=d))
    _same(lambda d: ops.vinterp_conservative_host(phi, centres_1d, bins, 1, theta_at_centers=True, device=d))
    _same(lambda d: ops.vinterp_linear_host(phi, centres, levels, 1, device=d))
    _same(lambda d: ops.vinterp_linear_host(phi, centres_1d, levels, 1, device=d))


def test_grid_routes_pass_the_group():
    """Grid(host_devices=...) on numpy fields: apply_many, multi-axis interp, cumsum, average and transform."""
    nz, ny, nx = 12, 40, 64
    rng = np.random.default_rng(19)
    ds = xg.Dataset(
        data_vars={"theta": (("z", "y", "x"), _rand((nz, ny, nx), seed=20)),
                   "tc": (("z", "y", "x"), np.cumsum(0.5 + rng.random((nz, ny, nx)), axis=0).astype(np.float32)),
                   "dz": (("z",), np.ones(nz, np.float32)), "area": (("y", "x"), np.ones((ny, nx), np.float32))},
        coords={"z": np.arange(nz) + 0.5, "zl": np.arange(nz) + 0.0, "y": np.arange(ny) + 0.5,
                "yl": np.arange(ny) + 0.0, "x": np.arange(nx) + 0.5, "xl": np.arange(nx) + 0.0})

    def grid(h):
        return xg.Grid(ds, coords={"X": {"center": "x", "left": "xl"}, "Y": {"center": "y", "left": "yl"},
                                   "Z": {"center": "z", "left": "zl"}},
                       padding={"X": "periodic", "Y": "fill", "Z": "extend"}, fill_value=0.0,
                       metrics={("Z",): ["dz"], ("X", "Y"): ["area"]}, autoparse_metadata=False, host_devices=h)

    th = ds["theta"]
    reqs = [(f, a) for a in ("X", "Y", "Z") for f in ("diff", "interp")]
    _grid_same(grid, lambda g: [r.data for r in g.apply_many(th, reqs)])
    _grid_same(grid, lambda g: g.interp(th, ["X", "Y"]).data)
    _grid_same(grid, lambda g: g.cumsum(th, "Z").data)
    _grid_same(grid, lambda g: g.average(th, ["X", "Y"]).data)
    levels = np.linspace(1.0, 10.0, 20).astype(np.float32)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _grid_same(grid, lambda g: g.transform(th, "Z", levels, target_data=ds["tc"], method="linear").data)


# ------------------------------------------------------------------------------------------------------ edge cases
def test_fewer_rows_than_members_and_short_extrapolated_fields():
    for n0 in (1, 2, 3, 5):
        x = _rand((n0, 24, 64), seed=n0)
        _same(lambda d: ops.stencil2_host(x, 1, "diff", 1, 0, "periodic", device=d))
        if n0 >= 2:  # extrapolate needs two rows; with three members and 3 or 5 rows, two blocks hold them
            _same(lambda d: ops.stencil2_host(x, 0, "interp", 1, 0, "extrapolate", device=d))
            _same(lambda d: ops.stencil2_host(x, 0, "diff", 1, 1, "extrapolate", device=d))


def test_calling_thread_keeps_the_first_members_label():
    x = _rand((30, 24, 64))
    ops.stencil2_host(x, 2, "diff", 1, 0, "periodic", device=0)
    want = _capi.last_launch()
    ops.wreduce_host(x, 1, device=0)
    assert _capi.last_launch() != want
    ops.stencil2_host(x, 2, "diff", 1, 0, "periodic", device=(0, 0, 0))
    assert _capi.last_launch() == want and want


def test_workspace_does_not_grow_over_the_single_device_call():
    x = _rand((41, 40, 96))
    bounds = np.cumsum(0.5 + np.random.default_rng(21).random((41, 13, 96)), axis=1).astype(np.float32)
    phi = _rand((41, 12, 96), seed=22)
    bins = np.linspace(0.0, 20.0, 9).astype(np.float32)
    calls = [lambda d: ops.stencil2_host(x, 0, "diff", 1, 0, "periodic", device=d),
             lambda d: ops.stencil2_host_multi(x, [(0, "interp", 1, 0, "fill", 0.0), (2, "diff", 1, 0, "extend", 0.0)],
                                               device=d),
             lambda d: ops.vinterp_conservative_host(phi, bounds, bins, 1, device=d)]
    for call in calls:
        _capi.check(_capi.load().xg_host_workspace_release())
        call(0)
        single = _workspace_bytes(0)
        assert single > 0
        for g in GROUPS:
            call(g)
            assert _workspace_bytes(0) == single, g


def test_argument_errors_through_a_group():
    lib = _capi.load()
    x = _rand((8, 16, 64))
    out = np.empty_like(x)
    shape = _capi.i64_array(x.shape)
    unknown = _capi.XG_HOST_GROUP_BASE + 63
    rc = lib.xg_stencil2_host(0, 0, x.ctypes.data, out.ctypes.data, 3, shape, 2, 1, 0, 1, 0.0, None, None, None,
                              None, unknown)
    assert rc == -1 and "unknown host device group" in _capi.last_error()
    with pytest.raises(ValueError, match="does not exist"):
        ops.stencil2_host(x, 2, "diff", 1, 0, "periodic", device=(0, torch.cuda.device_count()))
    with pytest.raises(ValueError, match="halo widths"):  # the entry point's own check, in front of the group
        lib_out = lib.xg_stencil2_host(0, 0, x.ctypes.data, out.ctypes.data, 3, shape, 2, 2, 0, 1, 0.0, None, None,
                                       None, None, ops.host_device_arg((0, 0)))
        _capi.check(lib_out)
    # the same member list gives the same handle
    h = C.c_int(0)
    _capi.check(lib.xg_host_group(2, (C.c_int * 2)(0, 0), C.byref(h)))
    assert h.value == ops.host_device_arg([0, 0]) >= _capi.XG_HOST_GROUP_BASE


# ---------------------------------------------------------------------------------------------- two or more GPUs
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("pinned", [True, False], ids=["page-locked", "pageable"])
def test_two_gpus_equal_device_0(pinned):
    x = _rand((37, 48, 96))
    if pinned:
        p = ops.pinned_empty(x.shape, x.dtype)
        p[...] = x
        x = p
    specs = [(0, "diff", 1, 0, "periodic", 0.0), (1, "interp", 1, 0, "fill", 0.0), (2, "diff", 1, 0, "extend", 0.0)]
    groups = [(0, 1), tuple(range(torch.cuda.device_count()))]
    _same(lambda d: ops.stencil2_host_multi(x, specs, device=d), groups)
    _same(lambda d: ops.stencil2_host(x, 0, "interp", 1, 0, "extrapolate", device=d), groups)
    _same(lambda d: ops.wreduce_host_multi(x, [1, 2], None, "mean", device=d), groups)
    pivot_grid = lambda h: _fold_grid("T", h)  # noqa: E731
    c = xg.DataArray(_rand((2, 31, 33, 40), seed=6), dims=("t", "z", "ycenter", "xcenter"))
    _same(lambda d: pivot_grid(None if d == 0 else "all").interp(c, "Y", to="right").data, ["all"])
    for dev in range(torch.cuda.device_count()):
        assert _workspace_bytes(dev) > 0, dev
