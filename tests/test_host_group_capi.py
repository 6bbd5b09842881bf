"""Host device groups without a GPU: xg_host_group is exported and checks its arguments before any CUDA call; every
slab-streaming host entry point refuses an unregistered group handle with XG_EINVAL before any CUDA call (a CUDA
call here would fail with XG_ECUDA); and Grid(host_devices=...) hands the group to the host twins for numpy fields
only (ops patched to record their arguments)."""

import ctypes as C
import warnings

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from xgcm_b200 import _build, _capi

EINVAL = -1
UNKNOWN = _capi.XG_HOST_GROUP_BASE + 63  # the last handle of the table: never registered in this process


@pytest.fixture(scope="module")
def lib():
    _build.build()
    return _capi.load()


def _ints(*v):
    return (C.c_int * len(v))(*v)


def _f64(*v):
    return (C.c_double * len(v))(*v)


def test_symbol_is_exported(lib):
    assert hasattr(C.CDLL(str(_capi.LIB_PATH)), "xg_host_group")
    assert "xg_host_group" in _capi.SIGNATURES


def test_host_group_checks_arguments_without_gpu(lib):
    handle = C.c_int(-7)
    cases = [
        (dict(devices=None), "null pointer"),
        (dict(group=None), "null pointer"),
        (dict(n=0), "between 1 and 64 members"),
        (dict(n=-1), "between 1 and 64 members"),
        (dict(n=65, devices=(C.c_int * 65)()), "between 1 and 64 members"),
        (dict(devices=_ints(0, -1)), "negative device index"),
    ]
    for kw, msg in cases:
        args = dict(n=2, devices=_ints(0, 0), group=C.byref(handle))
        args.update(kw)
        assert lib.xg_host_group(args["n"], args["devices"], args["group"]) == EINVAL, kw
        assert _capi.last_error().startswith("xg_host_group: ") and msg in _capi.last_error(), _capi.last_error()
    assert handle.value == -7  # nothing written on an error


def test_workspace_bytes_takes_device_indices_only(lib):
    n = C.c_int64(5)
    for who in ("xg_host_workspace_bytes", "xg_host_pipe_workspace_bytes"):
        assert getattr(lib, who)(_capi.XG_HOST_GROUP_BASE, C.byref(n)) == EINVAL
        assert "not a host device group" in _capi.last_error()


def _entry_point_calls(lib, dev):
    """One call with valid arguments of every host entry point that streams slabs, on `dev`."""
    a, b, o = (C.c_float * 64)(), (C.c_float * 64)(), (C.c_float * 64)()
    th = (C.c_float * 64)(*range(64))
    i64 = _capi.i64_array
    s3 = i64([2, 4, 6])
    outs = (C.c_void_p * 2)(C.addressof(o), C.addressof(b))
    return {
        "xg_stencil2_host": lambda: lib.xg_stencil2_host(0, 0, a, o, 3, s3, 2, 1, 0, 1, 0.0, None, None, None, None,
                                                         dev),
        "xg_stencil2_host_fold": lambda: lib.xg_stencil2_host_fold(0, 0, a, o, 3, s3, 1, 0, 1, 2, 0.0, None, None,
                                                                   None, None, 2, 0, 5, 6, 0, dev),
        "xg_stencil2_host_connected": lambda: lib.xg_stencil2_host_connected(
            0, 0, a, None, None, o, 3, s3, 1, 0, 0, 0.0, None, None, 0, 3, None, None, None, None, None, None, None,
            None, dev),
        "xg_stencil_pair_host": lambda: lib.xg_stencil_pair_host(0, a, b, o, 3, s3, 0, 1, 0, 1, 0.0, None, None, 1, 0,
                                                                 1, 0, 1, 0.0, None, None, 0, None, None, dev),
        "xg_stencil_pair_host_fold": lambda: lib.xg_stencil_pair_host_fold(
            0, a, b, o, 3, s3, 0, 1, 0, 1, 0.0, None, None, 1, 0, 0, 1, 2, 0.0, None, None, 0, None, None, 2, 0, 5, 6,
            0, dev),
        "xg_stencil2_host_multi": lambda: lib.xg_stencil2_host_multi(2, _ints(0, 1), 0, a, outs, 3, s3, _ints(2, 1),
                                                                     _ints(1, 0), _ints(0, 1), _ints(1, 2),
                                                                     _f64(0.0, 0.0), dev),
        "xg_stencil_multi_host": lambda: lib.xg_stencil_multi_host(0, a, o, 3, s3, 2, _ints(2, 1), _ints(1, 1),
                                                                   _ints(1, 1), _ints(0, 0), _ints(2, 2),
                                                                   _f64(0.0, 0.0), dev),
        "xg_cumscan_host": lambda: lib.xg_cumscan_host(0, a, o, 3, s3, 2, 0, 0, 0, 0, 0, 0.0, None, None, None, None,
                                                       1, dev),
        "xg_wreduce_host": lambda: lib.xg_wreduce_host(0, a, None, None, o, 3, s3, 2, 0, 1, dev),
        "xg_wreduce_host_multi": lambda: lib.xg_wreduce_host_multi(0, a, None, None, o, 3, s3, 2, _ints(2, 1), 1, 1,
                                                                   dev),
        "xg_vinterp_linear_host": lambda: lib.xg_vinterp_linear_host(0, a, th, i64([24, 6, 1]), th, None, 3, o, 3, s3,
                                                                     2, 1, 1, 0, dev),
        "xg_vinterp_conservative_host": lambda: lib.xg_vinterp_conservative_host(0, a, th, i64([28, 7, 1]), 0, th, 3,
                                                                                 0, o, 3, s3, 2, dev),
    }


def test_every_entry_point_refuses_an_unknown_group_before_cuda(lib):
    calls = _entry_point_calls(lib, UNKNOWN)
    assert len(calls) == 12
    for who, call in calls.items():
        assert call() == EINVAL, who
        assert _capi.last_error() == f"{who}: unknown host device group {UNKNOWN}", _capi.last_error()
    # a handle past the table's range is unknown too
    assert _entry_point_calls(lib, _capi.XG_HOST_GROUP_BASE + 10 ** 6)["xg_stencil2_host"]() == EINVAL


# ---------------------------------------------------------------------------------------------- Grid routing
class _Routed(Exception):
    pass


HOST_OPS = ("stencil2_host", "stencil2_host_fold", "stencil2_host_connected", "stencil_pair_host",
            "stencil_pair_host_fold", "stencil2_host_multi", "stencil_multi_host", "cumscan_host", "wreduce_host",
            "wreduce_host_multi", "vinterp_linear_host", "vinterp_conservative_host")


@pytest.fixture
def routed(monkeypatch):
    """The oracle-backed CPU ops, a grid device of type cuda, and every ops.*_host replaced by a recorder."""
    from _mock_backend import install

    from xgcm_b200 import device, ops

    install(monkeypatch)
    monkeypatch.setattr(device, "default_device", lambda: torch.device("cuda"))
    monkeypatch.setattr(torch.cuda, "device_count", lambda: 3)
    calls = []

    def recorder(name):
        def record(*args, device=None, **kw):
            calls.append((name, device))
            raise _Routed(name)

        return record

    for name in HOST_OPS:
        monkeypatch.setattr(ops, name, recorder(name))
    return calls


def _grid(host_devices):
    nz, ny, nx = 4, 5, 40
    rng = np.random.default_rng(0)
    ds = xg.Dataset(
        data_vars={"theta": (("z", "y", "x"), rng.random((nz, ny, nx)).astype(np.float32)),
                   "dz": (("z",), np.ones(nz)), "area": (("y", "x"), np.ones((ny, nx)))},
        coords={"z": np.arange(nz) + 0.5, "zl": np.arange(nz) + 0.0, "y": np.arange(ny) + 0.5,
                "yl": np.arange(ny) + 0.0, "x": np.arange(nx) + 0.5, "xl": np.arange(nx) + 0.0})
    return ds, xg.Grid(ds, coords={"X": {"center": "x", "left": "xl"}, "Y": {"center": "y", "left": "yl"},
                                   "Z": {"center": "z", "left": "zl"}},
                       padding={"X": "periodic", "Y": "fill", "Z": "extend"}, fill_value=0.0,
                       metrics={("Z",): ["dz"], ("X", "Y"): ["area"]}, autoparse_metadata=False,
                       host_devices=host_devices)


POS = ("center", "left", "right")


def _fold_grid(pivot, host_devices, ny=9, nx=40):
    """X periodic, Y folding under `pivot` (plain fill for None), dx / dy / area at every (Y, X) position."""
    rng = np.random.default_rng(1)
    coords = {"x" + p: np.arange(nx) for p in POS}
    coords.update({"y" + p: np.arange(ny) for p in POS})
    data, reg = {}, {("X",): [], ("Y",): [], ("X", "Y"): []}
    for yp in POS:
        for xp in POS:
            for name, key in (("dx", ("X",)), ("dy", ("Y",)), ("area", ("X", "Y"))):
                data[f"{name}_{yp}_{xp}"] = (("y" + yp, "x" + xp), (0.5 + rng.random((ny, nx))).astype(np.float32))
                reg[key].append(f"{name}_{yp}_{xp}")
    ds = xg.Dataset(data_vars=data, coords=coords)
    padding = {"X": "periodic", "Y": {"fold": pivot, "south": "fill"} if pivot else "fill"}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        return xg.Grid(ds, coords={"X": {p: "x" + p for p in POS}, "Y": {p: "y" + p for p in POS}}, padding=padding,
                       autoparse_metadata=False, metrics=reg, host_devices=host_devices)


def _fold_fields(ny=9, nx=40):
    rng = np.random.default_rng(2)
    f = lambda dims: xg.DataArray(rng.random((2, 3, ny, nx)).astype(np.float32), dims=("t", "z") + dims)  # noqa
    return f(("ycenter", "xleft")), f(("yleft", "xcenter")), f(("ycenter", "xcenter"))


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


def _connected(host_devices):
    n = 8
    ds = xg.Dataset(data_vars={"c": (("t", "k", "face", "y", "x"),
                                     np.random.default_rng(3).random((2, 3, 6, n, n)).astype(np.float32))},
                    coords={"x": np.arange(n) + 0.0, "xl": np.arange(n) - 0.5, "y": np.arange(n) + 0.0,
                            "yl": np.arange(n) - 0.5, "face": np.arange(6)})
    grid = xg.Grid(ds, coords={"X": {"center": "x", "left": "xl"}, "Y": {"center": "y", "left": "yl"}},
                   face_connections=CUBED_SPHERE, host_devices=host_devices)
    return lambda: grid.diff(ds["c"], "X")


def _transform(method, host_devices):
    rng = np.random.default_rng(4)
    nt, nz, ny, nx = 2, 6, 5, 8
    dims = ("t", "z", "y", "x")
    ds = xg.Dataset(data_vars={"q": (dims, rng.random((nt, nz, ny, nx)).astype(np.float32)),
                               "tc": (dims, np.cumsum(0.5 + rng.random((nt, nz, ny, nx)), 1).astype(np.float32)),
                               "sig": (("t", "zo", "y", "x"),
                                       np.cumsum(0.5 + rng.random((nt, nz + 1, ny, nx)), 1).astype(np.float32))},
                    coords={"z": np.arange(nz) + 0.5, "zo": np.arange(nz + 1.0)})
    grid = xg.Grid(ds, coords={"Z": {"center": "z", "outer": "zo"}}, host_devices=host_devices)
    theta = "tc" if method == "linear" else "sig"
    target = np.linspace(1.0, 5.0, 7).astype(np.float32)

    def call():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return grid.transform(ds["q"], "Z", target, target_data=ds[theta], method=method)

    return call


def _plain_route(fn):
    def case(host_devices):
        ds, grid = _grid(host_devices)
        return lambda: fn(grid, ds["theta"])

    return case


def _fold_route(pivot, fn):
    def case(host_devices):
        grid = _fold_grid(pivot, host_devices)
        u, v, c = _fold_fields()
        return lambda: fn(grid, u, v, c)

    return case


TO = {"X": "center", "Y": "center"}
PLAIN = [
    ("stencil2_host", lambda g, a: g.diff(a, "X")),
    ("stencil2_host_multi", lambda g, a: g.apply_many(a, [("diff", "X"), ("interp", "Y")])),
    ("stencil_multi_host", lambda g, a: g.interp(a, ["X", "Y"])),
    ("cumscan_host", lambda g, a: g.cumsum(a, "Z")),
    ("wreduce_host", lambda g, a: g.integrate(a, "Z")),
    ("wreduce_host_multi", lambda g, a: g.average(a, ["X", "Y"])),
]
ROUTES = [(name, _plain_route(fn)) for name, fn in PLAIN] + [
    ("stencil2_host_fold", _fold_route("T", lambda g, u, v, c: g.interp(c, "Y", to="right"))),
    ("stencil_pair_host", _fold_route(None, lambda g, u, v, c: g.divergence(u, v, to=TO))),
    ("stencil_pair_host_fold", _fold_route("T", lambda g, u, v, c: g.divergence(u, v, to=TO))),
    ("stencil_pair_host_fold", _fold_route("T", lambda g, u, v, c: g.vorticity(v, u, to=TO))),
    ("stencil2_host_connected", _connected),
    ("vinterp_linear_host", lambda h: _transform("linear", h)),
    ("vinterp_conservative_host", lambda h: _transform("conservative", h)),
]


@pytest.mark.parametrize("host_devices, want", [((0, 1), (0, 1)), ([2, 2, 0], (2, 2, 0)), (np.array([1, 0]), (1, 0)),
                                                ("all", (0, 1, 2))])
def test_numpy_fields_pass_the_group(routed, host_devices, want):
    for name, case in ROUTES:
        call = case(host_devices)
        routed.clear()
        with pytest.raises(_Routed):
            call()
        assert routed == [(name, want)], (name, routed)


def test_without_host_devices_numpy_fields_keep_the_grid_device(routed):
    for name, case in ROUTES:
        call = case(None)
        routed.clear()
        with pytest.raises(_Routed):
            call()
        assert routed == [(name, None)], (name, routed)  # torch.device("cuda").index: the current device


def test_device_tensors_never_reach_the_host_twins(routed):
    ds, grid = _grid((0, 1))
    da = ds["theta"]
    t = xg.DataArray(torch.from_numpy(np.asarray(da.data)), dims=da.dims, coords=da.coords)
    for _, fn in PLAIN:
        fn(grid, t)
    assert routed == []


@pytest.mark.parametrize("bad, exc", [((), ValueError), ((0, -1), ValueError), ((0, 1.0), ValueError),
                                      ((True,), ValueError), ("cuda", TypeError), (3, TypeError)])
def test_grid_refuses_bad_host_devices(bad, exc):
    ds = xg.Dataset(data_vars={}, coords={"x": np.arange(4) + 0.5})
    with pytest.raises(exc):
        xg.Grid(ds, coords={"X": {"center": "x"}}, autoparse_metadata=False, host_devices=bad)
