"""Grid.pair / divergence / vorticity across the north fold on the CPU: the C-ABI of xg_stencil_pair_halo and the
host pair twins (every argument checked before any CUDA call), and the routing of the two-field composites with the
kernels replaced by the oracle (tests/_mock_pair.py): which calls take the fused kernel with a fold halo plane, which
stream numpy fields through the host twins, and which keep the chain."""

import ctypes as C
import warnings

import numpy as np
import pytest

import xgcm_b200 as xg
from _mock_pair import install
from oracle import fold as F
from oracle import stencil as S
from xgcm_b200 import _build, _capi

# ---------------------------------------------------------------------------------------------- C-ABI
SHAPE = [4, 6, 5]  # (batch, y, x): axis_b = 1, the seam is x


@pytest.fixture(scope="module")
def lib():
    _build.build()
    return _capi.load()


def _pair_args(entry, **kw):
    a, b, out = (C.c_float * 128)(), (C.c_float * 128)(), (C.c_float * 128)()
    args = dict(dtype=0, a=a, b=b, out=out, ndim=3, shape=_capi.i64_array(SHAPE), op_a=0, lo_a=0, hi_a=1, bc_a=1,
                fill_a=0.0, pre_a=None, pre_a_st=None, axis_b=1, op_b=0, lo_b=0, hi_b=1, bc_b=2, fill_b=0.0,
                pre_b=None, pre_b_st=None, sub=0, post=None, post_st=None)
    if entry == "halo":
        args.update(halo_lo=None, halo_hi=None, stream=None)
    elif entry == "host":
        args.update(device=0)
    else:
        args.update(seam=2, skip=0, mirror=0, period=5, negate=1, device=0)
    args.update(kw)
    return list(args.values())


def _rc(lib, entry, **kw):
    fn = {"halo": lib.xg_stencil_pair_halo, "host": lib.xg_stencil_pair_host,
          "fold": lib.xg_stencil_pair_host_fold}[entry]
    return fn(*_pair_args(entry, **kw))


def _fails(rc, code, text):
    assert rc == code, (rc, _capi.last_error())
    assert text in _capi.last_error(), _capi.last_error()


@pytest.mark.parametrize("entry", ["halo", "host", "fold"])
def test_pair_entry_points_validate_without_gpu(lib, entry):
    for name in ("a", "b", "out", "shape"):
        _fails(_rc(lib, entry, **{name: None}), -1, "null pointer")
    _fails(_rc(lib, entry, axis_b=2), -1, "innermost")
    _fails(_rc(lib, entry, lo_b=1), -2, "length preserving")
    _fails(_rc(lib, entry, bc_b=4), -1, "periodic, fill or extend")
    _fails(_rc(lib, entry, op_a=7), -1, "unknown op")
    _fails(_rc(lib, entry, sub=3), -1, "subtract")
    _fails(_rc(lib, entry, pre_a=(C.c_float * 4)()), -1, "strides missing")
    _fails(_rc(lib, entry, dtype=5), -1, "dtype")
    if entry == "halo":
        buf = (C.c_float * 128)()
        _fails(_rc(lib, entry, out=buf, halo_hi=buf), -1, "halo plane")


@pytest.mark.parametrize("entry", ["host", "fold"])
def test_host_pair_dim0_must_be_a_batch_dim(lib, entry):
    _fails(_rc(lib, entry, axis_b=0), -1, "dim 0")  # the operated (fold) dim would be cut into slabs
    _fails(_rc(lib, entry, ndim=2, shape=_capi.i64_array([6, 5]), axis_b=0), -1, "dim 0")  # (y, x): no batch dim


def test_host_pair_fold_parameters(lib):
    _fails(_rc(lib, "fold", seam=0), -1, "seam dim")
    _fails(_rc(lib, "fold", seam=1), -1, "fold and seam axes must differ")
    _fails(_rc(lib, "fold", seam=3), -1, "seam axis out of range")
    _fails(_rc(lib, "fold", lo_b=1, hi_b=0), -1, "hi must be 1")
    _fails(_rc(lib, "fold", skip=2), -1, "skip")
    _fails(_rc(lib, "fold", period=0), -1, "period")
    _fails(_rc(lib, "fold", shape=_capi.i64_array([4, 1, 5]), skip=1), -1, "interior rows")
    _fails(_rc(lib, "fold", mirror=-1, period=6), -2, "incompatible")


# ---------------------------------------------------------------------------------------------- routing
NX, NY = 8, 5


@pytest.fixture
def calls(monkeypatch):
    """Install the oracle-backed kernels and record which pair entry points each Grid call reaches."""
    from xgcm_b200 import ops

    install(monkeypatch)
    log = []
    for name in ("stencil_pair", "stencil_pair_host", "stencil_pair_host_fold"):
        def wrap(*args, _fn=getattr(ops, name), _name=name, **kw):
            log.append((_name, args, kw))
            return _fn(*args, **kw)

        monkeypatch.setattr(ops, name, wrap)
    return log


def _grid(pivot="corner", south="fill"):
    rng = np.random.default_rng(0)
    data = {"dyu": (("ycenter", "xleft"), 1 + rng.random((NY, NX))), "dxv": (("yleft", "xcenter"), 1 + rng.random((NY, NX))),
            "area": (("ycenter", "xcenter"), 1 + rng.random((NY, NX)))}
    coords = {"xcenter": np.arange(NX), "xleft": np.arange(NX), "ycenter": np.arange(NY), "yleft": np.arange(NY)}
    ds = xg.Dataset(data_vars=data, coords=coords)
    padding = {"X": "periodic", "Y": {"fold": pivot, "south": south} if pivot else south}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        grid = xg.Grid(ds, coords={"X": {"center": "xcenter", "left": "xleft"},
                                   "Y": {"center": "ycenter", "left": "yleft"}},
                       padding=padding, autoparse_metadata=False)
    grid.set_metrics("Y", "dyu")
    grid.set_metrics("X", "dxv")
    grid.set_metrics(("X", "Y"), "area")
    return ds, grid


def _divergence_oracle(ds, u, v, pivot, south, fold=True):
    tx = S.stencil2("diff", u * ds["dyu"].values, u.ndim - 1, 0, 1, "periodic")
    vd = v * ds["dxv"].values
    fa = v.ndim - 2
    if fold:
        padded = F.pad_fold(vd, fa, fa + 1, "left", "center", F.resolve_pivot(pivot, "Y", "X"), {fa: (0, 1)},
                            {fa: south}, vector=True)
        ty = S.stencil2("diff", padded, fa, 0, 0, None)
    else:
        ty = S.stencil2("diff", vd, fa, 0, 1, south)
    return (tx + ty) / ds["area"].values


def test_fold_pair_fuses_with_a_halo_plane(calls):
    ds, grid = _grid("corner", "fill")
    rng = np.random.default_rng(1)
    u, v = rng.random((NY, NX)), rng.random((NY, NX))
    got = grid.divergence(xg.DataArray(u, dims=("ycenter", "xleft")), xg.DataArray(v, dims=("yleft", "xcenter")))
    [(name, args, kw)] = calls
    assert name == "stencil_pair" and kw["halo_lo_b"] is None and kw["halo_hi_b"] is not None
    assert tuple(kw["halo_hi_b"].shape) == (1, NX)
    np.testing.assert_array_equal(got.values, _divergence_oracle(ds, u, v, "corner", "fill"))
    # the pole row folds v as a vector: its sign flips (halo = -(v * dxv) at the mirrored cell)
    roles = F.resolve_pivot("corner", "Y", "X")
    want = -F.north_rows(v * ds["dxv"].values, 0, 1, "left", "center", roles, 1)
    np.testing.assert_array_equal(kw["halo_hi_b"].numpy(), want)


def test_fold_pair_lower_halo_stays_a_boundary_condition(calls):
    """center -> left pads only the south edge: no fold plane, the south mode pads it (also when periodic)."""
    ds, grid = _grid("corner", "periodic")
    rng = np.random.default_rng(2)
    u, v = rng.random((NY, NX)), rng.random((NY, NX))
    got = grid.pair("diff", xg.DataArray(u, dims=("yleft", "xcenter")), "X", "interp",
                    xg.DataArray(v, dims=("ycenter", "xleft")), "Y", combine="sub", to={"X": "left", "Y": "left"})
    [(name, _, kw)] = calls
    assert name == "stencil_pair" and kw.get("halo_lo_b") is None and kw.get("halo_hi_b") is None
    want = S.stencil2("diff", u, 1, 1, 0, "periodic") - S.stencil2("interp", v, 0, 1, 0, "periodic")
    np.testing.assert_array_equal(got.values, want)


def test_fold_halo_planes_south_rule(monkeypatch):
    """The one rule both the single operators and the pair use: the fold row is halo_lo only for lo = 1 under a
    periodic south edge."""
    import torch

    from xgcm_b200.padding import fold_halo_planes

    install(monkeypatch)
    _, grid = _grid("corner", "fill")
    x = torch.from_numpy(np.random.default_rng(3).random((NY, NX)))
    dims = ("ycenter", "xcenter")
    for lo, south, has_lo in ((1, "periodic", True), (1, "fill", False), (1, "extend", False), (0, "periodic", False)):
        lo_plane, hi_plane = fold_halo_planes(grid, "Y", dims, x, lo, south)
        assert hi_plane is not None and tuple(hi_plane.shape) == (1, NX)
        assert (lo_plane is hi_plane) if has_lo else lo_plane is None, (lo, south)


@pytest.mark.parametrize("south", ["fill", "periodic", "extend"])
def test_numpy_fields_stream_through_the_host_twins(calls, south):
    ds, grid = _grid("U", south)
    rng = np.random.default_rng(4)
    u, v = rng.random((2, 3, NY, NX)), rng.random((2, 3, NY, NX))
    got = grid.divergence(xg.DataArray(u, dims=("t", "z", "ycenter", "xleft")),
                          xg.DataArray(v, dims=("t", "z", "yleft", "xcenter")))
    name, args, kw = calls[0]  # (the oracle stand-in of the host twin then calls the device stand-in)
    assert name == "stencil_pair_host_fold"
    a, b, spec_a, spec_b, seam = args[:5]
    assert a.shape == b.shape == (6, NY, NX) and spec_b[0] == 1 and seam == 2
    assert kw["negate"] is True and kw["pre_b"].shape == (1, NY, NX)
    assert got.dims == ("t", "z", "ycenter", "xcenter") and isinstance(got.data, np.ndarray)
    np.testing.assert_array_equal(got.values, _divergence_oracle(ds, u, v, "U", south))
    # per-call padding string: X and the south edge extend, the north edge still folds
    calls.clear()
    got = grid.divergence(xg.DataArray(u, dims=("t", "z", "ycenter", "xleft")),
                          xg.DataArray(v, dims=("t", "z", "yleft", "xcenter")), padding="extend")
    assert calls[0][0] == "stencil_pair_host_fold"
    tx = S.stencil2("diff", u * ds["dyu"].values, 3, 0, 1, "extend")
    padded = F.pad_fold(v * ds["dxv"].values, 2, 3, "left", "center", F.resolve_pivot("U", "Y", "X"), {2: (0, 1)},
                        {2: "extend"}, vector=True)
    np.testing.assert_array_equal(got.values, (tx + S.stencil2("diff", padded, 2, 0, 0, None)) / ds["area"].values)


def test_plain_grid_numpy_pair_streams_and_2d_stays_whole(calls):
    ds, grid = _grid(None, "fill")
    rng = np.random.default_rng(5)
    u, v = rng.random((1, 4, NY, NX)), rng.random((1, 4, NY, NX))
    got = grid.divergence(xg.DataArray(u, dims=("one", "z", "ycenter", "xleft")),
                          xg.DataArray(v, dims=("one", "z", "yleft", "xcenter")))
    name, args, kw = calls[0]  # (the oracle stand-in of the host twin then calls the device stand-in)
    assert name == "stencil_pair_host" and args[0].shape == (4, NY, NX) and args[3][0] == 1  # leading 1 dropped
    np.testing.assert_array_equal(got.values, _divergence_oracle(ds, u, v, None, "fill", fold=False))
    calls.clear()
    grid.divergence(xg.DataArray(u[0, 0], dims=("ycenter", "xleft")), xg.DataArray(v[0, 0], dims=("yleft", "xcenter")))
    assert [c[0] for c in calls] == ["stencil_pair"]


def test_fold_axis_innermost_keeps_the_chain(calls):
    ds, grid = _grid("corner", "fill")
    rng = np.random.default_rng(6)
    u, v = rng.random((NX, NY)), rng.random((NX, NY))
    got = grid.pair("diff", xg.DataArray(u, dims=("xleft", "ycenter")), "X", "diff",
                    xg.DataArray(v, dims=("xcenter", "yleft")), "Y")
    assert calls == []
    padded = F.pad_fold(v, 1, 0, "left", "center", F.resolve_pivot("corner", "Y", "X"), {1: (0, 1)}, {1: "fill"})
    np.testing.assert_array_equal(got.values, S.stencil2("diff", u, 0, 0, 1, "periodic")
                                  + S.stencil2("diff", padded, 1, 0, 0, None))


def test_face_connections_keep_the_chain(calls):
    n = 6
    ds = xg.Dataset(coords={"x": np.arange(n), "xl": np.arange(n), "y": np.arange(n), "yl": np.arange(n),
                            "face": np.arange(2)})
    grid = xg.Grid(ds, coords={"X": {"center": "x", "left": "xl"}, "Y": {"center": "y", "left": "yl"}},
                   face_connections={"face": {0: {"X": (None, (1, "X", False))}, 1: {"X": ((0, "X", False), None)}}},
                   padding="fill")
    rng = np.random.default_rng(7)
    u, v = rng.random((2, n, n)), rng.random((2, n, n))
    got = grid.pair("diff", xg.DataArray(u, dims=("face", "y", "xl")), "X", "diff",
                    xg.DataArray(v, dims=("face", "yl", "x")), "Y")
    assert calls == []
    assert got.dims == ("face", "y", "x")
