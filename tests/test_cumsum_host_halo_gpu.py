"""Grid.cumsum / cumint of numpy fields on face-connected and north-fold grids stream through the host slab
pipelines (xg_cumscan_host_connected / xg_cumscan_host_fold, or xg_cumscan_host where no halo crosses a seam):
bit for bit equal to the same call on device tensors and to the oracle (scan, then pad across the faces or the
fold, then divide), with device memory bounded by the slab size.  XG_HOST_SLAB_MB=1 forces at least four slabs
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

N = 48
LEAD = (3, 5)  # (time, k): 15 slab rows of 6 x 48 x 48 cells -> slabs of 4, 4, 4, 3 at 1 MiB
COORDS = {"X": {"center": "x", "left": "xl", "outer": "xo"}, "Y": {"center": "y", "left": "yl", "outer": "yo"},
          "Z": {"center": "k", "left": "kl"}}
AXES = {"X": ("x", "xl", "xo"), "Y": ("y", "yl", "yo")}
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


@pytest.fixture(autouse=True)
def slab(monkeypatch):
    monkeypatch.setenv("XG_HOST_SLAB_MB", "1")


@pytest.fixture
def spy(monkeypatch):
    """Names of the streamed cumscan entry points each call ran."""
    ran = []
    for name in ("cumscan_host", "cumscan_host_fold", "cumscan_host_connected"):
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


def _cumsum_oracle(a, axis, reverse, trim, pre, post, pad):
    """scan (oracle.stencil.cumscan, no pad) -> the padding function ``pad`` of the scanned array -> / post."""
    scanned = S.cumscan(a, axis, reverse, trim, 0, 0, None, 0.0, pre, None)
    r = pad(scanned)
    return r if post is None else r / post


# ------------------------------------------------------------------ face connections
def _faces_grid(dtype, fc=CUBED_SPHERE, lead=LEAD, lead_dims=("time", "k"), seed=0, nan=False):
    rng = np.random.default_rng(seed)
    nf = len(fc["face"])
    shape = lead + (nf, N, N)
    coords = {"x": np.arange(N) + 0.0, "xl": np.arange(N) - 0.5, "xo": np.arange(N + 1) - 0.5,
              "y": np.arange(N) + 0.0, "yl": np.arange(N) - 0.5, "yo": np.arange(N + 1) - 0.5,
              "face": np.arange(nf), "k": np.arange(lead[-1]) + 0.0, "kl": np.arange(lead[-1]) - 0.5,
              "dx_c": (("face", "y", "x"), 1.0 + rng.random((nf, N, N))),
              "dx_o": (("face", "y", "xo"), 1.0 + rng.random((nf, N, N + 1)))}
    c = rng.standard_normal(shape).astype(dtype)
    if nan:
        c[rng.random(shape) < 0.05] = np.nan
    ds = xg.Dataset(data_vars={"c": (lead_dims + ("face", "y", "x"), c),
                               "u": (lead_dims + ("face", "y", "xl"), rng.standard_normal(shape).astype(dtype)),
                               "v": (lead_dims + ("face", "yl", "x"), rng.standard_normal(shape).astype(dtype))},
                    coords=coords)
    return ds, xg.Grid(ds, coords=COORDS, face_connections=fc, metrics={("X",): ["dx_c", "dx_o"]})


def _faces_pad(fc, dims, ax, lo, hi, padding, fill):
    return lambda s: pad_face_connections(s, dims, AXES, "face", fc["face"], {ax: (lo, hi)},
                                          {a: padding for a in AXES}, {a: fill for a in AXES})


def _table(src, to, reverse):
    from xgcm_b200.grid import _CUMSUM_FWD, _CUMSUM_REV

    return (_CUMSUM_REV if reverse else _CUMSUM_FWD)[(src, to)]


# every (axis, field, its dim along the axis, to, reverse, trim, pad widths) that pads: across a seam that swaps
# axes the reference needs the untrimmed entries (a trimmed array has faces of unequal size); the strip has none
def _faces_cases(fc):
    for ax in ("X", "Y"):
        cases = [("c", "outer", False), ("c", "outer", True)]
        if fc is STRIP:
            cases += [("c", "left", False), ("u" if ax == "X" else "v", "center", True)]
        for field, to, reverse in cases:
            src = "center" if field == "c" else "left"
            trim, (lo, hi) = _table(src, to, reverse)
            yield ax, field, AXES[ax][0 if src == "center" else 1], to, reverse, trim, lo, hi


@pytest.mark.parametrize("fc", [CUBED_SPHERE, STRIP], ids=["cubed_sphere", "strip"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_faces_every_padded_entry_and_padding(fc, dtype, spy):
    ds, grid = _faces_grid(dtype, fc=fc, nan=True)
    checked = 0
    for (padding, fill), (ax, field, dim, to, reverse, trim, lo, hi) in itertools.product(PADDINGS, _faces_cases(fc)):
        da = ds[field]
        kw = dict(to=to, reverse=reverse, padding=padding, fill_value=fill)
        spy.clear()
        got = grid.cumsum(da, ax, **kw)
        # the strip has no connection along Y: its Y edges take the basic boundary in xg_cumscan_host
        assert spy == ["cumscan_host_connected" if ax in fc["face"][0] else "cumscan_host"], (ax, field, to)
        dev = grid.cumsum(_on_device(da), ax, **kw)
        want = _cumsum_oracle(da.values, da.dims.index(dim), reverse, trim, None, None,
                              _faces_pad(fc, da.dims, ax, lo, hi, padding, fill))
        _same(got, dev, want, f"{ax} {field} -> {to} reverse={reverse} {padding} {fill}")
        checked += 1
    assert checked == len(PADDINGS) * (4 if fc is CUBED_SPHERE else 8)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_faces_cumint_and_metric_weighted(dtype, spy):
    ds, grid = _faces_grid(dtype, nan=True)
    c = ds["c"]
    dx_c, dx_o = ds["dx_c"].values.astype(dtype), ds["dx_o"].values.astype(dtype)  # rounded to the field's dtype
    pad = _faces_pad(CUBED_SPHERE, c.dims, "X", 0, 1, None, 0.0)
    spy.clear()
    got = grid.cumint(c, "X", to="outer", reverse=True)
    assert spy == ["cumscan_host_connected"]
    _same(got, grid.cumint(_on_device(c), "X", to="outer", reverse=True),
          _cumsum_oracle(c.values, 4, True, "none", dx_c, None, pad), "cumint")
    got = grid.cumsum(c, "X", to="outer", reverse=True, metric_weighted="X")
    _same(got, grid.cumsum(_on_device(c), "X", to="outer", reverse=True, metric_weighted="X"),
          _cumsum_oracle(c.values, 4, True, "none", dx_c, dx_o, pad), "metric_weighted")


def test_faces_axes_that_need_no_seam(spy):
    """Z on a face-connected grid, and a shift that pads nothing, run xg_cumscan_host; Z takes its own boundary,
    and none at all is the missing-boundary error of pad()."""
    ds, grid = _faces_grid(np.float32)
    c = ds["c"]
    for kw in (dict(padding="fill", fill_value=1.5), dict(padding="extend"), dict(padding="periodic")):
        spy.clear()
        got = grid.cumsum(c, "Z", to="left", **kw)
        assert spy == ["cumscan_host"]
        want = S.cumscan(c.values, 1, False, "drop_last", 1, 0, kw["padding"], kw.get("fill_value", 0.0))
        _same(got, grid.cumsum(_on_device(c), "Z", to="left", **kw), want, f"Z {kw}")
    with pytest.raises(ValueError, match="No boundary condition"):
        grid.cumsum(c, "Z", to="left")
    with pytest.raises(ValueError, match="No boundary condition"):
        grid.cumsum(_on_device(c), "Z", to="left")
    u = ds["u"]
    spy.clear()
    got = grid.cumsum(u, "X", to="center")  # left -> center: no halo
    assert spy == ["cumscan_host"]
    _same(got, grid.cumsum(_on_device(u), "X", to="center"), S.cumscan(u.values, 4), "left -> center")


def test_faces_parity_of_errors_and_whole_field_layouts(spy):
    ds, grid = _faces_grid(np.float64)
    c = ds["c"]
    # a trimmed array across a seam that swaps axes: the error of pad(), raised before anything streams
    for arg in (c, _on_device(c)):
        with pytest.raises(ValueError, match="equal size"):
            grid.cumsum(arg, "X", to="left", padding="fill")
    ds2, strip = _faces_grid(np.float64, fc=STRIP)
    with pytest.raises(ValueError, match="No boundary condition"):
        strip.cumsum(ds2["c"], "X", to="outer")
    # no batch dim in front of the face dim, and cumint + metric_weighted: the whole-field route, same values
    t = c.transpose("face", "time", "k", "y", "x")
    t = xg.DataArray(np.ascontiguousarray(t.values), dims=t.dims)
    spy.clear()
    got = grid.cumsum(t, "Y", to="outer", padding="extend")
    assert spy == []
    np.testing.assert_array_equal(_host(got), _host(grid.cumsum(_on_device(t), "Y", to="outer", padding="extend")))
    got = grid.cumint(c, "X", to="outer", metric_weighted="X")
    assert spy == []
    np.testing.assert_array_equal(_host(got), _host(grid.cumint(_on_device(c), "X", to="outer", metric_weighted="X")))


def test_faces_streaming_is_bounded_by_the_slab():
    ds, grid = _faces_grid(np.float32, lead=(1, 30), lead_dims=("one", "k"))  # (1, k, face, j, i)
    c = ds["c"]
    _capi.check(_capi.load().xg_host_workspace_release())
    grid.cumsum(c, "Y", to="outer", reverse=True)  # warm-up: workspace and plan
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    got = grid.cumsum(c, "Y", to="outer", reverse=True)
    assert torch.cuda.max_memory_allocated() - base < c.values.nbytes // 4
    rows = 8  # 30 rows of 6 x 48 x 48 fp32 (55 KiB): min(18, ceil(30 / 4)) = 8 rows per slab
    row_in, row_out, plane = 6 * N * N * 4, 6 * (N + 1) * N * 4, 6 * N * 4
    assert _workspace_bytes() <= rows * (3 * (row_in + row_out) + row_in + 2 * plane) + 8  # + scratch, fill
    want = _cumsum_oracle(c.values, 3, True, "none", None, None, _faces_pad(CUBED_SPHERE, c.dims, "Y", 0, 1, None, 0))
    np.testing.assert_array_equal(_host(got), want)


# ------------------------------------------------------------------ north fold
NX, NY = 40, 33
POS = ("center", "left", "right", "outer")
EXTRA = {"center": 0, "left": 0, "right": 0, "outer": 1}
XD = {p: "x" + p for p in POS}
YD = {p: "y" + p for p in POS}
PIVOTS = ["T", "F", "U", "V"]
FLEAD = (5, 6)  # (time, z): 30 rows of ~5 KiB -> ceil(30 / 8) = 4 slabs, the last ragged


def _fold_grid(south, pivot, dtype, seed=0):
    rng = np.random.default_rng(seed)
    coords = {XD[p]: np.arange(NX + EXTRA[p]) for p in POS}
    coords.update({YD[p]: np.arange(NY + EXTRA[p]) for p in POS})
    data = {f"dy_{p}": ((YD[p], "xcenter"), 0.5 + rng.random((NY + EXTRA[p], NX)).astype(dtype)) for p in POS}
    ds = xg.Dataset(data_vars=data, coords=coords)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        grid = xg.Grid(ds, coords={"X": dict(XD), "Y": dict(YD)},
                       padding={"X": "periodic", "Y": {"fold": pivot, "south": south}}, autoparse_metadata=False)
    grid.set_metrics("Y", [f"dy_{p}" for p in POS])
    return ds, grid


def _fold_field(src, dtype, seed=1, lead=FLEAD, nan=True):
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(lead + (NY + EXTRA[src], NX)).astype(dtype)
    if nan:
        a[rng.random(a.shape) < 0.05] = np.nan
    return xg.DataArray(a, dims=("time", "z")[:len(lead)] + (YD[src], "xcenter"))


def _fold_pad(src, pivot, lo, hi, south):
    def pad(s):
        fa = s.ndim - 2
        return F.pad_fold(s, fa, fa + 1, src, "center", F.resolve_pivot(pivot, "Y", "X"), {fa: (lo, hi)},
                          {fa: south})
    return pad


# (src, to, reverse): reverse scans that pad the north edge fold; forward ones pad the south edge alone
FOLD_CASES = [("center", "right", True), ("center", "outer", True), ("left", "center", True),
              ("center", "left", False), ("center", "outer", False)]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_fold_every_pivot_and_shift(dtype, spy):
    checked = 0
    for pivot, south in itertools.product(PIVOTS, ("fill", "periodic")):
        ds, grid = _fold_grid(south, pivot, dtype)
        for src, to, reverse in FOLD_CASES:
            da = _fold_field(src, dtype)
            trim, (lo, hi) = _table(src, to, reverse)
            spy.clear()
            got = grid.cumsum(da, "Y", to=to, reverse=reverse)
            assert spy == ["cumscan_host_fold" if hi else "cumscan_host"], (pivot, src, to, reverse)
            dev = grid.cumsum(_on_device(da), "Y", to=to, reverse=reverse)
            want = _cumsum_oracle(da.values, 2, reverse, trim, None, None, _fold_pad(src, pivot, lo, hi, south))
            _same(got, dev, want, f"{pivot} {south} {src} -> {to} reverse={reverse}")
            checked += 1
    assert checked == len(PIVOTS) * 2 * len(FOLD_CASES)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_fold_cumint_and_metric_weighted(dtype, spy):
    ds, grid = _fold_grid("fill", "F", dtype)
    da = _fold_field("center", dtype)
    pad = _fold_pad("center", "F", 0, 1, "fill")
    spy.clear()
    got = grid.cumint(da, "Y", to="right", reverse=True)
    assert spy == ["cumscan_host_fold"]
    _same(got, grid.cumint(_on_device(da), "Y", to="right", reverse=True),
          _cumsum_oracle(da.values, 2, True, "drop_first", ds["dy_center"].values, None, pad), "cumint")
    got = grid.cumsum(da, "Y", to="right", reverse=True, metric_weighted="Y")
    _same(got, grid.cumsum(_on_device(da), "Y", to="right", reverse=True, metric_weighted="Y"),
          _cumsum_oracle(da.values, 2, True, "drop_first", ds["dy_center"].values, ds["dy_right"].values, pad),
          "metric_weighted")
    # cumint + metric_weighted and a 2-D field keep the whole-field route and its values
    spy.clear()
    got = grid.cumint(da, "Y", to="right", reverse=True, metric_weighted="Y")
    assert spy == []
    np.testing.assert_array_equal(
        _host(got), _host(grid.cumint(_on_device(da), "Y", to="right", reverse=True, metric_weighted="Y")))
    flat = _fold_field("center", dtype, lead=())
    got = grid.cumsum(flat, "Y", to="outer", reverse=True)
    assert spy == []
    _same(got, grid.cumsum(_on_device(flat), "Y", to="outer", reverse=True),
          _cumsum_oracle(flat.values, 0, True, "none", None, None, _fold_pad("center", "F", 0, 1, "fill")), "2-D")


def test_fold_streaming_is_bounded_by_the_slab():
    ds, grid = _fold_grid("periodic", "F", np.float32)
    da = _fold_field("center", np.float32, lead=(12, 20), nan=False)
    _capi.check(_capi.load().xg_host_workspace_release())
    grid.cumsum(da, "Y", to="right", reverse=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    got = grid.cumsum(da, "Y", to="right", reverse=True)
    assert torch.cuda.max_memory_allocated() - base < da.values.nbytes // 4
    rows = min((1 << 20) // (NY * NX * 4), -(-240 // 4))
    assert -(-240 // rows) >= 4
    row = NY * NX * 4
    assert _workspace_bytes() <= rows * (3 * 2 * row + row + 2 * NX * 4)  # slots, scratch, planes
    want = _cumsum_oracle(da.values, 2, True, "drop_first", None, None, _fold_pad("center", "F", 0, 1, "periodic"))
    np.testing.assert_array_equal(_host(got), want)


def test_host_group_matches_one_device():
    ds, grid = _faces_grid(np.float32, nan=True)
    group = xg.Grid(ds, coords=COORDS, face_connections=CUBED_SPHERE, host_devices=[0, 0])
    c = ds["c"]
    for ax, reverse in (("X", True), ("Y", False)):
        np.testing.assert_array_equal(_host(group.cumsum(c, ax, to="outer", reverse=reverse)),
                                      _host(grid.cumsum(c, ax, to="outer", reverse=reverse)))
    fds, fgrid = _fold_grid("fill", "T", np.float64)
    da = _fold_field("center", np.float64)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        fgroup = xg.Grid(fds, coords={"X": dict(XD), "Y": dict(YD)}, host_devices=[0, 0], autoparse_metadata=False,
                         padding={"X": "periodic", "Y": {"fold": "T", "south": "fill"}})
    np.testing.assert_array_equal(_host(fgroup.cumsum(da, "Y", to="outer", reverse=True)),
                                  _host(fgrid.cumsum(da, "Y", to="outer", reverse=True)))
