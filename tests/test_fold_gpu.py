"""North-fold (tripolar) boundary on the H100: pad() and every operator across the fold, bit for bit against
oracle/fold.py composed with oracle/stencil.py, in fp32 and fp64.  An operator across the fold costs one
xg_fold_rows launch beside its xg_stencil2 launch."""

import itertools
import warnings

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from oracle import fold as F
from oracle import stencil as S

pytestmark = pytest.mark.gpu

NX, NY = 12, 7
POS = ("center", "left", "right", "outer", "inner")
EXTRA = {"center": 0, "left": 0, "right": 0, "outer": 1, "inner": -1}
PIVOTS = ["center", "T", "corner", "F", "U", "V", {"X": "right", "Y": "center"}]
XD = {p: "x" + p for p in POS}
YD = {p: "y" + p for p in POS}


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _host(da):
    return da.data.cpu().numpy() if isinstance(da.data, torch.Tensor) else np.asarray(da.data)


def _launches():
    from xgcm_b200 import _capi

    return _capi.load().xg_launch_count()


def _coords():
    c = {XD[p]: np.arange(NX + EXTRA[p]) for p in POS}
    c.update({YD[p]: np.arange(NY + EXTRA[p]) for p in POS})
    return c


def _grid(ds, y_padding, x_padding="periodic"):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        return xg.Grid(ds, coords={"X": dict(XD), "Y": dict(YD)}, padding={"X": x_padding, "Y": y_padding},
                       autoparse_metadata=False)


def _roles(pivot):
    return F.resolve_pivot(pivot, "Y", "X")


def _field(rng, ypos, xpos, dtype, lead=()):
    return rng.standard_normal(lead + (NY + EXTRA[ypos], NX + EXTRA[xpos])).astype(dtype)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("lead", [(), (2, 3)], ids=["2d", "4d"])
def test_pad_every_pivot_and_position(dtype, lead):
    rng = np.random.default_rng(len(lead))
    ds = xg.Dataset(coords=_coords())
    nd = len(lead) + 2
    fa, sa = nd - 2, nd - 1
    dims_lead = ("time", "z")[:len(lead)]
    checked = 0
    for pivot, south in itertools.product(PIVOTS, ("periodic", "fill", "extend")):
        grid = _grid(ds, {"fold": pivot, "south": south})
        roles = _roles(pivot)
        for xpos, ypos, vector in itertools.product(POS, POS, (False, True)):
            if xpos == "inner" and roles["seam"] == "center":
                continue
            a = _field(rng, ypos, xpos, dtype, lead)
            da = xg.DataArray(_dev(a), dims=dims_lead + (YD[ypos], XD[xpos]))
            skip = 1 if F.kind(ypos) == roles["fold"] else 0
            n = a.shape[fa]
            widths = [(0, 1), (1, 1), (0, n - skip)]
            for lo, hi in widths:
                arg = {"Y": da} if vector else da
                got = _host(xg.pad(arg, grid, padding_width={"Y": (lo, hi)}))
                want = F.pad_fold(a, fa, sa, ypos, xpos, roles, {fa: (lo, hi)}, {fa: south}, vector=vector)
                assert got.dtype == a.dtype
                np.testing.assert_array_equal(got, want, err_msg=f"{pivot} {south} {ypos} {xpos} {vector} {lo, hi}")
                checked += 1
    assert checked > 1000


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_pad_fold_with_seam_padding(dtype):
    rng = np.random.default_rng(3)
    ds = xg.Dataset(coords=_coords())
    grid = _grid(ds, {"fold": "corner", "south": "periodic"})
    a = _field(rng, "left", "center", dtype, (3,))
    da = xg.DataArray(_dev(a), dims=("z", "yleft", "xcenter"))
    got = _host(xg.pad(da, grid, padding_width={"X": (1, 1), "Y": (1, 2)}))
    want = F.pad_fold(a, 1, 2, "left", "center", _roles("corner"), {1: (1, 2), 2: (1, 1)},
                      {1: "periodic", 2: "periodic"})
    np.testing.assert_array_equal(got, want)


def _metric_ds(rng, dtype, lead=()):
    data = {}
    for ypos in POS:
        data[f"dy_{ypos}"] = ((YD[ypos], "xcenter"), 0.5 + rng.random((NY + EXTRA[ypos], NX)).astype(dtype))
        data[f"area_{ypos}"] = ((YD[ypos], "xcenter"), 0.5 + rng.random((NY + EXTRA[ypos], NX)).astype(dtype))
    return xg.Dataset(data_vars=data, coords=_coords())


def _with_metrics(grid):
    grid.set_metrics("Y", [f"dy_{p}" for p in POS])
    grid.set_metrics(("X", "Y"), [f"area_{p}" for p in POS])
    return grid


def _expect(op, a, ypos, pivot, lo, hi, south, fa, vector=False, pre=None, post=None):
    x = a if pre is None else a * pre
    padded = F.pad_fold(x, fa, fa + 1, ypos, "center", _roles(pivot), {fa: (lo, hi)}, {fa: south}, vector=vector)
    r = S.stencil2(op, padded, fa, 0, 0, None)
    return r if post is None else r / post


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("pivot", ["corner", "U"])
def test_operators_every_y_shift(dtype, pivot):
    rng = np.random.default_rng(7)
    ds = _metric_ds(rng, dtype)
    grid = _with_metrics(_grid(ds, {"fold": pivot, "south": "periodic"}))
    plain = _with_metrics(_grid(ds, "periodic"))
    lead = (3, 2)
    for (src, dst), (lo, hi) in S.PADDING_WIDTH.items():
        a = _field(rng, src, "center", dtype, lead)
        da = xg.DataArray(_dev(a), dims=("time", "z", YD[src], "xcenter"))
        for op, vector in itertools.product(("diff", "interp", "min", "max"), (False, True)):
            arg = {"Y": da} if vector else da
            getattr(plain, op)(arg, "Y", to=dst)
            n0 = _launches()
            getattr(plain, op)(arg, "Y", to=dst)
            n_plain = _launches() - n0
            n0 = _launches()
            got = getattr(grid, op)(arg, "Y", to=dst)
            n_fold = _launches() - n0
            assert n_fold == n_plain + (1 if hi else 0), (src, dst, op)
            np.testing.assert_array_equal(_host(got), _expect(op, a, src, pivot, lo, hi, "periodic", 2, vector),
                                          err_msg=f"{op} {src}->{dst} {vector}")
        if not hi:
            continue
        from xgcm_b200 import _capi

        dy, area_in, area_out = (ds[f"dy_{dst}"].values, ds[f"area_{src}"].values, ds[f"area_{dst}"].values)
        got = grid.derivative(da, "Y", to=dst)
        assert _capi.last_launch() in ("xg_stencil2(plane)", "xg_stencil2(tile_tma)"), _capi.last_launch()
        np.testing.assert_array_equal(_host(got), _expect("diff", a, src, pivot, lo, hi, "periodic", 2, post=dy))
        grid.interp(da, "Y", to=dst, metric_weighted=["X", "Y"])
        n0 = _launches()
        got = grid.interp(da, "Y", to=dst, metric_weighted=["X", "Y"])
        assert _launches() - n0 == 2
        assert _capi.last_launch() in ("xg_stencil2(plane)", "xg_stencil2(tile_tma)"), _capi.last_launch()
        np.testing.assert_array_equal(
            _host(got), _expect("interp", a, src, pivot, lo, hi, "periodic", 2, pre=area_in, post=area_out))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_multi_axis_pair_cumsum_numpy_and_vector(dtype):
    rng = np.random.default_rng(11)
    ds = _metric_ds(rng, dtype)
    grid = _grid(ds, {"fold": "corner"})
    roles = _roles("corner")
    q = _field(rng, "left", "left", dtype, (4,))
    dq = xg.DataArray(_dev(q), dims=("z", "yleft", "xleft"))
    # multi-axis interp: X (periodic) then Y across the fold; per-call extend still folds the north edge
    for kw, mode in (({}, None), ({"padding": "extend"}, "extend")):
        step = S.stencil2("interp", q, 2, 0, 1, mode or "periodic")
        want = F.pad_fold(step, 1, 2, "left", "center", roles, {1: (0, 1)}, {1: mode or "fill"})
        got = grid.interp(dq, ["X", "Y"], **kw)
        np.testing.assert_array_equal(_host(got), S.stencil2("interp", want, 1, 0, 0, None))
    # numpy input and the vector dict
    got = grid.diff(xg.DataArray(q, dims=("z", "yleft", "xleft")), "Y")
    assert isinstance(got.data, np.ndarray)
    want = F.pad_fold(q, 1, 2, "left", "left", roles, {1: (0, 1)}, {1: "fill"})
    np.testing.assert_array_equal(got.data, S.stencil2("diff", want, 1, 0, 0, None))
    got = grid.diff({"Y": dq}, "Y")
    want = F.pad_fold(q, 1, 2, "left", "left", roles, {1: (0, 1)}, {1: "fill"}, vector=True)
    np.testing.assert_array_equal(_host(got), S.stencil2("diff", want, 1, 0, 0, None))
    # divergence: (diff_X(u dy) + diff_Y(v dx)) / area, v folded as a vector component
    u = _field(rng, "center", "left", dtype)
    v = _field(rng, "left", "center", dtype)
    dyu = (0.5 + rng.random(u.shape)).astype(dtype)
    dxv = (0.5 + rng.random(v.shape)).astype(dtype)
    area = (0.5 + rng.random((NY, NX))).astype(dtype)
    mds = xg.Dataset(data_vars={"dyu": (("ycenter", "xleft"), dyu), "dxv": (("yleft", "xcenter"), dxv),
                                "area": (("ycenter", "xcenter"), area)}, coords=_coords())
    mgrid = _grid(mds, {"fold": "corner"})
    mgrid.set_metrics("Y", "dyu")
    mgrid.set_metrics("X", "dxv")
    mgrid.set_metrics(("X", "Y"), "area")
    du = xg.DataArray(_dev(u), dims=("ycenter", "xleft"))
    dv = xg.DataArray(_dev(v), dims=("yleft", "xcenter"))
    tx = S.stencil2("diff", u * dyu, 1, 0, 1, "periodic")
    vd = v * dxv
    ty = S.stencil2("diff", F.pad_fold(vd, 0, 1, "left", "center", roles, {0: (0, 1)}, {0: "fill"}, vector=True),
                    0, 0, 0, None)
    np.testing.assert_array_equal(_host(mgrid.divergence(du, dv)), (tx + ty) / area)
    # vorticity with u at (yleft, xleft) and v at (ycenter, xcenter): the Y term of u crosses the fold
    uq = _field(rng, "left", "left", dtype)
    vc = _field(rng, "center", "center", dtype)
    dxq = (0.5 + rng.random(uq.shape)).astype(dtype)
    dyc = (0.5 + rng.random(vc.shape)).astype(dtype)
    aq = (0.5 + rng.random((NY, NX))).astype(dtype)
    vds = xg.Dataset(data_vars={"dxq": (("yleft", "xleft"), dxq), "dyc": (("ycenter", "xcenter"), dyc),
                                "aq": (("ycenter", "xleft"), aq)}, coords=_coords())
    vgrid = _grid(vds, {"fold": "corner"})
    vgrid.set_metrics("X", "dxq")
    vgrid.set_metrics("Y", "dyc")
    vgrid.set_metrics(("X", "Y"), "aq")
    ta = S.stencil2("diff", vc * dyc, 1, 1, 0, "periodic")
    tb = S.stencil2("diff", F.pad_fold(uq * dxq, 0, 1, "left", "left", roles, {0: (0, 1)}, {0: "fill"}, vector=True),
                    0, 0, 0, None)
    got = vgrid.vorticity(xg.DataArray(_dev(uq), dims=("yleft", "xleft")),
                          xg.DataArray(_dev(vc), dims=("ycenter", "xcenter")))
    np.testing.assert_array_equal(_host(got), (ta - tb) / aq)
    # cumsum c -> outer: forward pads the south edge (the spec's south mode), reversed folds the north edge
    c = _field(rng, "center", "center", dtype, (2,))
    dc = xg.DataArray(_dev(c), dims=("z", "ycenter", "xcenter"))
    fwd = np.cumsum(c, axis=1, dtype=dtype)
    np.testing.assert_array_equal(_host(grid.cumsum(dc, "Y", to="outer")), S.pad_axis(fwd, 1, 1, 0, "fill"))
    rev = np.flip(np.cumsum(np.flip(c, 1), axis=1, dtype=dtype), 1)
    want = F.pad_fold(rev, 1, 2, "center", "center", roles, {1: (0, 1)}, {1: "fill"})
    np.testing.assert_array_equal(_host(grid.cumsum(dc, "Y", to="outer", reverse=True)), want)


@pytest.mark.parametrize("op", ["diff", "interp"])
def test_c3_sized_left_field_only_the_top_row_changes(op):
    """A (75, 2400, 3600) fp32 field at `left` under a corner pivot (skip = 1): the top output row is the
    oracle's fold row, every other row is bitwise the plain fill grid's."""
    nz, ny, nx = 75, 2400, 3600
    ds = xg.Dataset(coords={"xc": np.arange(nx), "yl": np.arange(ny), "yc": np.arange(ny)})
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        grid = xg.Grid(ds, coords={"X": {"center": "xc"}, "Y": {"center": "yc", "left": "yl"}},
                       padding={"X": "periodic", "Y": {"fold": "corner"}}, autoparse_metadata=False)
    plain = xg.Grid(ds, coords={"X": {"center": "xc"}, "Y": {"center": "yc", "left": "yl"}},
                    padding={"X": "periodic", "Y": "fill"}, autoparse_metadata=False)
    from xgcm_b200 import ops

    x = torch.empty((nz, ny, nx), dtype=torch.float32, device="cuda:0")
    ops.fill_uniform(x, 2026)
    da = xg.DataArray(x, dims=("z", "yl", "xc"))
    got = getattr(grid, op)(da, "Y").data
    ref = getattr(plain, op)(da, "Y").data
    assert torch.equal(got[:, :-1], ref[:, :-1])
    top = x[:, -2:].cpu().numpy()  # the last interior row and, folded, the row below it (skip = 1)
    halo = F.north_rows(x[:, -3:].cpu().numpy(), 1, 2, "left", "center", _roles("corner"), 1)
    want = S.stencil2(op, np.concatenate([top[:, 1:], halo], axis=1), 1, 0, 0, None)
    np.testing.assert_array_equal(got[:, -1:].cpu().numpy(), want)
