"""Grid.divergence / vorticity / pair across the north fold on the H100: one xg_fold_rows launch of the strided
term's folded row, then one xg_stencil_pair launch that takes it as its halo plane.  Every case is bit for bit
equal to oracle/fold.py + oracle/stencil.py and to the explicit chain a user writes from Grid.diff calls and array
arithmetic, in fp32 and fp64; numpy fields stream through xg_stencil_pair_host[_fold] and equal the device call."""

import itertools
import warnings

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from oracle import fold as F
from oracle import stencil as S
from xgcm_b200 import _capi, ops

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
POS = ("center", "left", "right")
XD = {p: "x" + p for p in POS}
YD = {p: "y" + p for p in POS}
PIVOTS = ["center", "T", "corner", "F", "U", "V"]
# (u position, v position, to): divergence diff_X(u dy) + diff_Y(v dx), output where both terms land
DIV_LAYOUTS = [(("center", "left"), ("left", "center"), "center"),   # Y term left -> center: north edge folds
               (("right", "center"), ("center", "right"), "right"),  # center -> right: north edge folds
               (("left", "center"), ("center", "left"), "left"),     # center -> left: south edge only
               (("center", "right"), ("right", "center"), "center")]  # right -> center: south edge only


def _launches():
    return _capi.load().xg_launch_count()


def _host(x):
    d = x.data if hasattr(x, "data") else x
    return d.cpu().numpy() if isinstance(d, torch.Tensor) else np.asarray(d)


def _dev(a, offset=0):
    """``a`` on the GPU, ``offset`` elements past the start of its allocation (a misaligned view for offset 1-3)."""
    a = np.ascontiguousarray(a)
    base = torch.empty(a.size + offset, dtype=torch.float32 if a.dtype == np.float32 else torch.float64, device=DEV)
    t = base[offset:offset + a.size].view(a.shape)
    t.copy_(torch.from_numpy(a))
    return t


def _fields(rng, shape, dtype, specials):
    a = rng.standard_normal(shape).astype(dtype)
    if specials:
        flat = a.reshape(-1)
        idx = rng.choice(flat.size, size=min(flat.size, 24), replace=False)
        flat[idx] = np.resize(np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, np.nan], dtype=dtype), idx.size)
        flat[-1] = np.nan  # the top row, the one the fold mirrors
    return a


def _grid(pivot, south, ny, nx, dtype, metrics="2d", nz=None, seed=0):
    """X periodic, Y folding under ``pivot`` (or plain ``south`` when pivot is None); dx / dy / area at every
    (Y, X) position, shared between levels ("2d") or per level (hFac-like, "3d": dims (z, y, x))."""
    rng = np.random.default_rng(seed)
    coords = {XD[p]: np.arange(nx) for p in POS}
    coords.update({YD[p]: np.arange(ny) for p in POS})
    data, reg = {}, {("X",): [], ("Y",): [], ("X", "Y"): []}
    if metrics:
        lead_dims, lead = (("z",), (nz,)) if metrics == "3d" else ((), ())
        for yp, xp in itertools.product(POS, POS):
            for name, key in (("dx", ("X",)), ("dy", ("Y",)), ("area", ("X", "Y"))):
                data[f"{name}_{yp}_{xp}"] = (lead_dims + (YD[yp], XD[xp]),
                                             (0.5 + rng.random(lead + (ny, nx))).astype(dtype))
                reg[key].append(f"{name}_{yp}_{xp}")
        if metrics == "3d":
            coords["z"] = np.arange(nz)
    ds = xg.Dataset(data_vars=data, coords=coords)
    padding = {"X": "periodic", "Y": {"fold": pivot, "south": south} if pivot else south}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        grid = xg.Grid(ds, coords={"X": dict(XD), "Y": dict(YD)}, padding=padding, autoparse_metadata=False,
                       metrics={k: v for k, v in reg.items() if v})
    return ds, grid


def _metric(ds, name, yp, xp, nd):
    m = ds[f"{name}_{yp}_{xp}"].values
    return m.reshape((1,) * (nd - m.ndim) + m.shape)


def _want(op_a, a, xa, to_x, op_b, b, yb, xb, to_y, pivot, south, xpad, sub, pre_a=None, pre_b=None, post=None,
          vector=False):
    """oracle: term a along x, term b along y padded by pad_fold (north fold + south mode), then +-, then /."""
    lo_a, hi_a = S.PADDING_WIDTH[(xa, to_x)]
    lo_b, hi_b = S.PADDING_WIDTH[(yb, to_y)]
    nd = a.ndim
    with np.errstate(all="ignore"):
        ta = S.stencil2(op_a, a if pre_a is None else a * pre_a, nd - 1, lo_a, hi_a, xpad)
        wb = b if pre_b is None else b * pre_b
        padded = F.pad_fold(wb, nd - 2, nd - 1, yb, xb, F.resolve_pivot(pivot, "Y", "X"), {nd - 2: (lo_b, hi_b)},
                            {nd - 2: south}, vector=vector)
        tb = S.stencil2(op_b, padded, nd - 2, 0, 0, None)
        r = ta + tb if sub == "add" else ta - tb
        return (r if post is None else r / post).astype(a.dtype)


def _chain(grid, op_a, da_a, op_b, da_b, to, combine, metric_a=None, metric_b=None, divide_by=None, vector=False,
           **kw):
    """The explicit user chain: Grid.diff-like calls on the metric-weighted fields, then array arithmetic."""
    xa = da_a * grid.get_metric(da_a, metric_a) if metric_a else da_a
    xb = da_b * grid.get_metric(da_b, metric_b) if metric_b else da_b
    ta = getattr(grid, op_a)(xa, "X", to=to["X"], **kw)
    tb = getattr(grid, op_b)({"Y": xb} if vector else xb, "Y", to=to["Y"], **kw)
    r = ta + tb if combine == "add" else ta - tb
    return r / grid.get_metric(r, divide_by) if divide_by else r


def _counted(fn, *args, **kw):
    """``fn(*args, **kw)``, the number of kernels it launched and the label of its last one."""
    n0 = _launches()
    r = fn(*args, **kw)
    return r, _launches() - n0, _capi.last_launch()


def _check(got, want, chain, ran, n_fold, label, msg):
    assert ran == (1 + n_fold, label), (msg, ran)
    got = _host(got)
    assert got.dtype == want.dtype, msg
    np.testing.assert_array_equal(got, want, err_msg=f"{msg}: oracle")
    np.testing.assert_array_equal(got, _host(chain), err_msg=f"{msg}: chain")


def _run_div_vort(dtype, lead, lead_dims, ny, nx, metrics, offset, label, specials, pivots, souths, seed):
    rng = np.random.default_rng(seed)
    checked = 0
    nd = len(lead) + 2
    for pivot, south in itertools.product(pivots, souths):
        ds, grid = _grid(pivot, south, ny, nx, dtype, metrics, nz=lead[-1] if lead else None, seed=seed)
        for (upos, vpos, to), kw in itertools.product(DIV_LAYOUTS, ({}, {"padding": "extend"}, {"padding": "fill"})):
            s_eff = kw.get("padding", south)
            x_eff = kw.get("padding", "periodic")
            u = _fields(rng, lead + (ny, nx), dtype, specials)
            v = _fields(rng, lead + (ny, nx), dtype, specials)
            du = xg.DataArray(_dev(u, offset), dims=lead_dims + (YD[upos[0]], XD[upos[1]]))
            dv = xg.DataArray(_dev(v, offset), dims=lead_dims + (YD[vpos[0]], XD[vpos[1]]))
            tos = {"X": to, "Y": to}
            n_fold = 1 if S.PADDING_WIDTH[(vpos[0], to)][1] else 0
            # divergence: (diff_X(u dy) + diff_Y(v dx)) / area, v folded as a vector component
            grid.divergence(du, dv, to=tos, **kw)  # metric upload
            got, *n = _counted(grid.divergence, du, dv, to=tos, **kw)
            want = _want("diff", u, upos[1], to, "diff", v, vpos[0], vpos[1], to, pivot, s_eff, x_eff, "add",
                         _metric(ds, "dy", *upos, nd), _metric(ds, "dx", *vpos, nd), _metric(ds, "area", to, to, nd),
                         vector=True)
            chain = _chain(grid, "diff", du, "diff", dv, tos, "add", ("Y",), ("X",), ("X", "Y"), vector=True, **kw)
            _check(got, want, chain, tuple(n), n_fold, label, f"div {pivot} {south} {kw} {upos} {vpos}")
            # vorticity: (diff_X(v dy) - diff_Y(u dx)) / area with the roles of the two layouts swapped
            vv = xg.DataArray(du.data, dims=du.dims)  # on the u layout: the x term
            uu = xg.DataArray(dv.data, dims=dv.dims)  # on the v layout: the term across the fold
            grid.vorticity(uu, vv, to=tos, **kw)
            got, *n = _counted(grid.vorticity, uu, vv, to=tos, **kw)
            want = _want("diff", u, upos[1], to, "diff", v, vpos[0], vpos[1], to, pivot, s_eff, x_eff, "sub",
                         _metric(ds, "dy", *upos, nd), _metric(ds, "dx", *vpos, nd), _metric(ds, "area", to, to, nd),
                         vector=True)
            chain = _chain(grid, "diff", vv, "diff", uu, tos, "sub", ("Y",), ("X",), ("X", "Y"), vector=True, **kw)
            _check(got, want, chain, tuple(n), n_fold, label, f"vort {pivot} {south} {kw} {upos} {vpos}")
            checked += 2
    return checked


SHAPES = {  # name: (lead, lead dims, ny, nx, metrics, view offset, kernel label)
    "yx short rows": ((), (), 7, 40, "2d", 0, "xg_stencil_pair"),
    "zyx ragged rows hFac": ((4,), ("z",), 7, 37, "3d", 0, "xg_stencil_pair"),
    "tzyx": ((2, 3), ("time", "z"), 7, 40, "2d", 0, "xg_stencil_pair"),
    "tzyx hFac": ((2, 3), ("time", "z"), 6, 40, "3d", 0, "xg_stencil_pair"),
    "zyx aligned TMA rows": ((4,), ("z",), 9, 512, "2d", 0, "xg_stencil_pair(tile_tma)"),
    "zyx aligned TMA rows hFac": ((3,), ("z",), 9, 512, "3d", 0, "xg_stencil_pair(tile_tma)"),
}


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", list(SHAPES))
def test_divergence_vorticity_across_the_fold(dtype, name):
    lead, lead_dims, ny, nx, metrics, offset, label = SHAPES[name]
    checked = _run_div_vort(dtype, lead, lead_dims, ny, nx, metrics, offset, label, True, PIVOTS,
                            ("periodic", "fill", "extend"), seed=len(name))
    assert checked == 2 * len(PIVOTS) * 3 * len(DIV_LAYOUTS) * 3


@pytest.mark.parametrize("offset", [1, 2, 3])
def test_misaligned_views_fp32(offset):
    """(Z, Y, X) views 1-3 elements past a 16-byte boundary: the register-staged kernel, one element per lane, on
    rows that would otherwise take the TMA-staged one."""
    _run_div_vort(np.float32, (3,), ("z",), 7, 512, "2d", offset, "xg_stencil_pair", True, ["corner", "V"],
                  ("periodic", "fill"), seed=offset)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("lead", [(), (3,)], ids=["yx", "zyx"])
def test_generic_pair_terms_across_the_fold(dtype, lead):
    """Grid.pair with every diff / interp / min / max combination, add and sub, scalar and vector fields, NaN and
    +-inf among the inputs, no metrics."""
    rng = np.random.default_rng(20 + len(lead))
    ny, nx = 8, 44
    lead_dims = ("z",) * len(lead)
    checked = 0
    for pivot, south in (("T", "periodic"), ("F", "fill"), ("U", "extend"), ("V", "periodic")):
        _, grid = _grid(pivot, south, ny, nx, dtype, metrics=None)
        for op_a, op_b, combine, vector in itertools.product(("diff", "interp", "min", "max"),
                                                             ("diff", "interp", "min", "max"), ("add", "sub"),
                                                             (False, True)):
            a = _fields(rng, lead + (ny, nx), dtype, True)
            b = _fields(rng, lead + (ny, nx), dtype, True)
            da = xg.DataArray(_dev(a), dims=lead_dims + ("ycenter", "xleft"))
            db = xg.DataArray(_dev(b), dims=lead_dims + ("yleft", "xcenter"))
            to = {"X": "center", "Y": "center"}
            comp = ("X", "Y") if vector else None
            grid.pair(op_a, da, "X", op_b, db, "Y", combine=combine, to=to, _components=comp)
            got, *n = _counted(grid.pair, op_a, da, "X", op_b, db, "Y", combine=combine, to=to, _components=comp)
            want = _want(op_a, a, "left", "center", op_b, b, "left", "center", "center", pivot, south, "periodic",
                         combine, vector=vector)
            chain = _chain(grid, op_a, da, op_b, db, to, combine, vector=vector)
            _check(got, want, chain, tuple(n), 1, "xg_stencil_pair", f"{pivot} {op_a} {op_b} {combine} {vector}")
            checked += 1
    assert checked == 4 * 64


def test_tma_many_tiles_per_cta_with_a_halo_plane():
    """The C3-sized divergence under a corner pivot: the persistent TMA-staged pair kernel walks at least 8 tiles
    per CTA at 4 x 132 CTAs while reading the fold plane for its top row; every cell against the oracle."""
    from test_tma_schedule_gpu import MAX_CTAS, MIN_TILES_PER_CTA, SMS, schedule

    nz, ny, nx = 45, 265, 1124
    assert schedule(np.float32, nx, ny, nz)["ntiles"] >= MIN_TILES_PER_CTA * MAX_CTAS * SMS
    rng = np.random.default_rng(30)
    ds, grid = _grid("corner", "fill", ny, nx, np.float32)
    u = _fields(rng, (nz, ny, nx), np.float32, True)
    v = _fields(rng, (nz, ny, nx), np.float32, True)
    du = xg.DataArray(_dev(u), dims=("z", "ycenter", "xleft"))
    dv = xg.DataArray(_dev(v), dims=("z", "yleft", "xcenter"))
    to = {"X": "center", "Y": "center"}
    grid.divergence(du, dv, to=to)
    got, *n = _counted(grid.divergence, du, dv, to=to)
    want = _want("diff", u, "left", "center", "diff", v, "left", "center", "center", "corner", "fill", "periodic",
                 "add", _metric(ds, "dy", "center", "left", 3), _metric(ds, "dx", "left", "center", 3),
                 _metric(ds, "area", "center", "center", 3), vector=True)
    chain = _chain(grid, "diff", du, "diff", dv, to, "add", ("Y",), ("X",), ("X", "Y"), vector=True)
    _check(got, want, chain, tuple(n), 1, "xg_stencil_pair(tile_tma)", "C3-sized divergence")


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("nx, halo_offset, label", [(512, 0, "xg_stencil_pair(tile_tma)"), (40, 0, "xg_stencil_pair"),
                                                    (512, 1, "xg_stencil_pair")])
def test_ops_halo_planes_replace_the_boundary_on_their_side(dtype, nx, halo_offset, label):
    """ops.stencil_pair with distinct lo / hi planes (already weighted: taken as they are) on both kernels, a
    misaligned plane included: each plane pads exactly its own side of the term along axis_b."""
    rng = np.random.default_rng(40)
    nz, ny = 4, 9
    a, b = _fields(rng, (nz, ny, nx), dtype, True), _fields(rng, (nz, ny, nx), dtype, True)
    pre_b = (0.5 + rng.random((1, ny, nx))).astype(dtype)
    post = (0.5 + rng.random((1, ny, nx))).astype(dtype)
    planes = [rng.standard_normal((nz, 1, nx)).astype(dtype) for _ in range(2)]
    ta, tb, tpre, tpost = _dev(a), _dev(b), _dev(pre_b), _dev(post)
    tl, th = (_dev(p, halo_offset) for p in planes)
    for lo_b, bc_b in itertools.product((0, 1), ("periodic", "fill", "extend")):
        got = ops.stencil_pair(ta, tb, ("interp", 1, 0, "extend", 0.0), (1, "diff", lo_b, 1 - lo_b, bc_b, 2.5), 2,
                               pre_b=tpre, post=tpost, halo_lo_b=tl, halo_hi_b=th)
        assert _capi.last_launch() == label, _capi.last_launch()
        with np.errstate(all="ignore"):
            padded = np.concatenate([planes[0], b * pre_b] if lo_b else [b * pre_b, planes[1]], axis=1)
            tb_ = S.stencil2("diff", padded, 1, 0, 0, None)
            want = ((tb_ - S.stencil2("interp", a, 2, 1, 0, "extend")) / post).astype(dtype)
        np.testing.assert_array_equal(_host(got), want, err_msg=f"lo_b={lo_b} {bc_b}")


# ------------------------------------------------------------------ host twins
def _workspace_bytes():
    v = _capi.i64_array([0])
    _capi.check(_capi.load().xg_host_workspace_bytes(0, v))
    return int(v[0])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("pivot, south", [("corner", "periodic"), ("U", "fill"), (None, "fill")],
                         ids=["fold-periodic", "fold-fill", "plain"])
def test_host_pair_streams_in_slabs(monkeypatch, dtype, pivot, south):
    """Numpy (T, Z, Y, X) fields at 1 MiB slabs: 4 slabs, the last ragged; one pair launch (plus one fold row) per
    slab; equal bit for bit to the device call; device memory bounded by the slab size.  (Z, Y, X) streams too,
    (Y, X) keeps the whole-field path."""
    monkeypatch.setenv("XG_HOST_SLAB_MB", "1")
    ny, nx = 33, 40
    lead = (2, 31)
    rng = np.random.default_rng(50)
    ds, grid = _grid(pivot, south, ny, nx, dtype)
    u = _fields(rng, lead + (ny, nx), dtype, True)
    v = _fields(rng, lead + (ny, nx), dtype, True)
    hu = xg.DataArray(u, dims=("time", "z", "ycenter", "xleft"))
    hv = xg.DataArray(v, dims=("time", "z", "yleft", "xcenter"))
    to = {"X": "center", "Y": "center"}
    es = np.dtype(dtype).itemsize
    per_slab = 2 if pivot else 1
    _capi.check(_capi.load().xg_host_workspace_release())
    # vorticity takes (u, v) = (hv, hu): its x term is hu, its term across the fold hv, as in the divergence
    for fn, (f, g) in ((grid.divergence, (hu, hv)), (grid.vorticity, (hv, hu))):
        fn(f, g, to=to)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.max_memory_allocated()
        n0 = _launches()
        got = fn(f, g, to=to)
        n = _launches() - n0
        assert isinstance(got.data, np.ndarray) and got.dims == ("time", "z", "ycenter", "xcenter")
        rows = min((1 << 20) // (ny * nx * es), -(-62 // 4))
        n_slabs = -(-62 // rows)
        assert n_slabs == 4 and 62 % rows != 0
        assert n == per_slab * n_slabs, (n, n_slabs)
        assert torch.cuda.max_memory_allocated() - base < u.nbytes // 4
        row = ny * nx * es
        assert _workspace_bytes() <= 3 * 3 * rows * row + 3 * row + 2 * rows * nx * es
        dev = fn(xg.DataArray(_dev(f.values), dims=f.dims), xg.DataArray(_dev(g.values), dims=g.dims), to=to)
        np.testing.assert_array_equal(got.data, _host(dev), err_msg=fn.__name__)
    if pivot:
        want = _want("diff", u, "left", "center", "diff", v, "left", "center", "center", pivot, south, "periodic",
                     "sub", _metric(ds, "dy", "center", "left", 4), _metric(ds, "dx", "left", "center", 4),
                     _metric(ds, "area", "center", "center", 4), vector=True)
        np.testing.assert_array_equal(got.data, want)
    # (Z, Y, X): Z is the slab dim; (Y, X): no batch dim, one whole-field device launch
    for sl, launches in ((np.s_[0], per_slab * 4), (np.s_[0, 0], per_slab)):
        hu2 = xg.DataArray(u[sl], dims=hu.dims[-u[sl].ndim:])
        hv2 = xg.DataArray(v[sl], dims=hv.dims[-v[sl].ndim:])
        n0 = _launches()
        got = grid.divergence(hu2, hv2, to=to)
        assert _launches() - n0 == launches
        dev = grid.divergence(xg.DataArray(_dev(u[sl]), dims=hu2.dims), xg.DataArray(_dev(v[sl]), dims=hv2.dims),
                              to=to)
        np.testing.assert_array_equal(_host(got), _host(dev))
