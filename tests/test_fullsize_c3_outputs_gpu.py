"""The benchmark's C3-sized metric-fused and multi-axis calls (75 x 2400 x 3600 fp32, grid and metrics as
``bench.py`` ``run_extras`` builds them), compared with the oracle over EVERY output cell, slab by slab so host
memory stays bounded: operators along X or Y level by level, along Z per block of Y rows with the full Z extent,
the fused X, Y, Z chain per block of Y rows carrying the row below the block (applied with lo = hi = 0 there, so
the block's own rows come out exactly).  Each call also asserts the kernel that served it."""

import numpy as np
import pytest
import torch

from oracle import stencil as oracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 0xC0FFEE
NZ, NY, NX = 75, 2400, 3600
YBLOCK = 80


@pytest.fixture(scope="module")
def c3():
    """The field, the second velocity component, dx(Y, X) and dz(Z), and the grid of run_extras."""
    import xgcm_b200 as xg
    from xgcm_b200 import ops

    x = ops.fill_uniform(torch.empty((NZ, NY, NX), dtype=torch.float32, device=DEV), SEED)
    v = ops.fill_uniform(torch.empty_like(x), SEED + 7)
    jj = np.arange(NY, dtype=np.float64)[:, None]
    dx = (1e3 * (1 + 0.1 * np.cos(2 * np.pi * jj / NY)) * np.ones((1, NX))).astype(np.float32)
    dz = (10 * 1.05 ** np.arange(NZ)).astype(np.float32)
    ds = xg.Dataset(coords={"Z": np.arange(NZ) + 0.5, "Zl": np.arange(NZ) + 0.0, "YC": np.arange(NY) + 0.5,
                            "YG": np.arange(NY) + 0.0, "XC": np.arange(NX) + 0.5, "XG": np.arange(NX) + 0.0})
    for nm, dims, arr in (("dxC", ("YC", "XC"), dx), ("dxG", ("YC", "XG"), dx), ("drF", ("Z",), dz), ("drC", ("Zl",), dz)):
        ds[nm] = xg.DataArray(torch.from_numpy(arr).to(DEV), dims=dims)
    grid = xg.Grid(ds, coords={"X": {"center": "XC", "left": "XG"}, "Y": {"center": "YC", "left": "YG"},
                               "Z": {"center": "Z", "left": "Zl"}},
                   metrics={("X",): ["dxC", "dxG"], ("Z",): ["drF", "drC"]},
                   padding={"X": "periodic", "Y": "fill", "Z": "extend"}, autoparse_metadata=False)
    da = xg.DataArray(x, dims=("Z", "YC", "XC"))
    yield {"x": x, "v": v, "dx": dx, "dz": dz, "grid": grid, "da": da}
    del x, v


def _label():
    from xgcm_b200 import _capi

    torch.cuda.synchronize()
    return _capi.last_launch()


def test_c3_derivative_x_every_cell(c3):
    out = c3["grid"].derivative(c3["da"], "X").data
    assert _label() == "xg_stencil2(row_tma)"
    assert tuple(out.shape) == (NZ, NY, NX)
    for k in range(NZ):
        want = oracle.stencil2("diff", c3["x"][k].cpu().numpy(), 1, 1, 0, "periodic", 0.0, None, c3["dx"])
        np.testing.assert_array_equal(out[k].cpu().numpy(), want, err_msg=f"level {k}")


def test_c3_metric_weighted_interp_z_every_cell(c3):
    out = c3["grid"].interp(c3["da"], "Z", metric_weighted="Z").data
    assert _label() == "xg_stencil2(tile_tma)"
    assert tuple(out.shape) == (NZ, NY, NX)
    dz = c3["dz"].reshape(NZ, 1, 1)
    for j0 in range(0, NY, YBLOCK):
        a = c3["x"][:, j0:j0 + YBLOCK].cpu().numpy()
        want = oracle.stencil2("interp", a, 0, 1, 0, "extend", 0.0, dz, dz)  # x drF, / drC (both dz here)
        np.testing.assert_array_equal(out[:, j0:j0 + YBLOCK].cpu().numpy(), want, err_msg=f"rows {j0}+")


def test_c3_interp_xyz_every_cell(c3):
    out = c3["grid"].interp(c3["da"], ["X", "Y", "Z"]).data
    assert _label() == "xg_stencil_multi(tile_tma)"
    assert tuple(out.shape) == (NZ, NY, NX)
    for j0 in range(0, NY, YBLOCK):
        j1 = min(j0 + YBLOCK, NY)
        h = 1 if j0 > 0 else 0  # the row below a cut: Y then needs no padding on that side
        a = c3["x"][:, j0 - h:j1].cpu().numpy()
        t = oracle.stencil2("interp", a, 2, 1, 0, "periodic", 0.0)
        t = oracle.stencil2("interp", t, 1, 1 - h, 0, "fill" if not h else None, 0.0)
        want = oracle.stencil2("interp", t, 0, 1, 0, "extend", 0.0)
        assert want.shape == (NZ, j1 - j0, NX)
        np.testing.assert_array_equal(out[:, j0:j1].cpu().numpy(), want, err_msg=f"rows {j0}+")


@pytest.mark.parametrize("subtract", [0, 1])
def test_c3_divergence_and_vorticity_every_cell(c3, subtract):
    """(diff(u dy, X) +|- diff(v dx, Y)) / rA in one pass; subtract=1 is the vorticity form."""
    from xgcm_b200 import ops

    dx_t = torch.from_numpy(c3["dx"]).to(DEV)
    area_t = dx_t * dx_t
    area = area_t.cpu().numpy()
    out = ops.stencil_pair(c3["x"], c3["v"], ("diff", 0, 1, "periodic", 0.0), (1, "diff", 0, 1, "periodic", 0.0),
                           subtract, pre_a=dx_t, pre_b=dx_t, post=area_t)
    assert _label() == "xg_stencil_pair(tile_tma)"
    for k in range(NZ):
        u, v = c3["x"][k].cpu().numpy(), c3["v"][k].cpu().numpy()
        want = oracle.stencil_pair("diff", u, 1, 0, 1, "periodic", 0.0, c3["dx"], "diff", v, 0, 0, 1, "periodic", 0.0,
                                   c3["dx"], subtract, area)
        np.testing.assert_array_equal(out[k].cpu().numpy(), want, err_msg=f"level {k}")
