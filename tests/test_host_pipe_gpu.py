"""Host-buffer twins (csrc/xg_host_pipe.cu): slab pipelines must give exactly the device entry points' results.

xg_stencil2_host_multi / xg_cumscan_host / xg_wreduce_host / xg_vinterp_linear_host against the oracle
(bit-exact where the device kernels are), with slab sizes small enough that every case is cut into several
slabs (XG_HOST_SLAB_MB=1) and once with the default.
"""

import numpy as np
import pytest

from oracle import stencil as oracle

pytestmark = pytest.mark.gpu


def _field(shape, dtype, seed=0, nan_frac=0.0):
    rng = np.random.default_rng(seed)
    a = rng.random(shape).astype(dtype)
    if nan_frac:
        a[rng.random(shape) < nan_frac] = np.nan
    return a


@pytest.fixture(params=["1", None], ids=["slab1MB", "default"])
def slab(request, monkeypatch):
    if request.param:
        monkeypatch.setenv("XG_HOST_SLAB_MB", request.param)
    return request.param


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape", [(40, 96, 200), (9, 33, 70), (300, 1000), (5000,)])
def test_stencil2_host_multi_matches_oracle(slab, dtype, shape):
    from xgcm_b200 import ops

    a = _field(shape, dtype, seed=3, nan_frac=0.01)
    nd = len(shape)
    specs = []
    for axis in range(nd):
        specs.append((axis, "diff", 1, 0, "periodic", 0.0))
        specs.append((axis, "interp", 0, 1, "fill", 1.5))
    specs = specs[:8]
    if nd >= 2:
        specs[-1] = (nd - 1, "max", 1, 1, "extend", 0.0)   # outer shift on a non-slab dim: n + 1 outputs
        specs[-2] = (nd - 1, "min", 0, 0, None, 0.0)       # inner shift: n - 1 outputs
    outs = ops.stencil2_host_multi(a, specs)
    for (axis, op, lo, hi, bc, fv), got in zip(specs, outs):
        want = oracle.stencil2(op, a, axis, lo, hi, bc, fv)
        np.testing.assert_array_equal(got, want, err_msg=f"{op} axis={axis} ({lo},{hi}) {bc}")


def test_stencil2_host_multi_refuses_what_it_cannot_slab():
    from xgcm_b200 import ops

    a = _field((8, 16, 32), np.float32)
    with pytest.raises(NotImplementedError):
        ops.stencil2_host_multi(a, [(0, "diff", 1, 1, "fill", 0.0)])  # outer shift along dim 0
    with pytest.raises(ValueError):
        ops.stencil2_host_multi(a, [(1, "diff", 1, 0, None, 0.0)])   # pad without a boundary condition


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape,axis", [((30, 64, 100), 0), ((30, 64, 100), 1), ((30, 64, 100), 2), ((70, 500), 0),
                                        ((70, 500), 1), ((4000,), 0)])
def test_cumscan_host_matches_oracle(slab, dtype, shape, axis):
    from xgcm_b200 import ops

    a = _field(shape, dtype, seed=4, nan_frac=0.01)
    rng = np.random.default_rng(5)
    mshape = [1] * len(shape)
    mshape[axis] = shape[axis]
    for reverse, trim, pl, ph, bc in [(False, "none", 0, 0, None), (False, "drop_last", 1, 0, "fill"),
                                      (True, "drop_first", 0, 1, "extend"), (False, "none", 1, 0, "periodic")]:
        kept = shape[axis] - (0 if trim == "none" else 1)
        oshape = list(shape)
        oshape[axis] = kept + pl + ph
        pre = (rng.random(shape) + 0.5).astype(dtype)
        post = (rng.random(oshape) + 0.5).astype(dtype) if len(shape) < 3 else None
        want = oracle.cumscan(a, axis, reverse, trim, pl, ph, bc, 0.25, pre, post, True)
        got = ops.cumscan_host(a, axis, reverse, trim, pl, ph, bc, 0.25, pre=pre, post=post)
        np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape,axis", [((30, 64, 100), 0), ((30, 64, 100), 1), ((30, 64, 100), 2), ((3000,), 0)])
def test_wreduce_host_matches_oracle(slab, dtype, shape, axis):
    from xgcm_b200 import ops

    a = _field(shape, dtype, seed=6, nan_frac=0.02)
    rng = np.random.default_rng(7)
    wshape = [1] * len(shape)
    wshape[axis] = shape[axis]
    w1 = (rng.random(wshape) + 0.5).astype(dtype)
    wfull = (rng.random(shape) + 0.5).astype(dtype)
    for w in (None, w1, wfull):
        for mode, skipna in (("sum", True), ("sum", False), ("mean", True), ("mean", False)):
            if mode == "mean" and w is None:
                continue
            want = oracle.wreduce(a, w, axis, mode, skipna)
            got = ops.wreduce_host(a, axis, w, mode, skipna)
            if axis == len(shape) - 1:  # contiguous axis: fp64 accumulation rounded once, against the exact sum
                from test_kernel_instances_gpu import _fsum_bound_check

                _fsum_bound_check(got, a, w, axis, mode, skipna, f"{shape} {mode} skipna={skipna}")
            else:
                np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_vinterp_linear_host_matches_oracle(slab, dtype):
    from xgcm_b200 import ops

    rng = np.random.default_rng(8)
    for shape, axis in [((25, 40, 64), 0), ((6, 25, 64), 1), ((12, 30), 1), ((40,), 0)]:
        phi = _field(shape, dtype, seed=9, nan_frac=0.01)
        n = shape[axis]
        th1 = np.cumsum(0.1 + rng.random(n)).astype(dtype)
        b = [1] * len(shape)
        b[axis] = n
        theta = th1.reshape(b)
        target = np.linspace(th1[0] - 0.2, th1[-1] + 0.2, 17).astype(dtype)
        want = oracle.vinterp_linear(phi, np.broadcast_to(theta, shape), target, axis, True, False)
        got = ops.vinterp_linear_host(phi, theta, target, axis, True, False)
        np.testing.assert_array_equal(got, want)
        if len(shape) == 3 and axis == 0:  # theta as a full field: uploaded whole, offset per slab
            thf = np.cumsum(0.1 + rng.random(shape), axis=0).astype(dtype)
            want = oracle.vinterp_linear(phi, thf, target, 0, True, False)
            np.testing.assert_array_equal(ops.vinterp_linear_host(phi, thf, target, 0, True, False), want)


def test_grid_host_paths_equal_device_paths():
    """Grid.cumsum / cumint / integrate / average / transform / apply_many on numpy-backed fields go through
    the host twins and must equal the device-resident results bit for bit."""
    import torch

    import xgcm_b200 as xg

    nz, ny, nx = 20, 48, 96
    rng = np.random.default_rng(11)
    a = rng.random((nz, ny, nx)).astype(np.float32)
    a[rng.random(a.shape) < 0.01] = np.nan
    dz = (10 * 1.05 ** np.arange(nz)).astype(np.float32)
    depth = (np.cumsum(dz) - dz / 2).astype(np.float32)
    ds = xg.Dataset(coords={"Z": depth, "Zl": depth - dz / 2, "YC": np.arange(ny) + 0.5, "YG": np.arange(ny) + 0.0,
                            "XC": np.arange(nx) + 0.5, "XG": np.arange(nx) + 0.0})
    ds["drF"] = xg.DataArray(dz, dims=("Z",))
    ds["drC"] = xg.DataArray(dz, dims=("Zl",))
    grid = xg.Grid(ds, coords={"X": {"center": "XC", "left": "XG"}, "Y": {"center": "YC", "left": "YG"},
                               "Z": {"center": "Z", "left": "Zl"}}, metrics={("Z",): ["drF", "drC"]},
                   padding={"X": "periodic", "Y": "fill", "Z": "extend"}, autoparse_metadata=False)
    host = xg.DataArray(a, dims=("Z", "YC", "XC"), name="t")
    dev = xg.DataArray(torch.from_numpy(a).cuda(), dims=("Z", "YC", "XC"), name="t")

    def same(h, d):
        assert isinstance(h.data, np.ndarray) and h.dims == d.dims
        np.testing.assert_array_equal(h.data, d.data.cpu().numpy())

    same(grid.cumsum(host, "Z", padding="fill"), grid.cumsum(dev, "Z", padding="fill"))
    same(grid.cumsum(host, "X"), grid.cumsum(dev, "X"))
    same(grid.cumint(host, "Z", padding="fill"), grid.cumint(dev, "Z", padding="fill"))
    same(grid.integrate(host, "Z"), grid.integrate(dev, "Z"))
    same(grid.average(host, "Z"), grid.average(dev, "Z"))
    same(grid.average(host, "Z", skipna=False), grid.average(dev, "Z", skipna=False))
    levels = np.linspace(depth[0] - 1, depth[-1] + 1, 12).astype(np.float32)
    same(grid.transform(host, "Z", levels), grid.transform(dev, "Z", levels))
    reqs = [("diff", "X"), ("interp", "X"), ("diff", "Y"), ("interp", "Y"), ("diff", "Z"), ("interp", "Z")]
    for h, d, (f, ax) in zip(grid.apply_many(host, reqs), grid.apply_many(dev, reqs), reqs):
        same(h, d)
        same(h, getattr(grid, f)(dev, ax))
    # cumint == cumsum of the explicit product (the reference's formulation, grid.py:1656-1660)
    prod = dev * ds["drF"].to_device(dev.data.device)
    np.testing.assert_array_equal(grid.cumint(dev, "Z", padding="fill").data.cpu().numpy(),
                                  grid.cumsum(prod, "Z", padding="fill").data.cpu().numpy())
    # skipna=False: a NaN cell makes its column's mean NaN (da.weighted(w).mean(skipna=False))
    got = grid.average(dev, "Z", skipna=False).data.cpu().numpy()
    assert np.array_equal(np.isnan(got), np.isnan(a).any(axis=0))
    with pytest.raises(NotImplementedError):
        grid.integrate(dev, "Z", min_count=1)
