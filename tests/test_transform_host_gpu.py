"""xg_vinterp_conservative_host (and the theta streaming of xg_vinterp_linear_host) on the GPU: bit for bit against
the device entry points and the oracle, with several slabs per call (XG_HOST_SLAB_MB=1) and with the default."""

import ctypes as C
import warnings

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from oracle import stencil as oracle
from test_transform_host import slab_dim, slab_rows, transform_total_bytes
from xgcm_b200 import _capi, ops

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["1", None], ids=["slab1MB", "default"])
def slab_env(request, monkeypatch):
    if request.param is None:
        monkeypatch.delenv("XG_HOST_SLAB_MB", raising=False)
    else:
        monkeypatch.setenv("XG_HOST_SLAB_MB", request.param)
    return request.param


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _device_ref(phi, theta, bins, axis):
    return ops.vinterp_conservative(_cuda(phi), _cuda(theta), _cuda(bins), axis).cpu().numpy()


def _fields(shape, axis, dtype, seed=0, theta="dense"):
    rng = np.random.default_rng(seed)
    phi = rng.random(shape).astype(dtype)
    phi[rng.random(shape) < 0.03] = np.nan
    tshape = list(shape)
    tshape[axis] += 1
    if theta == "dense":
        th = np.cumsum(0.5 + rng.random(tshape), axis=axis).astype(dtype)
        flat = np.moveaxis(th, axis, -1).reshape(-1, tshape[axis])
        if flat.shape[0] > 8 and tshape[axis] > 3:
            flat[:3] = flat[:3, ::-1]                # non-monotonic columns
            flat[3, 1] = np.nan                      # one NaN bound
            flat[4, 1:3] = np.nan                    # two NaN bounds
        th = np.moveaxis(flat.reshape([tshape[d] for d in range(len(shape)) if d != axis] + [tshape[axis]]), -1, axis)
        th = np.ascontiguousarray(th)
    elif theta == "1d":
        v = np.cumsum(0.5 + rng.random(tshape[axis])).astype(dtype)
        th = v.reshape([tshape[axis] if d == axis else 1 for d in range(len(shape))])
    else:  # (T, Z+1, 1, 1): dense along the leading dims only
        lead = [tshape[d] if d <= axis else 1 for d in range(len(shape))]
        th = np.cumsum(0.5 + rng.random(lead), axis=axis).astype(dtype)
    return phi, th


CASES = [
    # shape, axis, theta layout
    ((6, 9, 40, 70), 1, "dense"),
    ((6, 9, 40, 70), 1, "1d"),
    ((6, 9, 40, 70), 1, "lead"),
    ((1, 12, 50, 64), 1, "dense"),     # leading size-1 dim
    ((11, 60, 80), 0, "dense"),        # axis first
    ((40, 30, 13), 2, "dense"),        # axis last
    ((25, 14, 33), 1, "1d"),           # axis in the middle
    ((17,), 0, "dense"),               # 1-D
]


@pytest.mark.parametrize("shape,axis,theta", CASES)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("direction", ["up", "down"])
def test_conservative_host_matches_device_and_oracle(slab_env, shape, axis, theta, dtype, direction):
    phi, th = _fields(shape, axis, dtype, theta=theta)
    hi = float(np.nanmax(th)) + 1
    bins = np.linspace(0, hi, 12).astype(dtype)
    if direction == "down":
        bins = bins[::-1].copy()
    got = ops.vinterp_conservative_host(phi, th, bins, axis)
    assert got.dtype == dtype
    tshape = list(shape)
    tshape[axis] += 1
    full = np.broadcast_to(th, tshape)
    np.testing.assert_array_equal(got, _device_ref(phi, full, bins, axis))
    np.testing.assert_array_equal(got, oracle.vinterp_conservative(phi, full, bins, axis))


def test_conservative_host_mixed_dtype_promotes(slab_env):
    phi, th = _fields((5, 9, 30, 40), 1, np.float32)
    bins = np.linspace(0, float(np.nanmax(th)) + 1, 9).astype(np.float32).astype(np.float64)  # exact in f32
    got = ops.vinterp_conservative_host(phi, th.astype(np.float64), bins.astype(np.float32), 1)
    assert got.dtype == np.float64
    np.testing.assert_array_equal(got, _device_ref(phi.astype(np.float64), th.astype(np.float64), bins, 1))
    np.testing.assert_array_equal(got, oracle.vinterp_conservative(phi.astype(np.float64), th.astype(np.float64),
                                                                   bins, 1))


@pytest.mark.parametrize("dtype,m", [(np.float32, 1700), (np.float64, 900)])
def test_conservative_host_multipass_bins(slab_env, dtype, m):
    """More bins than one shared-memory tile holds: the multi-pass configuration with one warp per block."""
    phi, th = _fields((4, 10, 24, 40), 1, dtype, seed=5)
    bins = np.linspace(0, float(np.nanmax(th)) + 1, m).astype(dtype)
    got = ops.vinterp_conservative_host(phi, th, bins, 1)
    np.testing.assert_array_equal(got, _device_ref(phi, th, bins, 1))
    np.testing.assert_array_equal(got, oracle.vinterp_conservative(phi, th, bins, 1))


def test_conservative_host_degenerate_sizes(slab_env):
    phi, th = _fields((3, 6, 5), 1, np.float64)
    got = ops.vinterp_conservative_host(phi, th, np.array([1.0]), 1)
    assert got.shape == (3, 5, 0)
    # zero-length operated axis: every bin NaN, as k_vconserv leaves bins that receive nothing
    phi0 = np.zeros((3, 0, 5))
    th0 = np.zeros((3, 1, 5))
    bins = np.linspace(0, 1, 4)
    for dtype in (np.float32, np.float64):
        got = ops.vinterp_conservative_host(phi0.astype(dtype), th0.astype(dtype), bins.astype(dtype), 1)
        assert got.shape == (3, 5, 3) and got.dtype == dtype and np.isnan(got).all()


@pytest.mark.parametrize("theta", ["dense", "1d"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_centred_theta_equals_interp_extend_then_twin(slab_env, theta, dtype):
    rng = np.random.default_rng(9)
    shape, axis = (4, 12, 30, 50), 1
    phi = rng.random(shape).astype(dtype)
    if theta == "dense":
        tc = np.cumsum(0.5 + rng.random(shape), axis=axis).astype(dtype)
    else:
        tc = np.cumsum(0.5 + rng.random(shape[axis])).astype(dtype).reshape(1, -1, 1, 1)
    bounds = ops.stencil2(_cuda(tc), axis, "interp", 1, 1, "extend").cpu().numpy()
    bins = np.linspace(0, float(bounds.max()) + 1, 10).astype(dtype)
    got = ops.vinterp_conservative_host(phi, tc, bins, axis, theta_at_centers=True)
    np.testing.assert_array_equal(got, ops.vinterp_conservative_host(phi, bounds, bins, axis))
    np.testing.assert_array_equal(got, oracle.vinterp_conservative(
        phi, np.broadcast_to(oracle.stencil2("interp", tc, axis, 1, 1, "extend").astype(dtype),
                             (4, 13, 30, 50)), bins, axis))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_linear_host_with_a_dense_theta_field_still_equals_the_device(slab_env, dtype):
    rng = np.random.default_rng(2)
    shape = (5, 14, 40, 60)
    phi = rng.random(shape).astype(dtype)
    th = np.cumsum(0.1 + rng.random(shape), axis=1).astype(dtype)
    levels = np.linspace(0, float(th.max()), 17).astype(dtype)
    got = ops.vinterp_linear_host(phi, th, levels, 1, mask_edges=True)
    want = ops.vinterp_linear(_cuda(phi), _cuda(th), _cuda(levels), 1, mask_edges=True).cpu().numpy()
    np.testing.assert_array_equal(got, want)


def _grid_case(dtype):
    rng = np.random.default_rng(21)
    nt, nz, ny, nx = 3, 10, 24, 36
    q = rng.random((nt, nz, ny, nx)).astype(dtype)
    sig = np.cumsum(0.5 + rng.random((nt, nz + 1, ny, nx)), axis=1).astype(dtype)
    tc = np.cumsum(0.5 + rng.random((nt, nz, ny, nx)), axis=1).astype(dtype)
    coords = {"z": np.arange(nz) + 0.5, "zo": np.arange(nz + 1.0)}
    dims4 = ("t", "z", "y", "x")
    host = xg.Dataset(data_vars={"q": (dims4, q), "sig": (("t", "zo", "y", "x"), sig), "tc": (dims4, tc)},
                      coords=coords)
    dev = xg.Dataset(data_vars={"q": (dims4, _cuda(q)), "sig": (("t", "zo", "y", "x"), _cuda(sig)),
                                "tc": (dims4, _cuda(tc))}, coords=coords)
    grid = {"Z": {"center": "z", "outer": "zo"}}
    return xg.Grid(host, coords=grid), host, xg.Grid(dev, coords=grid), dev, float(sig.max()) + 1


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("theta", ["sig", "tc"])
@pytest.mark.parametrize("method", ["conservative", "linear"])
def test_grid_transform_numpy_equals_device(slab_env, monkeypatch, dtype, theta, method):
    gh, host, gd, dev, hi = _grid_case(dtype)
    if method == "linear" and theta == "sig":
        pytest.skip("linear transforms take theta at the field's own position")
    calls = {"host": 0, "device": 0}
    host_fn, dev_fn = ops.vinterp_conservative_host, ops.vinterp_conservative

    def spy_host(*a, **k):
        calls["host"] += 1
        return host_fn(*a, **k)

    def spy_dev(*a, **k):
        calls["device"] += 1
        return dev_fn(*a, **k)

    bins = np.linspace(0, hi, 14).astype(dtype)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = gd.transform(dev["q"], "Z", bins, target_data=dev[theta], method=method)
        monkeypatch.setattr(ops, "vinterp_conservative_host", spy_host)
        monkeypatch.setattr(ops, "vinterp_conservative", spy_dev)
        got = gh.transform(host["q"], "Z", bins, target_data=host[theta], method=method)
    assert isinstance(got.data, np.ndarray)
    assert got.dims == want.dims and got.name == want.name
    np.testing.assert_array_equal(got.values, want.values)
    for k in got.coords:
        np.testing.assert_array_equal(got.coords[k].values, want.coords[k].values)
    if method == "conservative":
        assert calls == {"host": 1, "device": 0}


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_grid_transform_centred_theta_equals_interp_then_twin(slab_env, dtype):
    gh, host, _, _, hi = _grid_case(dtype)
    bins = np.linspace(0, hi, 14).astype(dtype)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got = gh.transform(host["q"], "Z", bins, target_data=host["tc"], method="conservative")
    bounds = gh.interp(host["tc"], "Z", padding="extend")
    want = ops.vinterp_conservative_host(host["q"].values, bounds.values, bins, 1)
    np.testing.assert_array_equal(got.values, want)


def test_workspace_stays_within_the_slab_bound(monkeypatch):
    """phi and theta of 64+ MB each with a 1 MB slab budget: the pipe workspace holds three slots of the per-index
    slab plus the bins -- far below theta, so theta streamed rather than went up whole."""
    monkeypatch.setenv("XG_HOST_SLAB_MB", "1")
    lib = _capi.load()
    lib.xg_host_workspace_release()
    shape, axis, m = (4, 32, 256, 512), 1, 11
    rng = np.random.default_rng(1)
    phi = ops.pinned_empty(shape, np.float32)
    phi[...] = rng.random(shape, dtype=np.float32)
    tshape = (4, 33, 256, 512)
    th = ops.pinned_empty(tshape, np.float32)
    th[...] = np.cumsum(rng.random(tshape, dtype=np.float32) + 0.5, axis=1)
    assert phi.nbytes >= 64 << 20 and th.nbytes >= 64 << 20
    bins = np.linspace(0, float(th.max()) + 1, m).astype(np.float32)
    got = ops.vinterp_conservative_host(phi, th, bins, axis)
    total = transform_total_bytes(shape, axis, m - 1, 4)
    sd = slab_dim(shape, axis, total, budget=1 << 20)
    rows = slab_rows(shape[sd], total // shape[sd], budget=1 << 20)
    bound = 3 * rows * (total // shape[sd]) + m * 4
    used = C.c_int64(0)
    assert lib.xg_host_pipe_workspace_bytes(torch.cuda.current_device(), C.byref(used)) == 0
    assert 0 < used.value <= bound and used.value < th.nbytes // 8
    # spot-check a few columns against the oracle
    for t, y, x in ((0, 0, 0), (3, 255, 511), (2, 100, 7)):
        np.testing.assert_array_equal(got[t, y, x], oracle.vinterp_conservative(phi[t, :, y, x], th[t, :, y, x], bins, 0))
    lib.xg_host_workspace_release()
