"""The conservative transform's host twin on CPU: argument checks of its C-ABI (no GPU needed), the routes
Grid.transform / conservative_interpolation / interp_1d_conservative take for numpy and device inputs (kernels
replaced by the oracle, tests/_mock_transform.py), and the slab-dim rule of the transform twins restated."""

import ctypes as C
import warnings

import numpy as np
import pytest
import torch

import xgcm_b200 as xg
from oracle import stencil as oracle
from xgcm_b200 import _capi


# ---------------------------------------------------------------------------------------------- C-ABI, no GPU
def _conservative_host(lib, phi=True, theta=True, strides=(1,), centers=0, bins=True, m=4, dtype=0, ndim=1,
                       shape=(3,), axis=0, out=True):
    buf = (C.c_double * 64)()
    return lib.xg_vinterp_conservative_host(
        dtype, buf if phi else None, buf if theta else None, _capi.i64_array(strides) if strides else None, centers,
        buf if bins else None, m, 0, buf if out else None, ndim, _capi.i64_array(shape) if shape else None, axis, 0)


@pytest.mark.parametrize("kwargs,msg", [
    (dict(phi=False), "null"),
    (dict(theta=False), "null"),
    (dict(bins=False), "null"),
    (dict(out=False), "null"),
    (dict(shape=None), "null"),
    (dict(strides=None), "strides missing"),
    (dict(dtype=7), "dtype"),
    (dict(ndim=0), "ndim"),
    (dict(ndim=9, shape=(3,) * 9, strides=(1,) * 9), "ndim"),
    (dict(axis=1), "axis"),
    (dict(axis=-1), "axis"),
    (dict(shape=(-3,)), "negative extent"),
    (dict(m=1), "two bin edges"),
    (dict(strides=(0,)), "broadcast along"),                          # 4 bounds wanted, theta broadcast along axis
    (dict(strides=(0,), centers=1), "broadcast along"),               # 3 centres wanted
    (dict(strides=(-1,)), "negative theta stride"),
    # centres, broadcast over dim 1 and not C-contiguous over dims 0, 2: the center -> outer stencil cannot read it
    (dict(ndim=3, shape=(2, 3, 4), axis=0, strides=(1, 0, 2), centers=1), "C-contiguous"),
])
def test_capi_rejects_bad_arguments_without_gpu(kwargs, msg):
    lib = _capi.load()
    assert _conservative_host(lib, **kwargs) == -1
    assert msg in _capi.last_error()


def test_capi_zero_length_axis_gives_nan_bins_without_gpu():
    """No source cells: every bin stays NaN, as k_vconserv leaves it; nothing touches a device."""
    lib = _capi.load()
    for dtype, ct in ((0, C.c_float), (1, C.c_double)):
        phi, theta, bins = (ct * 1)(), (ct * 3)(), (ct * 4)(0, 1, 2, 3)
        out = (ct * 9)(*([7.0] * 9))
        rc = lib.xg_vinterp_conservative_host(dtype, phi, theta, _capi.i64_array([1, 1]), 0, bins, 4, 0, out, 2,
                                              _capi.i64_array([3, 0]), 1, 0)
        assert rc == 0
        assert np.isnan(np.array(out[:])).all()


def test_workspace_query_arguments_without_gpu():
    lib = _capi.load()
    assert lib.xg_host_pipe_workspace_bytes(0, None) == -1 and "null" in _capi.last_error()
    got = C.c_int64(-1)
    assert lib.xg_host_pipe_workspace_bytes(12345, C.byref(got)) == 0 and got.value == 0  # no workspace there


# ------------------------------------------------------------------------------------- slab-dim rule, restated
def slab_dim(shape, axis, per_index_total_bytes, budget=128 << 20):
    """xg_host_pipe.cu transform_slab_dim: the outermost non-operated dim of extent > 1 whose one index (its share of
    phi + streamed theta + theta-bounds scratch + result bytes) fits the slab budget; else the innermost such dim;
    -1 when there is none."""
    total = per_index_total_bytes
    inner = -1
    for d, n in enumerate(shape):
        if d == axis or n <= 1:
            continue
        if total // n <= budget:
            return d
        inner = d
    return inner


def slab_rows(L, row_bytes, budget=128 << 20):
    """xg_host.cu slab_rows: the budget's rows, at least one, and at least 4 slabs when the dim allows."""
    rows = max(1, budget // row_bytes) if row_bytes > 0 else L
    return max(1, min(rows, (L + 3) // 4))


def transform_total_bytes(shape, axis, m_out, itemsize, theta="dense", centers=False):
    """Bytes of phi, the streamed theta, the theta-bounds scratch and the result of a transform-twin call."""
    n = int(np.prod(shape))
    cols = n // shape[axis] if shape[axis] else int(np.prod([s for d, s in enumerate(shape) if d != axis]))
    tn = shape[axis] + (0 if centers else 1)
    th = cols * tn if theta == "dense" else 0
    scratch = cols * (shape[axis] + 1) if theta == "dense" and centers else 0
    return (n + th + scratch + cols * m_out) * itemsize


@pytest.mark.parametrize("shape,axis,want", [
    ((1, 75, 3059, 4322), 1, 2),   # NEMO (time_counter=1, deptht, y, x): the length-1 dim is skipped
    ((2, 75, 3059, 4322), 1, 2),   # a short time axis whose one index is far over the budget
    ((12, 75, 300, 400), 1, 0),    # one time index fits: the outermost dim
    ((75, 3059, 4322), 0, 1),      # (Z, Y, X), axis 0
    ((3059, 4322, 75), 2, 0),      # (Y, X, Z), axis last
    ((75,), 0, -1),                # 1-D: one slab
    ((1, 75, 1, 1), 1, -1),        # nothing but the axis has extent > 1
])
def test_slab_dim_rule(shape, axis, want):
    total = transform_total_bytes(shape, axis, 60, 4)
    assert slab_dim(shape, axis, total) == want


def test_slab_dim_rule_falls_back_to_the_innermost_dim():
    # with a 1 MB budget no single index of (8, 64, 4096, 4096) fits: the innermost non-operated dim is cut
    shape = (8, 64, 4096, 4096)
    total = transform_total_bytes(shape, 1, 60, 4)
    assert slab_dim(shape, 1, total, budget=1 << 20) == 3
    # the rows come from the per-index total, not from phi alone: m >> n makes the result dominate
    shape, m_out = (40, 2, 30, 30), 5000
    total = transform_total_bytes(shape, 1, m_out, 8)
    sd = slab_dim(shape, 1, total)
    assert sd == 0 and slab_rows(shape[0], total // shape[0]) == 3 < slab_rows(shape[0], 8 * 2 * 30 * 30) == 10


# ------------------------------------------------------------------------------------------- routes (mocked)
@pytest.fixture
def mocked(monkeypatch):
    import _mock_transform

    _mock_transform.install(monkeypatch)
    from xgcm_b200 import ops

    device_calls = []
    plain = ops.vinterp_conservative

    def spy(*a, **k):
        device_calls.append(a)
        return plain(*a, **k)

    monkeypatch.setattr(ops, "vinterp_conservative", spy)
    return _mock_transform.CALLS, device_calls


def _dataset(dtype=np.float64, left=False, seed=3):
    rng = np.random.default_rng(seed)
    nt, nz, ny, nx = 2, 6, 3, 5
    q = rng.random((nt, nz, ny, nx)).astype(dtype)
    bounds = np.cumsum(0.5 + rng.random((nt, nz + 1, ny, nx)), axis=1).astype(dtype)
    cent = np.cumsum(0.5 + rng.random((nt, nz, ny, nx)), axis=1).astype(dtype)
    coords = {"z": np.arange(nz) + 0.5, "zo": np.arange(nz + 1.0)}
    zc = {"center": "z", "outer": "zo"}
    if left:
        coords["zl"] = np.arange(nz + 0.0)
        zc["left"] = "zl"
    ds = xg.Dataset(data_vars={"q": (("t", "z", "y", "x"), q), "sig": (("t", "zo", "y", "x"), bounds),
                               "tc": (("t", "z", "y", "x"), cent)}, coords=coords)
    return ds, xg.Grid(ds, coords={"Z": zc}), q, bounds, cent


def test_grid_transform_sends_numpy_fields_to_the_twin(mocked):
    calls, device_calls = mocked
    ds, grid, q, bounds, _ = _dataset()
    bins = np.linspace(0, 12, 9)
    got = grid.transform(ds["q"], "Z", bins, target_data=ds["sig"], method="conservative")
    assert isinstance(got.data, np.ndarray) and got.dims == ("t", "y", "x", "sig")
    assert len(calls) == 1 and not device_calls
    c = calls[0]
    assert c["axis"] == 1 and c["theta_at_centers"] == 0 and c["flip"] == 0 and c["m"] == 9
    assert c["theta_shape"] == bounds.shape and c["theta_strides"] == (7 * 15, 15, 5, 1)  # dense theta field
    np.testing.assert_array_equal(got.values, oracle.vinterp_conservative(q, bounds, bins, 1))
    np.testing.assert_array_equal(got.coords["sig"].values, (bins[1:] + bins[:-1]) / 2)
    # decreasing bins: the twin gets them ascending and flips its output
    got = grid.transform(ds["q"], "Z", bins[::-1].copy(), target_data=ds["sig"], method="conservative")
    assert calls[-1]["flip"] == 1
    np.testing.assert_array_equal(got.values, oracle.vinterp_conservative(q, bounds, bins[::-1].copy(), 1))


def test_conservative_interpolation_routes_and_broadcast_theta(mocked):
    from xgcm_b200.transform import conservative_interpolation

    calls, device_calls = mocked
    ds, grid, q, _, _ = _dataset(np.float32)
    zo = xg.DataArray(np.arange(7.0, dtype=np.float32) * 1.5, dims=("zo",))
    bins = xg.DataArray(np.linspace(0, 9, 6).astype(np.float32), dims=("lev",))
    got = conservative_interpolation(ds["q"], zo, bins, "z", "zo", "lev", suffix="_c", grid=grid)
    assert got.name == "q_c" and got.dims == ("t", "y", "x", "lev") and got.dtype == np.float32
    assert len(calls) == 1 and not device_calls
    assert calls[0]["theta_strides"] == (0, 1, 0, 0) and calls[0]["dtype"] == np.float32
    want = oracle.vinterp_conservative(q, np.broadcast_to(zo.values.reshape(1, 7, 1, 1), (2, 7, 3, 5)), bins.values, 1)
    np.testing.assert_array_equal(got.values, want)
    # mixed dtypes promote to f64, as on the device route
    got = conservative_interpolation(ds["q"], zo.astype(np.float64), bins, "z", "zo", "lev", grid=grid)
    assert got.dtype == np.float64 and calls[-1]["dtype"] == np.float64


def test_centred_theta_is_fused_and_warns_once(mocked):
    calls, device_calls = mocked
    ds, grid, q, _, cent = _dataset()
    bins = np.linspace(0, 12, 9)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        got = grid.transform(ds["q"], "Z", bins, target_data=ds["tc"], method="conservative")
    assert [str(w.message).startswith("The `target data` input is not located on the cell bounds") for w in rec] == [True]
    assert len(calls) == 1 and not device_calls
    assert calls[0]["theta_at_centers"] == 1 and calls[0]["theta_shape"] == cent.shape and calls[0]["axis"] == 1
    want = oracle.vinterp_conservative(q, oracle.stencil2("interp", cent, 1, 1, 1, "extend"), bins, 1)
    np.testing.assert_array_equal(got.values, want)
    assert got.dims == ("t", "y", "x", "tc")


def test_other_inputs_keep_the_old_routes(mocked):
    from xgcm_b200.transform import conservative_interpolation, interp_1d_conservative

    calls, device_calls = mocked
    ds, grid, q, bounds, cent = _dataset()
    bins = np.linspace(0, 12, 9)
    # device-resident (here: torch) fields, and mixed host / device inputs
    tq = xg.DataArray(torch.from_numpy(q), dims=ds["q"].dims)
    tsig = xg.DataArray(torch.from_numpy(bounds), dims=ds["sig"].dims, name="sig")
    grid.transform(tq, "Z", bins, target_data=tsig, method="conservative")
    grid.transform(ds["q"], "Z", bins, target_data=tsig, method="conservative")
    grid.transform(tq, "Z", bins, target_data=ds["sig"], method="conservative")
    # an integer field
    iq = xg.DataArray((q * 10).astype(np.int64), dims=ds["q"].dims)
    grid.transform(iq, "Z", bins, target_data=ds["sig"], method="conservative")
    # centred theta, fields on the device: grid.interp then the device op
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        tc = xg.DataArray(torch.from_numpy(cent), dims=ds["tc"].dims)
        grid.transform(tq, "Z", bins, target_data=tc, method="conservative")
    assert not calls and len(device_calls) == 5
    # a target on the device
    conservative_interpolation(ds["q"], ds["sig"], xg.DataArray(torch.from_numpy(bins), dims=("sig",)), "z", "zo", "sig",
                               grid=grid)
    interp_1d_conservative(torch.from_numpy(q[0, :, 0, 0]), torch.from_numpy(bounds[0, :, 0, 0]), torch.from_numpy(bins))
    assert not calls and len(device_calls) == 7


def test_centred_theta_with_a_left_default_shift_keeps_todays_sequence(mocked):
    """center -> left is the default shift: grid.interp gives left values, not bounds, and the remap rejects them
    exactly as before (no fused call)."""
    calls, device_calls = mocked
    ds, grid, _, _, _ = _dataset(left=True)
    assert grid.axes["Z"].default_shifts["center"] == "left"
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        with pytest.raises(ValueError, match="cell-bounds dimension 'zo'"):
            grid.transform(ds["q"], "Z", np.linspace(0, 12, 9), target_data=ds["tc"], method="conservative")
    assert len([w for w in rec if "cell bounds" in str(w.message)]) == 1
    assert not calls and not device_calls


def test_interp_1d_conservative_takes_the_twin_for_numpy(mocked):
    from xgcm_b200.transform import interp_1d_conservative

    calls, _ = mocked
    rng = np.random.default_rng(4)
    phi = rng.random((4, 6))
    theta = np.cumsum(rng.random((4, 7)), axis=-1)
    bins = np.linspace(0, 4, 5)
    got = interp_1d_conservative(phi, theta, bins)
    assert isinstance(got, np.ndarray) and calls[-1]["axis"] == 1
    np.testing.assert_array_equal(got, oracle.vinterp_conservative(phi, theta, bins, -1))
    with pytest.raises(AssertionError):
        interp_1d_conservative(phi, theta[:, :-1], bins)
    with pytest.raises(ValueError, match="not monotonic"):
        interp_1d_conservative(phi, theta, np.array([0.0, 2.0, 1.0]))
    assert interp_1d_conservative(phi, theta, np.array([1.0])).shape == (4, 0)
