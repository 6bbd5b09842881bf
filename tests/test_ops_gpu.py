"""Parity of cumscan / wreduce / vinterp / pad / binary / host-streamed stencil vs the oracle."""

import itertools

import numpy as np
import pytest
import torch

from oracle import stencil as oracle

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
BCS = [("periodic", 0.0), ("fill", 0.0), ("fill", 1.5), ("fill", float("nan")), ("extend", 0.0)]


def _field(shape, dtype, seed=0, nan_frac=0.0):
    rng = np.random.default_rng(seed)
    a = rng.random(shape).astype(dtype)
    if nan_frac:
        a[rng.random(shape) < nan_frac] = np.nan
    return a


def _t(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ----------------------------------------------------------------------------- pad
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape", [(5,), (3, 8), (4, 6, 12), (2, 3, 4, 5), (7, 1, 3)])
def test_pad_matches_np_pad(dtype, shape):
    """xgcm/test/test_padding.py:20-165: pad == DataArray.pad(wrap | constant | edge)."""
    from xgcm_b200 import ops

    a = _field(shape, dtype, seed=11)
    for axis in range(len(shape)):
        for (lo, hi), (bc, fill) in itertools.product([(1, 0), (0, 1), (1, 1), (2, 3), (0, 0)], BCS):
            if bc == "periodic" and False:
                continue
            want = oracle.pad_axis(a, axis, lo, hi, bc, fill)
            got = ops.pad(_t(a), axis, lo, hi, bc, fill).cpu().numpy()
            np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_pad_innermost_flat_stream_kernel(dtype):
    """xg_pad(rows): the output of an innermost-dim pad is written as one flat stream of aligned vectors that may
    straddle rows — every width / boundary / row length combination against np.pad."""
    from xgcm_b200 import _capi, ops

    for shape in [(7, 1027), (3, 5, 130), (1, 9), (2, 3, 4, 33), (4099,)]:
        a = _field(shape, dtype, seed=13)
        for (lo, hi), (bc, fill) in itertools.product([(1, 0), (0, 1), (1, 1), (3, 2), (0, 0), (5, 7)], BCS):
            if bc == "periodic" and max(lo, hi) > shape[-1]:
                continue
            want = oracle.pad_axis(a, len(shape) - 1, lo, hi, bc, fill)
            got = ops.pad(_t(a), len(shape) - 1, lo, hi, bc, fill).cpu().numpy()
            if shape[-1] + lo + hi >= 8:
                assert _capi.last_launch() == "xg_pad(rows)"
            np.testing.assert_array_equal(got, want)


# ----------------------------------------------------------------------------- binary
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_binary_broadcast(dtype):
    from xgcm_b200 import ops

    rng = np.random.default_rng(12)
    a = (rng.random((3, 4, 6, 8)) + 0.5).astype(dtype)
    for bshape in [(3, 4, 6, 8), (1, 1, 6, 8), (1, 4, 1, 1), (3, 1, 1, 1), (1, 1, 1, 8), (1, 4, 1, 8), (1, 1, 1, 1), (6, 8), (8,)]:
        b = (rng.random(bshape) + 0.5).astype(dtype)
        for name, fn in (("mul", np.multiply), ("div", np.true_divide), ("add", np.add), ("sub", np.subtract)):
            got = ops.binary(name, _t(a), _t(b)).cpu().numpy()
            np.testing.assert_array_equal(got, fn(a, b))
    # a broadcast against a bigger b
    small = (rng.random((6, 1)) + 0.5).astype(dtype)
    got = ops.binary("div", _t(small), _t(a)).cpu().numpy()
    np.testing.assert_array_equal(got, small / a)
    odd = (rng.random((5, 7)) + 0.5).astype(dtype)
    got = ops.binary("sub", _t(odd), _t(odd[:, :1].copy())).cpu().numpy()
    np.testing.assert_array_equal(got, odd - odd[:, :1])


# ----------------------------------------------------------------------------- cumscan
def _cumscan_cases():
    seen = set()
    for table, rev in ((oracle.CUMSUM_TABLE_FWD, False), (oracle.CUMSUM_TABLE_REV, True)):
        for trim, (plo, phi) in table.values():
            key = (rev, trim, plo, phi)
            if key not in seen:
                seen.add(key)
                yield key


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape", [(1,), (2,), (33,), (100,), (5, 40), (6, 20, 36), (3, 4, 10, 16), (40, 3), (70, 1, 5), (2, 3600), (33, 520), (3, 2, 1032)])
def test_cumscan_bit_exact(dtype, shape):
    """Sequential order => bit-equal to np.cumsum for every shift of grid.py:1326-1383."""
    from xgcm_b200 import ops

    a = _field(shape, dtype, seed=13)
    for axis in range(len(shape)):
        for (rev, trim, plo, phi), (bc, fill) in itertools.product(_cumscan_cases(), BCS):
            kept = shape[axis] - (0 if trim == "none" else 1)
            if kept + plo + phi <= 0 or (kept == 0 and bc != "fill"):
                continue
            want = oracle.cumscan(a, axis, rev, trim, plo, phi, bc if (plo or phi) else None, fill)
            got = ops.cumscan(_t(a), axis, rev, trim, plo, phi, bc, fill).cpu().numpy()
            assert got.shape == want.shape
            np.testing.assert_array_equal(got, want, err_msg=f"axis={axis} rev={rev} trim={trim} pad=({plo},{phi}) bc={bc}")


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_cumscan_metrics_and_nan(dtype):
    from xgcm_b200 import ops

    shape = (6, 20, 36)
    a = _field(shape, dtype, seed=14, nan_frac=0.03)
    rng = np.random.default_rng(15)
    for axis in range(3):
        pre = (1 + rng.random([shape[d] if d >= 1 else 1 for d in range(3)])).astype(dtype)
        for (rev, trim, plo, phi) in _cumscan_cases():
            oshape = list(shape)
            oshape[axis] = shape[axis] - (0 if trim == "none" else 1) + plo + phi
            post = (1 + rng.random([oshape[d] if d != 1 else 1 for d in range(3)])).astype(dtype)
            for skipna in (True, False):
                want = oracle.cumscan(a, axis, rev, trim, plo, phi, "extend" if (plo or phi) else None, 0.0, pre, post, skipna)
                got = ops.cumscan(_t(a), axis, rev, trim, plo, phi, "extend", 0.0, _t(pre), _t(post), skipna).cpu().numpy()
                np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_cumscan_wide_rows_metrics(dtype):
    """Innermost-axis scan through the 16-byte tile kernel, with metrics, NaNs, reverse, ragged rows."""
    from xgcm_b200 import ops

    shape = (37, 776)
    a = _field(shape, dtype, seed=31, nan_frac=0.02)
    rng = np.random.default_rng(32)
    pre = (1 + rng.random((1, shape[1]))).astype(dtype)
    for (rev, trim, plo, phi) in _cumscan_cases():
        n_out = shape[1] - (0 if trim == "none" else 1) + plo + phi
        post = (1 + rng.random((shape[0], n_out))).astype(dtype)
        for bc in ("fill", "extend", "periodic"):
            want = oracle.cumscan(a, 1, rev, trim, plo, phi, bc if (plo or phi) else None, 0.5, pre, post, True)
            got = ops.cumscan(_t(a), 1, rev, trim, plo, phi, bc, 0.5, _t(pre), _t(post), True).cpu().numpy()
            np.testing.assert_array_equal(got, want)


def test_cumscan_known_answers():
    """xgcm/test/test_grid.py:549-552: cumsum(arange(1,15)) center->outer fill -> [0,1,3,6,...]."""
    from xgcm_b200 import ops

    a = np.arange(1, 15, dtype=np.float64)
    got = ops.cumscan(_t(a), 0, False, "none", 1, 0, "fill", 0.0).cpu().numpy()
    np.testing.assert_array_equal(got, np.concatenate([[0.0], np.cumsum(a)]))


# ----------------------------------------------------------------------------- wreduce
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_wreduce_strided_exact(dtype):
    """Along a non-contiguous axis numpy sums sequentially: bit-exact."""
    from xgcm_b200 import ops

    shape = (30, 12, 40)
    a = _field(shape, dtype, seed=16, nan_frac=0.02)
    rng = np.random.default_rng(17)
    for axis in (0, 1):
        for wshape in (None, shape, tuple(s if d == axis else 1 for d, s in enumerate(shape)), (1,) + shape[1:]):
            w = None if wshape is None else (0.5 + rng.random(wshape)).astype(dtype)
            for skipna in (True, False):
                want = oracle.wreduce(a, w, axis, "sum", skipna)
                got = ops.wreduce(_t(a), axis, _t(w), "sum", skipna).cpu().numpy()
                np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_wreduce_rows_and_mean(dtype):
    """Row reductions (fp64 accumulation, one rounding) against the exact sum; strided means bit-exact."""
    from test_kernel_instances_gpu import _fsum_bound_check
    from xgcm_b200 import ops

    shape = (7, 9, 1000)
    a = _field(shape, dtype, seed=18, nan_frac=0.02)
    w = (0.5 + np.random.default_rng(19).random((1, 1, 1000))).astype(dtype)
    got = ops.wreduce(_t(a), 2, _t(w), "sum", True).cpu().numpy()
    _fsum_bound_check(got, a, w, 2, "sum", True, "rows sum")
    for axis in range(3):
        for wt in (None, (0.5 + np.random.default_rng(20).random(shape)).astype(dtype)):
            got = ops.wreduce(_t(a), axis, _t(wt), "mean", True).cpu().numpy()
            if axis == 2:
                _fsum_bound_check(got, a, wt, 2, "mean", True, "rows mean")
            else:
                np.testing.assert_array_equal(got, oracle.wreduce(a, wt, axis, "mean", True))
    allnan = np.full((4, 5), np.nan, dtype=dtype)
    got = ops.wreduce(_t(allnan), 0, None, "mean", True).cpu().numpy()
    assert np.isnan(got).all()  # xarray weighted mean: 0/0 -> NaN


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_wreduce_rows_vector_and_scalar_loads(dtype):
    """The innermost-axis reduction reads 16-byte vectors when the rows allow it, else single elements."""
    from test_kernel_instances_gpu import _fsum_bound_check
    from xgcm_b200 import _capi, ops

    for n, side in ((1000, "vec"), (999, "scalar")):
        a = _field((7, 9, n), dtype, seed=21, nan_frac=0.02)
        w = (0.5 + np.random.default_rng(22).random((1, 1, n))).astype(dtype)
        for mode in ("sum", "mean"):
            got = ops.wreduce(_t(a), 2, _t(w), mode, True).cpu().numpy()
            assert _capi.last_launch() == f"xg_wreduce(rows, {side})"
            _fsum_bound_check(got, a, w, 2, mode, True, f"n={n} {mode}")


# ----------------------------------------------------------------------------- strided scan / reduce at the 16-byte switch
# k_scan_strided and k_reduce_strided read 16-byte column vectors only from outer x inner / VEC >= XG_SMS x 64 = 8448
# vector columns on (xg_cumscan.cu scan_launch, xg_wreduce.cu reduce_launch); below that, one element per thread.
# Shapes exactly at the switch and just below it, along Z and along Y.
VEC_COLUMNS = 132 * 64
STRIDED_SWITCH = {
    np.float32: [((40, 48, 704), 0, "vec"), ((40, 48, 700), 0, "scalar"), ((22, 30, 1536), 1, "vec"),
                 ((22, 30, 1524), 1, "scalar")],
    np.float64: [((40, 24, 704), 0, "vec"), ((40, 24, 700), 0, "scalar"), ((22, 30, 768), 1, "vec"),
                 ((22, 30, 762), 1, "scalar")],
}
SWITCH_CASES = [(dt, shape, axis, side) for dt, cases in STRIDED_SWITCH.items() for shape, axis, side in cases]


def _vector_columns(shape, axis, dtype):
    vec = 16 // np.dtype(dtype).itemsize
    return int(np.prod(shape[:axis])) * (int(np.prod(shape[axis + 1:])) // vec)


def _switch_field(shape, dtype, seed):
    """Uniform values with 3 % NaN and a few +-inf and -0."""
    rng = np.random.default_rng(seed)
    a = (rng.random(shape) - 0.25).astype(dtype)
    r = rng.random(shape)
    a[r < 0.03] = np.nan
    a[(r >= 0.03) & (r < 0.031)] = np.inf
    a[(r >= 0.031) & (r < 0.032)] = -np.inf
    a[(r >= 0.032) & (r < 0.04)] = -0.0
    return a


@pytest.mark.parametrize("dtype,shape,axis,side", SWITCH_CASES)
def test_cumscan_strided_at_vector_switch(dtype, shape, axis, side):
    """Bit-exact cumsum either side of the switch: every trim / pad entry and boundary, reverse, skipna both ways,
    pre-metrics shared along the axis or full, post-metrics per level along the axis or shared."""
    from xgcm_b200 import _capi, ops

    assert (_vector_columns(shape, axis, dtype) >= VEC_COLUMNS) == (side == "vec")
    a = _switch_field(shape, dtype, 40)
    rng = np.random.default_rng(41)
    pres = [None, (1.0 + rng.random((1,) + shape[1:])).astype(dtype), (0.5 + rng.random(shape)).astype(dtype)]
    k = 0
    for (rev, trim, plo, phi), (bc, fill) in itertools.product(_cumscan_cases(), BCS):
        oshape = list(shape)
        oshape[axis] = shape[axis] - (0 if trim == "none" else 1) + plo + phi
        level = [n if d == axis else 1 for d, n in enumerate(oshape)]
        posts = [None, (1.0 + rng.random(level)).astype(dtype), (1.0 + rng.random([1] + oshape[1:])).astype(dtype)]
        pre, post, skipna = pres[k % 3], posts[(k // 3) % 3], k % 2 == 0
        k += 1
        with np.errstate(invalid="ignore"):
            want = oracle.cumscan(a, axis, rev, trim, plo, phi, bc if (plo or phi) else None, fill, pre, post, skipna)
        got = ops.cumscan(_t(a), axis, rev, trim, plo, phi, bc, fill, _t(pre), _t(post), skipna).cpu().numpy()
        assert _capi.last_launch() == f"xg_cumscan(strided, {side})"
        np.testing.assert_array_equal(got, want, err_msg=f"rev={rev} trim={trim} pad=({plo},{phi}) bc={bc} skipna={skipna}")


@pytest.mark.parametrize("dtype,shape,axis,side", SWITCH_CASES)
def test_wreduce_strided_at_vector_switch(dtype, shape, axis, side):
    """Bit-exact weighted sum and mean either side of the switch: no, full, (1, Y, X) and per-level weights,
    skipna both ways."""
    from xgcm_b200 import _capi, ops

    assert (_vector_columns(shape, axis, dtype) >= VEC_COLUMNS) == (side == "vec")
    a = _switch_field(shape, dtype, 42)
    rng = np.random.default_rng(43)
    level = [n if d == axis else 1 for d, n in enumerate(shape)]
    for wshape, mode, skipna in itertools.product((None, shape, (1,) + shape[1:], level), ("sum", "mean"), (True, False)):
        w = None if wshape is None else (0.5 + rng.random(wshape)).astype(dtype)
        with np.errstate(invalid="ignore"):
            want = oracle.wreduce(a, w, axis, mode, skipna)
        got = ops.wreduce(_t(a), axis, _t(w), mode, skipna).cpu().numpy()
        assert _capi.last_launch() == f"xg_wreduce(strided, {side})"
        np.testing.assert_array_equal(got, want, err_msg=f"w={wshape} {mode} skipna={skipna}")


# ----------------------------------------------------------------------------- vinterp
def _theta_field(shape, axis, dtype, rng, decreasing_frac=0.3, nan_frac=0.0):
    n = shape[axis]
    inc = np.cumsum(0.1 + rng.random(shape), axis=axis).astype(dtype)
    th = inc.copy()
    if decreasing_frac:
        flip_shape = [s if d != axis else 1 for d, s in enumerate(shape)]
        flip = rng.random(flip_shape) < decreasing_frac
        th = np.where(flip, np.flip(inc, axis=axis), inc).astype(dtype)
    if nan_frac:
        th[rng.random(shape) < nan_frac] = np.nan
    return th


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape,axis", [((20,), 0), ((20, 50), 0), ((7, 20), 1), ((20, 6, 37), 0), ((3, 25, 40), 1), ((2, 75, 8, 33), 1), ((1, 5), 0), ((4, 100), 0)])
def test_vinterp_linear_matches_reference_port(dtype, shape, axis):
    from xgcm_b200 import ops

    rng = np.random.default_rng(21)
    phi = _field(shape, dtype, seed=22, nan_frac=0.02)
    n = shape[axis]
    for kind in ("shared", "field", "field_nan"):
        if kind == "shared":
            th1 = np.cumsum(0.1 + rng.random(n)).astype(dtype)
            bshape = [1] * len(shape)
            bshape[axis] = n
            theta = th1.reshape(bshape)
        else:
            theta = _theta_field(shape, axis, dtype, rng, nan_frac=0.05 if kind == "field_nan" else 0.0)
        lo, hi = np.nanmin(theta), np.nanmax(theta)
        for m in (1, 5, 33, 100):
            target = np.linspace(lo - 0.3, hi + 0.3, m).astype(dtype)
            if m >= 5:
                target[2] = np.nan
                target[3] = theta.reshape(-1)[0] if not np.isnan(theta.reshape(-1)[0]) else target[3]
            for mask, bypass in ((True, False), (False, False), (True, True)):
                want = oracle.vinterp_linear(phi, np.broadcast_to(theta, shape), target, axis, mask, bypass)
                got = ops.vinterp_linear(_t(phi), _t(theta), _t(target), axis, mask, bypass).cpu().numpy()
                assert got.shape == want.shape and got.dtype == want.dtype
                np.testing.assert_array_equal(got, want, err_msg=f"{kind} m={m} mask={mask} bypass={bypass}")
            # reversed target order (test_transform.py cases with decreasing targets)
            want = oracle.vinterp_linear(phi, np.broadcast_to(theta, shape), target[::-1].copy(), axis, True, False)
            got = ops.vinterp_linear(_t(phi), _t(theta), _t(target[::-1].copy()), axis, True, False).cpu().numpy()
            np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_vinterp_log(dtype):
    """method="log" (transform.py:82-84: np.log of theta and targets in the field dtype).  float32: the device
    evaluates numpy's own float32 log (csrc/xg_vinterp.cuh, pinned by test_oracle_golden.test_log32_port_is_numpys),
    so on x86 hosts where np.log takes numpy's SIMD path the result is BIT-IDENTICAL to the reference port;
    elsewhere (libm logf under numpy) it stays within the north-star 1e-6 only up to the amplification of a
    1-ulp log difference by 1 / (log spacing), checked at 5e-5.  float64: CUDA log vs numpy's, 1e-12."""
    from test_oracle_golden import _numpy_simd_log
    from xgcm_b200 import ops

    rng = np.random.default_rng(23)
    shape = (30, 5, 40)
    phi = _field(shape, dtype, seed=24)
    for theta in (np.cumsum(1.0 + rng.random(shape), axis=0).astype(dtype),            # a theta field
                  np.cumsum(1.0 + rng.random(30)).astype(dtype).reshape(30, 1, 1)):    # the shared coordinate
        target = np.linspace(0.5, float(theta.max()) + 1, 17).astype(dtype)
        want = oracle.vinterp_linear(phi, np.broadcast_to(theta, shape), target, 0, True, False, True)
        got = ops.vinterp_linear(_t(phi), _t(theta), _t(target), 0, True, False, True).cpu().numpy()
        if dtype == np.float32 and _numpy_simd_log():
            np.testing.assert_array_equal(got, want)
        else:
            tol = 5e-5 if dtype == np.float32 else 1e-12
            np.testing.assert_allclose(got, want, rtol=tol, atol=tol, equal_nan=True)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_vinterp_shared_slope_division_is_correctly_rounded(dtype):
    """The shared-theta kernels form slope = dy/dx from a precomputed reciprocal plus FMA corrections;
    they must round exactly like the reference's fp64 division: many columns, wide dynamic range,
    zeros, NaNs, non power-of-two spacings.  An aligned phi takes the TMA kernel; a phi one element
    past a 16-byte boundary (a time slice of a larger field) the fallback k_vinterp_shared."""
    from xgcm_b200 import _capi, ops

    rng = np.random.default_rng(77)
    ncol, n = 200_000, 5
    phi = (rng.standard_normal((n, ncol)) * 10.0 ** rng.integers(-12, 12, size=(n, ncol))).astype(dtype)
    phi[:, :50] = 0.0
    phi[2, 50:80] = np.nan
    phi[1, 100:200] = phi[2, 100:200]  # dy == 0
    theta = np.array([0.1, 0.7, 1.9, 3.0000001, 7.3], dtype=dtype).reshape(n, 1)
    target = np.array([0.05, 0.1, 0.33, 0.7000001, 1.0, 2.5, 3.0, 3.5, 7.0, 7.3, 9.0], dtype=dtype)
    want = oracle.vinterp_linear(phi, np.broadcast_to(theta, phi.shape), target, 0, True)
    shifted = torch.empty(phi.size + 1, dtype=_t(phi).dtype, device=DEV)[1:].view(phi.shape)
    shifted.copy_(torch.from_numpy(phi))
    for field, label in ((_t(phi), "xg_vinterp_linear(shared, tma)"), (shifted, "xg_vinterp_linear(shared)")):
        got = ops.vinterp_linear(field, _t(theta), _t(target), 0, True).cpu().numpy()
        assert _capi.last_launch() == label
        np.testing.assert_array_equal(got, want)


def test_vinterp_mixed_dtypes_promote_like_numba():
    """transform.py:15-22: float32 loop only if phi, theta, target are ALL float32."""
    from xgcm_b200 import ops

    phi = _field((10, 6), np.float32, seed=25)
    theta = np.arange(10, dtype=np.float64).reshape(10, 1)
    target = np.linspace(0, 9, 4)
    got = ops.vinterp_linear(_t(phi), _t(theta), _t(target), 0, True).cpu().numpy()
    want = oracle.vinterp_linear(phi, np.broadcast_to(theta, phi.shape), target, 0, True)
    assert got.dtype == np.float64 == want.dtype
    np.testing.assert_array_equal(got, want)


# ----------------------------------------------------------------------------- synthetic fields
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_fill_uniform_host_equals_device(dtype):
    from xgcm_b200 import ops

    tdt = torch.float32 if dtype == np.float32 else torch.float64
    d = ops.fill_uniform(torch.empty(100_003, dtype=tdt, device=DEV), seed=0xC0FFEE, offset=12345).cpu().numpy()
    h = ops.fill_uniform_host(np.empty(100_003, dtype=dtype), seed=0xC0FFEE, offset=12345)
    np.testing.assert_array_equal(d, h)
    assert 0.0 <= d.min() and d.max() < 1.0 and abs(d.mean() - 0.5) < 0.01
    # any sub-block can be generated independently
    sub = ops.fill_uniform_host(np.empty(100, dtype=dtype), seed=0xC0FFEE, offset=12345 + 500)
    np.testing.assert_array_equal(sub, h[500:600])


# ----------------------------------------------------------------------------- host-streamed stencil
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_stencil2_host_streams_slabs(dtype):
    from xgcm_b200 import ops

    shape = (9, 40, 64)
    a = _field(shape, dtype, seed=26)
    rng = np.random.default_rng(27)
    dx = (1 + rng.random((1, 40, 64))).astype(dtype)
    dz = (1 + rng.random((9, 1, 1))).astype(dtype)
    for axis, (lo, hi), (bc, fill), op in itertools.product(range(3), [(1, 0), (0, 1), (1, 1), (0, 0)], BCS, ("diff", "interp")):
        if shape[axis] + lo + hi - 1 <= 0:
            continue
        want = oracle.stencil2(op, a, axis, lo, hi, bc if (lo or hi) else None, fill)
        got = ops.stencil2_host(a, axis, op, lo, hi, bc, fill)
        np.testing.assert_array_equal(got, want)
    for axis in range(3):
        n_out = shape[axis]
        post = dx if axis != 0 else dz
        want = oracle.stencil2("diff", a, axis, 1, 0, "fill", 0.0, dz, post)
        got = ops.stencil2_host(a, axis, "diff", 1, 0, "fill", 0.0, pre=dz, post=post)
        np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("n0", [3, 4, 5, 9, 10, 13])
def test_stencil2_host_extrapolate_edge_slabs(n0):
    """ADVICE r1: with the opt-in `extrapolate` boundary along the slabbed (outermost) axis the edge slab must
    hold two source planes; host result == device result for slab heights that used to leave a one-row tail."""
    from xgcm_b200 import ops

    a = _field((n0, 6, 40), np.float32, seed=28)
    for (lo, hi) in [(1, 0), (0, 1), (1, 1)]:
        for op in ("diff", "interp"):
            got = ops.stencil2_host(a, 0, op, lo, hi, "extrapolate")
            want = ops.stencil2(_t(a), 0, op, lo, hi, "extrapolate").cpu().numpy()
            np.testing.assert_array_equal(got, want)


def test_stencil2_host_large_pinned():
    """Many slabs, page-locked buffers: identical to the device path."""
    from xgcm_b200 import ops

    shape = (64, 256, 512)  # 32 MiB fp32 -> 4+ slabs
    x = ops.pinned_empty(shape, np.float32)
    ops.fill_uniform_host(x.reshape(-1), seed=7)
    for axis in range(3):
        got = ops.stencil2_host(x, axis, "interp", 1, 0, "periodic")
        want = ops.stencil2(torch.from_numpy(x).to(DEV), axis, "interp", 1, 0, "periodic").cpu().numpy()
        np.testing.assert_array_equal(got, want)
