"""The plane-strided stencil kernel (`xg_stencil2(plane)`, k_stencil_plane) against the oracle, bit for bit: inner
widths that leave partial 128-byte lines and partial warps, every boundary rule, shifts that change the length,
axes shorter and longer than one warp's chunk of rows, halo planes, and fused metrics on the layouts the
TMA-staged kernels leave to it."""

import itertools

import numpy as np
import pytest
import torch

from oracle import stencil as oracle

pytestmark = pytest.mark.gpu

SHIFTS = [(1, 0), (0, 1), (1, 1), (0, 0)]
BCS = [("periodic", 0.0), ("fill", 0.0), ("fill", 1.5), ("extend", 0.0), ("extrapolate", 0.0)]
# inner widths: partial line, partial line of a second, a row ending 4 elements into a warp's 4th line, whole warps
INNER = {np.float32: [4, 36, 904, 3600, 37], np.float64: [2, 18, 452, 1800, 19]}


def _dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _run(a, axis, op, lo, hi, bc, fill, pre=None, post=None, halo_lo=None, halo_hi=None):
    from xgcm_b200 import _capi, ops

    out = ops.stencil2(_dev(a), axis, op, lo, hi, bc, fill, pre=_dev(pre), post=_dev(post), halo_lo=_dev(halo_lo),
                       halo_hi=_dev(halo_hi))
    torch.cuda.synchronize()
    return out.cpu().numpy(), _capi.last_launch()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", [1, 5, 33, 300])
def test_plane_kernel_every_rule(dtype, n):
    rng = np.random.default_rng(n)
    for inner in INNER[dtype]:
        a = rng.random((3, n, inner)).astype(dtype)
        for op, (lo, hi), (bc, fill) in itertools.product(("diff", "interp", "min"), SHIFTS, BCS):
            if n + lo + hi - 1 <= 0 or (bc == "extrapolate" and n < 2):
                continue
            want = oracle.stencil2(op, a, 1, lo, hi, bc if (lo or hi) else None, fill)
            got, label = _run(a, 1, op, lo, hi, bc if (lo or hi) else None, fill)
            assert label == "xg_stencil2(plane)", label
            np.testing.assert_array_equal(got, want, err_msg=f"{op} {lo}{hi} {bc} inner={inner}")


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_plane_kernel_z_of_a_field(dtype):
    """The outermost axis: a single plane of (Y, X) lines marched along Z, chunks spanning many line groups."""
    a = np.random.default_rng(7).random((75, 24, 904 if dtype == np.float32 else 452)).astype(dtype)
    for op, (bc, fill) in itertools.product(("diff", "interp"), BCS[:4]):
        got, label = _run(a, 0, op, 1, 0, bc, fill)
        assert label == "xg_stencil2(plane)", label
        np.testing.assert_array_equal(got, oracle.stencil2(op, a, 0, 1, 0, bc, fill))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("lo,hi", [(1, 0), (0, 1), (1, 1)])
def test_plane_kernel_halo_planes(dtype, lo, hi):
    rng = np.random.default_rng(11)
    for inner in INNER[dtype]:
        a = rng.random((4, 70, inner)).astype(dtype)
        hl = rng.random((4, 1, inner)).astype(dtype) if lo else None
        hh = rng.random((4, 1, inner)).astype(dtype) if hi else None
        padded = np.concatenate([p for p in (hl, a, hh) if p is not None], axis=1)
        for op in ("diff", "interp"):
            want = oracle.stencil2(op, padded, 1, 0, 0, None)
            got, label = _run(a, 1, op, lo, hi, "fill", 0.0, halo_lo=hl, halo_hi=hh)
            assert label == "xg_stencil2(plane)", label
            np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_plane_kernel_fused_metrics(dtype):
    """pre / post metrics on an odd inner width (no 16-byte vectors: not a TMA-staged layout)."""
    rng = np.random.default_rng(5)
    inner = INNER[dtype][-1]
    a = rng.random((3, 40, inner)).astype(dtype)
    pre = (0.5 + rng.random((1, 40, inner))).astype(dtype)
    for lo, hi in ((1, 0), (0, 1)):
        post = (0.5 + rng.random((1, 40, inner))).astype(dtype)
        for bc in ("periodic", "extend"):
            want = oracle.stencil2("diff", a, 1, lo, hi, bc, 0.0, pre, post)
            got, label = _run(a, 1, "diff", lo, hi, bc, 0.0, pre=pre, post=post)
            assert label == "xg_stencil2(plane)", label
            np.testing.assert_array_equal(got, want)
