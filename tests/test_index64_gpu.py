"""64-bit index paths on the device: one fp32 field per gate an 80 GB device can flip (tests/test_index64.py restates
each gate and checks these shapes cross it), and the generic (strided) operand path at small sizes.

Every large case
* compares every output cell, bit for bit, with a reference that never takes the path under test: the same op on
  contiguous pieces below the gate, or plain torch arithmetic with one IEEE operation per call in the kernel's order;
* checks the cells where a 32-bit error would show (flat offsets 2^31 - 1, 2^31, 2^32 - 1 / 2^32, the last cell, and
  for the transposed metric the vectors that straddle two rows) against the CPU oracle;
* writes into an output with a sentinel guard band where the op takes ``out=``, and asserts, with torch.profiler,
  that the intended kernel ran.

Each case states the peak device memory it needs (every tensor it holds at once, the reference's block temporaries
included) and skips, naming both numbers, when less is free (the machines are shared); after the case the caching
allocator's peak is checked against the stated need.  Tensors are released between cases.  The free memory, the
measured peak and the time of each case are printed; pytest shows them for passing tests with ``-rP``:

    python -m pytest tests/test_index64_gpu.py -m gpu -v -rP
"""

import gc
import time

import numpy as np
import pytest
import torch

from oracle import fold as fold_oracle
from oracle import stencil as oracle
from test_index64 import N30, N31, SHAPE
from test_kernel_instances_gpu import _key

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GB = 10**9
SENTINEL = 1.2345e30
PIECE = 1 << 28  # cells per piece of a reference: far below every gate


_NEED = {}  # the stated need of the running case, in GB


@pytest.fixture(autouse=True)
def _release():
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    _NEED.clear()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_reserved()
    print(f"  case time {time.perf_counter() - t0:.1f} s; peak device memory {peak / GB:.2f} GB")
    gc.collect()
    torch.cuda.empty_cache()
    if "gb" in _NEED:
        assert peak <= _NEED["gb"] * GB, f"the case reserved {peak / GB:.2f} GB, more than the {_NEED['gb']} GB it states"


def _need(gb):
    free, total = torch.cuda.mem_get_info()
    print(f"\n  device memory: {free / GB:.1f} GB free of {total / GB:.1f} GB; this case needs {gb} GB")
    if free < gb * GB:
        pytest.skip(f"needs {gb} GB of device memory, {free / GB:.1f} GB free")
    _NEED["gb"] = gb


def _ops():
    from xgcm_b200 import ops

    return ops


def _field(shape, seed, lo=0.0):
    x = torch.empty(shape, dtype=torch.float32, device=DEV)
    _ops().fill_uniform(x, seed)
    return x.add_(lo) if lo else x


def _guarded(shape):
    """An output view with a 16-byte SENTINEL band on each side: (allocation, view)."""
    n = int(np.prod(shape, dtype=np.int64))
    base = torch.full((4 + n + 4,), SENTINEL, dtype=torch.float32, device=DEV)
    return base, base[4:4 + n].view(shape)


def _check_guard(base, ctx):
    assert bool((base[:4] == SENTINEL).all()), f"{ctx}: a store landed before the output"
    assert bool((base[-4:] == SENTINEL).all()), f"{ctx}: a store landed past the output"


class _Kernels:
    """Names (test_kernel_instances_gpu._key form) of the kernels launched inside the block."""

    def __enter__(self):
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.synchronize()
        self.prof = profile(activities=[ProfilerActivity.CUDA])
        self.prof.__enter__()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.prof.__exit__(*exc)
        self.names = {_key(e.name) for e in self.prof.events() if e.name.startswith("void ")}
        return False

    def ran(self, prefix):
        assert any(n.startswith(prefix) for n in self.names), f"{prefix} did not run: {sorted(self.names)}"


def _bits(got, want, ctx):
    assert tuple(got.shape) == tuple(want.shape), f"{ctx}: shape {tuple(got.shape)} != {tuple(want.shape)}"
    ne = got.contiguous().view(torch.int32) != want.contiguous().view(torch.int32)
    if bool(ne.any()):
        i = tuple(ne.nonzero()[0].tolist())
        raise AssertionError(f"{ctx}: first differing cell {i} of the block: {float(got[i])!r} != {float(want[i])!r}")


def _blocks(out, dim, step, want, ctx):
    """out.narrow(dim, s, l) against want(s, l), block by block."""
    n = out.shape[dim]
    for s in range(0, n, step):
        l = min(step, n - s)
        _bits(out.narrow(dim, s, l), want(s, l), f"{ctx} [{s}:{s + l}] of dim {dim}")


def _cell(shape, flat):
    return tuple(int(v) for v in np.unravel_index(flat, shape))


def _far_cells(shape):
    """Cells at the flat offsets where a 32-bit error shows, as far as the array reaches."""
    n = int(np.prod(shape, dtype=np.int64))
    return [_cell(shape, f) for f in sorted({N31 - 1, N31, 2 * N31 - 1, 2 * N31, n - 1}) if f < n]


def _np(t):
    return t.cpu().numpy()


# ---------------------------------------------------------------------------------------------- 1a / 1b
def _stencil0_want(op, lo, A, f=1.5):
    """stencil2 along an axis of extent 1 with fill f: OP(P[0], P[1]) with P = (f, A) or (A, f)."""
    if op == "diff":
        return A - f if lo else f - A
    return (A + f) * 0.5  # (a + b) * 0.5, a + b commutes


@pytest.mark.parametrize("layout", ["broadcast", "transposed"])
def test_stencil2_generic_operands_past_2_31(layout):
    """1a: broadcast (1, 32768, 1) / (1, 1, 65539) metrics have two inner index groups past 2^31 (64-bit group
    offsets) and k_stencil_plane<float, 4> runs.  1b: the transposed (65539, 32768) pre-metric spans 2^31 elements
    with vectors straddling rows; it must take k_stencil_plane<float, 1>."""
    ops = _ops()
    shape = SHAPE["stencil2_operand_groups"]
    _need(20 if layout == "broadcast" else 29)  # x, out 8.6 GB each (+ w 8.6 GB); three 0.54 GB block temporaries
    x = _field(shape, 11)
    if layout == "broadcast":
        pre = _field((1, shape[1], 1), 12, 0.5)
    else:
        w = _field((shape[2], shape[1]), 12, 0.5)
        pre = w.T[None]
        assert pre.stride()[1:] == (1, shape[1])
    post = _field((1, 1, shape[2]), 13, 0.5)
    base, out = _guarded(shape)
    ny, nx = shape[1], shape[2]
    straddle = []  # (y, x0) of vectors that cross from row y into row y + 1, past 2^31
    for x0 in (65536, 65537, 65538):
        y = next(y for y in range(ny - 8, ny - 1) if (y * nx + x0) % 4 == 0)
        straddle.append((y, x0))
    for op in ("diff", "interp"):
        for lo, hi in ((1, 0), (0, 1)):
            ctx = f"stencil2 axis 0 {op} lo={lo} hi={hi} {layout}"
            with _Kernels() as k:
                ops.stencil2(x, 0, op, lo, hi, "fill", 1.5, pre=pre, post=post, out=out)
            k.ran("k_stencil_plane<float, 4," if layout == "broadcast" else "k_stencil_plane<float, 1,")
            _check_guard(base, ctx)
            _blocks(out, 1, 2048, lambda s, l: _stencil0_want(op, lo, x[:, s:s + l] * pre[:, s:s + l]) / post, ctx)
            cells = [c for c in _far_cells(shape)]
            for y, x0 in straddle:
                cells += [(0, y, x0 + k_) for k_ in range(nx - x0)] + [(0, y + 1, k_) for k_ in range(4 - (nx - x0))]
            for c in cells:
                sl = tuple(slice(v, v + 1) for v in c)
                want = oracle.stencil2(op, _np(x[sl]), 0, lo, hi, "fill", 1.5, pre=_np(pre.expand(shape)[sl]),
                                       post=_np(post.expand(shape)[sl]))
                np.testing.assert_array_equal(_np(out[sl]), want, err_msg=f"{ctx} cell {c}")


# ---------------------------------------------------------------------------------------------- 2
def test_stencil2_plane_strips_past_2_31():
    """2: (2^31 + 64, 1, 2) along axis 1: 2^31 + 64 strips of k_stencil_plane<float, 1> (XgPlanePlan.small = 0)."""
    ops = _ops()
    shape = SHAPE["stencil2_plane_strips"]
    _need(41)  # x, out 17.2 GB each; two 2.1 GB block temporaries
    x = _field(shape, 21)
    base, out = _guarded(shape)
    for op, bc, want in (("diff", "fill", lambda s, l: x[s:s + l] - 1.5),
                         ("interp", "periodic", lambda s, l: (x[s:s + l] + x[s:s + l]) * 0.5)):
        ctx = f"stencil2 axis 1 {op} {bc}"
        with _Kernels() as k:
            ops.stencil2(x, 1, op, 1, 0, bc, 1.5, out=out)
        k.ran("k_stencil_plane<float, 1,")
        _check_guard(base, ctx)
        _blocks(out, 0, PIECE, want, ctx)
        for c in _far_cells(shape):
            sl = (slice(c[0], c[0] + 1), slice(None), slice(None))
            np.testing.assert_array_equal(_np(out[sl]), oracle.stencil2(op, _np(x[sl]), 1, 1, 0, bc, 1.5), err_msg=ctx)


# ---------------------------------------------------------------------------------------------- 3 / 4
def _by_pieces(fn, x, dim, *args, **kw):
    """fn on contiguous pieces of x along dim: the concatenation is the reference."""
    def want(s, l):
        return fn(x.narrow(dim, s, l).contiguous(), *args, **kw)
    return want


def test_wreduce_strided_past_2_31():
    """3: k_reduce_strided<float, 1, true, 8> with small_index = 0, sum and mean with a (2, 1) weight."""
    ops = _ops()
    shape = SHAPE["wreduce_strided"]
    _need(31)  # x 17.2 GB, result 8.6 GB, a 2.1 GB piece and its 1.1 GB result
    x = _field(shape, 31)
    w = torch.tensor([[0.75], [1.3]], dtype=torch.float32, device=DEV)
    for mode in ("sum", "mean"):
        ctx = f"wreduce axis 0 {mode}"
        with _Kernels() as k:
            got = ops.wreduce(x, 0, w, mode)
        k.ran("k_reduce_strided<float, 1, true,")
        _blocks(got, 0, PIECE, lambda s, l: ops.wreduce(x[:, s:s + l].contiguous(), 0, w, mode), ctx)
        for (c,) in [(f,) for f in (N31 - 1, N31, shape[1] - 1)]:
            want = oracle.wreduce(_np(x[:, c:c + 1]), _np(w), 0, mode)
            np.testing.assert_array_equal(_np(got[c:c + 1]), want, err_msg=f"{ctx} column {c}")
        del got


def test_cumscan_strided_past_2_31():
    """4: k_scan_strided<float, 1, true, 8> with small_index = 0, one trim / pad case per direction."""
    ops = _ops()
    shape = SHAPE["cumscan_strided"]
    _need(43)  # x, result 17.2 GB each, a 2.1 GB piece, its 2.1 GB result and a 2.1 GB copy of the result block
    x = _field(shape, 41)
    pre = torch.tensor([[0.75], [1.3]], dtype=torch.float32, device=DEV)
    for rev, trim, plo, phi, bc in ((False, "drop_last", 1, 0, "fill"), (True, "drop_first", 0, 1, "extend")):
        ctx = f"cumscan axis 0 reverse={rev} {trim} pad=({plo}, {phi}) {bc}"
        with _Kernels() as k:
            got = ops.cumscan(x, 0, rev, trim, plo, phi, bc, 0.0, pre=pre)
        k.ran("k_scan_strided<float, 1, true,")
        _blocks(got, 1, PIECE,
                lambda s, l: ops.cumscan(x[:, s:s + l].contiguous(), 0, rev, trim, plo, phi, bc, 0.0, pre=pre), ctx)
        for c in (N31 - 1, N31, shape[1] - 1):
            want = oracle.cumscan(_np(x[:, c:c + 1]), 0, rev, trim, plo, phi, bc, 0.0, pre=_np(pre))
            np.testing.assert_array_equal(_np(got[:, c:c + 1]), want, err_msg=f"{ctx} column {c}")
        del got


# ---------------------------------------------------------------------------------------------- 5 / 6
def test_pad_past_2_31():
    """5: k_pad<float, 1> over (1, 2^31 + 5) along axis 0 and k_pad_rows<float, 4> over (268435457, 7) -> rows of 8,
    both with small = 0."""
    ops = _ops()
    _need(28)  # x 8.6 GB, result 17.2 GB, a 1.1 GB block (the rows part: 7.5 + 8.6 GB + 2.1 GB of blocks)
    x = _field(SHAPE["pad_strided"], 51)
    for lo, hi, bc in ((1, 0, "periodic"), (0, 1, "extend"), (1, 0, "fill")):
        ctx = f"pad axis 0 ({lo}, {hi}) {bc}"
        with _Kernels() as k:
            got = ops.pad(x, 0, lo, hi, bc, 1.5)
        k.ran("k_pad<float, 1>")
        for r in range(2):
            if (r == 0) == bool(lo) and bc == "fill":  # the halo row
                want = lambda s, l: torch.full((1, l), 1.5, dtype=torch.float32, device=DEV)
            else:  # the field row, or a halo that repeats it (periodic / extend of a one-row axis)
                want = lambda s, l: x[:, s:s + l]
            _blocks(got[r:r + 1], 1, PIECE, want, f"{ctx} row {r}")
        for c in (N31 - 1, N31, x.shape[1] - 1):
            want = oracle.pad_axis(_np(x[:, c:c + 1]), 0, lo, hi, bc, 1.5)
            np.testing.assert_array_equal(_np(got[:, c:c + 1]), want, err_msg=f"{ctx} column {c}")
        del got
    del x
    gc.collect()
    torch.cuda.empty_cache()
    x = _field(SHAPE["pad_rows"], 52)
    for lo, hi, bc in ((1, 0, "periodic"), (0, 1, "extend")):
        ctx = f"pad last axis ({lo}, {hi}) {bc}"
        with _Kernels() as k:
            got = ops.pad(x, 1, lo, hi, bc)
        k.ran("k_pad_rows<float, 4>")
        edge = x[:, 6:7] if bc == "periodic" else (x[:, 6:7] if hi else x[:, :1])
        want = lambda s, l: torch.cat([edge[s:s + l], x[s:s + l]] if lo else [x[s:s + l], edge[s:s + l]], dim=1)
        _blocks(got, 0, PIECE // 8, want, ctx)
        for c in _far_cells(got.shape):
            r = c[0]
            np.testing.assert_array_equal(_np(got[r:r + 1]), oracle.pad_axis(_np(x[r:r + 1]), 1, lo, hi, bc), err_msg=ctx)
        del got


def test_binary_past_2_31():
    """6: k_binary<float, 1, op> with small = 0: rows of 2^30 + 3 against a row-broadcast b."""
    ops = _ops()
    shape = SHAPE["binary"]
    _need(28)  # a, result 8.6 GB each, b 4.3 GB, a 2.1 GB reference block and a 2.1 GB copy of the result block
    a = _field(shape, 61)
    b = _field(shape[1:], 62, 0.5)
    for name, fn, np_fn in (("sub", torch.sub, np.subtract), ("div", torch.div, np.divide)):
        with _Kernels() as k:
            got = ops.binary(name, a, b)
        k.ran("k_binary<float, 1,")
        _blocks(got, 1, PIECE, lambda s, l: fn(a[:, s:s + l], b[s:s + l]), f"binary {name}")
        for r, c in _far_cells(shape):  # numpy, one float32 operation, as the elementwise sweep's oracle
            want = np_fn(_np(a[r, c:c + 1]), _np(b[c:c + 1]))
            np.testing.assert_array_equal(_np(got[r, c:c + 1]), want, err_msg=f"binary {name} cell {(r, c)}")
        del got


# ---------------------------------------------------------------------------------------------- 7 / 8
def test_vinterp_linear_past_2_31():
    """7: 2^31 + 5 columns (small_cols = 0); the TMA route refuses inner >= 2^31, so a non-TMA kernel runs."""
    ops = _ops()
    shape = SHAPE["vinterp_linear"]
    _need(31)  # phi 17.2 GB, result 8.6 GB, a 2.1 GB piece and its 1.1 GB result
    phi = _field(shape, 71)
    theta = torch.tensor([[0.0], [1.0]], dtype=torch.float32, device=DEV)
    target = torch.tensor([0.3], dtype=torch.float32, device=DEV)
    with _Kernels() as k:
        got = ops.vinterp_linear(phi, theta, target, 0)
    assert any(n.startswith(("k_vinterp_shared<", "k_vinterp_columns<")) for n in k.names), sorted(k.names)
    assert not any("tma" in n for n in k.names), sorted(k.names)
    _blocks(got, 0, PIECE, lambda s, l: ops.vinterp_linear(phi[:, s:s + l].contiguous(), theta, target, 0), "vinterp_linear")
    for c in (N31 - 1, N31, shape[1] - 1):
        want = oracle.vinterp_linear(_np(phi[:, c:c + 1]), _np(theta), _np(target), 0)
        np.testing.assert_array_equal(_np(got[c:c + 1]), want, err_msg=f"vinterp_linear column {c}")


def test_vinterp_conservative_past_2_31():
    """8: k_vconserv<float> over 2^31 + 5 columns (small_cols = 0)."""
    ops = _ops()
    shape = SHAPE["vinterp_conservative"]
    _need(21)  # phi, result 8.6 GB each, a 1.1 GB piece and its 1.1 GB result
    phi = _field(shape, 81)
    theta = torch.tensor([[0.0], [1.0]], dtype=torch.float32, device=DEV)
    bins = torch.tensor([0.2, 0.7], dtype=torch.float32, device=DEV)
    with _Kernels() as k:
        got = ops.vinterp_conservative(phi, theta, bins, 0)
    k.ran("k_vconserv<float>")
    _blocks(got, 0, PIECE, lambda s, l: ops.vinterp_conservative(phi[:, s:s + l].contiguous(), theta, bins, 0),
            "vinterp_conservative")
    for c in (N31 - 1, N31, shape[1] - 1):
        want = oracle.vinterp_conservative(_np(phi[:, c:c + 1]), _np(theta), _np(bins), 0)
        np.testing.assert_array_equal(_np(got[c:c + 1]), want, err_msg=f"vinterp_conservative column {c}")


# ---------------------------------------------------------------------------------------------- 9
@pytest.mark.parametrize("case", ["stencil_pair_inner", "stencil_pair_units"])
def test_stencil_pair_past_2_31(case):
    """9: max along X + min along axis 0 of (1, 32768, 65540): k_stencil_pair<float, 4> with small_inner = 0.
    9b: (2^31 + 8, 1, 1) along axis 1: 2^31 + 8 warp units (small_units = 0) of k_stencil_pair<float, 1>."""
    ops = _ops()
    shape = SHAPE[case]
    _need(31)  # a, b, result 8.6 GB each; pieces of a, b and their result, up to 1.1 GB each
    a, b = _field(shape, 91), _field(shape, 92)
    axis_b, dim = (0, 1) if case == "stencil_pair_inner" else (1, 0)
    spec_a, spec_b = ("max", 1, 0, "periodic", 0.0), (axis_b, "min", 1, 0, "fill", 0.5)
    with _Kernels() as k:
        got = ops.stencil_pair(a, b, spec_a, spec_b)
    k.ran("k_stencil_pair<float, 4," if case == "stencil_pair_inner" else "k_stencil_pair<float, 1,")
    step = 2048 if dim == 1 else PIECE
    _blocks(got, dim, step, lambda s, l: ops.stencil_pair(a.narrow(dim, s, l).contiguous(),
                                                          b.narrow(dim, s, l).contiguous(), spec_a, spec_b), case)
    for c in _far_cells(shape):
        sl = tuple(slice(v, v + 1) if d != 2 else slice(None) for d, v in enumerate(c))
        want = oracle.stencil_pair("max", _np(a[sl]), 2, 1, 0, "periodic", 0.0, None,
                                   "min", _np(b[sl]), axis_b, 1, 0, "fill", 0.5, None)
        np.testing.assert_array_equal(_np(got[sl]), want, err_msg=f"{case} cell {c}")


# ---------------------------------------------------------------------------------------------- 10 / 11
def test_stencil2_row_tma_refused_past_2_30():
    """10: rows of 2^30 + 512 with level-shared (1, n) metrics: the row TMA kernel refuses n >= 2^30 and
    k_stencil_row_zb takes the call (divisor shared between the two levels)."""
    ops = _ops()
    shape = SHAPE["stencil2_row_zb"]
    n = shape[1]
    _need(32)  # x, out 8.6 GB each, pre, post 4.3 GB each, up to seven 0.54 GB block temporaries
    x = _field(shape, 101)
    pre, post = _field((1, n), 102, 0.5), _field((1, n), 103, 0.5)
    base, out = _guarded(shape)
    with _Kernels() as k:
        ops.stencil2(x, 1, "diff", 1, 0, "periodic", pre=pre, post=post, out=out)
    k.ran("k_stencil_row_zb<float, 4,")
    assert not any(nm.startswith("k_stencil_row_tma") for nm in k.names)
    _check_guard(base, "stencil2 row_zb")

    def want(s, l):
        A = x[:, s:s + l] * pre[:, s:s + l]
        if s == 0:
            prev = torch.cat([x[:, n - 1:n] * pre[:, n - 1:n], x[:, :l - 1] * pre[:, :l - 1]], dim=1)
        else:
            prev = x[:, s - 1:s + l - 1] * pre[:, s - 1:s + l - 1]
        return (A - prev) / post[:, s:s + l]

    _blocks(out, 1, PIECE // 4, want, "stencil2 row_zb")
    for c in (0, N30 - 1, N30, n - 1):
        cols = [n - 1, 0] if c == 0 else [c - 1, c]  # column c and its periodic lower neighbour
        want_c = oracle.stencil2("diff", _np(x[:, cols]), 1, 0, 0, None, pre=_np(pre[:, cols]),
                                 post=_np(post[:, c:c + 1]))
        np.testing.assert_array_equal(_np(out[:, c:c + 1]), want_c, err_msg=f"row_zb column {c}")


def test_stencil2_tile_refused_past_2_30():
    """11: a unit axis of (2, 1, 2^30 + 512) with a (1, 1, n) divisor: the tile kernel refuses n >= 2^30 and
    k_stencil_plane<float, 4> runs."""
    ops = _ops()
    shape = SHAPE["stencil2_tile_refused"]
    _need(30)  # x, out 8.6 GB each, post 4.3 GB, three 2.1 GB block temporaries
    x = _field(shape, 111)
    post = _field((1, 1, shape[2]), 112, 0.5)
    base, out = _guarded(shape)
    with _Kernels() as k:
        ops.stencil2(x, 1, "diff", 0, 1, "fill", 0.25, post=post, out=out)
    k.ran("k_stencil_plane<float, 4,")
    assert not any(nm.startswith("k_tile_stencil") for nm in k.names)
    _check_guard(base, "stencil2 tile refused")
    _blocks(out, 2, PIECE, lambda s, l: (0.25 - x[:, :, s:s + l]) / post[:, :, s:s + l], "stencil2 tile refused")
    for c in (N30 - 1, N30, shape[2] - 1):
        sl = (slice(None), slice(None), slice(c, c + 1))
        want = oracle.stencil2("diff", _np(x[sl]), 1, 0, 1, "fill", 0.25, post=_np(post[sl]))
        np.testing.assert_array_equal(_np(out[sl]), want, err_msg=f"tile refused column {c}")


# ---------------------------------------------------------------------------------------------- 12
@pytest.mark.parametrize("op", ["diff", "interp"])
def test_grid_north_fold_past_2_31(op):
    """12: Grid.diff / Grid.interp along Y of a (9, 16384, 16400) device field at `left` under a corner pivot: the
    folded north row (k_fold_rows) is read from source offsets past 2^31 and handed to k_stencil_plane<float, 4> as
    its upper halo plane.  Reference: the same call level by level (268 M cells each); oracle/fold.py at the far
    cells and along the whole folded row of the last level."""
    import warnings

    import xgcm_b200 as xg

    nz, ny, nx = SHAPE["grid_fold_y"]
    _need(24)  # x, result 9.7 GB each, a 1.1 GB level and its 1.1 GB result
    ds = xg.Dataset(coords={"xc": np.arange(nx), "yl": np.arange(ny), "yc": np.arange(ny)})
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        grid = xg.Grid(ds, coords={"X": {"center": "xc"}, "Y": {"center": "yc", "left": "yl"}},
                       padding={"X": "periodic", "Y": {"fold": "corner"}}, autoparse_metadata=False)
    dims = ("z", "yl", "xc")
    x = _field((nz, ny, nx), 131)
    with _Kernels() as k:
        got = getattr(grid, op)(xg.DataArray(x, dims=dims), "Y").data
    k.ran("k_fold_rows<float>")
    k.ran("k_stencil_plane<float, 4,")
    assert tuple(got.shape) == (nz, ny, nx)
    _blocks(got, 0, 1, lambda s, l: getattr(grid, op)(xg.DataArray(x[s:s + l].contiguous(), dims=dims), "Y").data,
            f"fold {op}")
    for z, y, c in _far_cells((nz, ny, nx)):
        if y < ny - 1:  # an interior row: OP(x[y], x[y + 1])
            want = oracle.stencil2(op, _np(x[z:z + 1, y:y + 2, c:c + 1]), 1, 0, 0, None)
            np.testing.assert_array_equal(_np(got[z:z + 1, y:y + 1, c:c + 1]), want, err_msg=f"fold {op} {(z, y, c)}")
    z = nz - 1  # the folded row of the last level, every cell past 2^31
    top = _np(x[z:z + 1, -2:])
    halo = fold_oracle.north_rows(_np(x[z:z + 1, -3:]), 1, 2, "left", "center",
                                  fold_oracle.resolve_pivot("corner", "Y", "X"), 1)
    want = oracle.stencil2(op, np.concatenate([top[:, 1:], halo], axis=1), 1, 0, 0, None)
    np.testing.assert_array_equal(_np(got[z:z + 1, -1:]), want, err_msg=f"fold {op} top row")


def test_torch_reference_matches_oracle():
    """The torch formulas above, one IEEE operation per call, agree with the CPU oracle on a small case."""
    x = _field((1, 5, 7), 121)
    pre, post = _field((1, 5, 1), 122, 0.5), _field((1, 1, 7), 123, 0.5)
    for op in ("diff", "interp"):
        for lo, hi in ((1, 0), (0, 1)):
            got = _stencil0_want(op, lo, x * pre) / post
            want = oracle.stencil2(op, _np(x), 0, lo, hi, "fill", 1.5, pre=_np(pre), post=_np(post))
            np.testing.assert_array_equal(_np(got), want)


# ---------------------------------------------------------------------------------------------- strided operands
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _views(dt, seed, shape):
    """(name, device view, host array) of metrics for a field of ``shape`` = (Z, Y, X) with non-zero strides in more
    than one inner group: a transposed (X, Y) array, a permuted (X, Z, Y) one, and a slice of a wider array."""
    rng = np.random.default_rng(seed)
    Z, Y, X = shape
    t = _dev((0.5 + rng.random((X, Y))).astype(dt))
    p = _dev((0.5 + rng.random((X, Z, Y))).astype(dt))
    s = _dev((0.5 + rng.random((Z, Y, X + 5))).astype(dt))
    out = [("transposed", t.T[None]), ("permuted", p.permute(1, 2, 0)), ("sliced", s[:, :, :X])]
    return [(name, v, v.cpu().numpy()) for name, v in out]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_strided_operands_against_oracle(dtype):
    """Operands as permuted and sliced views (XG_IM_GENERIC with two inner groups), innermost extents that are not a
    multiple of the vector width so vectors straddle rows: stencil2 (plane, row_vec and row_scalar routes), stencil_pair,
    cumscan against the oracle; wreduce and the vertical interpolations against the same call with contiguous copies
    of the operands (which the generic path must match bit for bit).  The kernels each shape must reach are checked
    with the profiler: (3, 4, 37) and (3, 300, 117) along Z give plane rows that are a multiple of the vector width
    of an odd X, so the vector instances see straddling vectors; (3, 300, 117) has enough columns (35100 / VEC >=
    XG_SMS * 64) for the vector instances of the strided scan and reduction."""
    ops = _ops()
    tdt = torch.float32 if dtype == np.float32 else torch.float64
    t, vec = ("float", 4) if dtype == np.float32 else ("double", 2)
    expect = {
        (3, 6, 37): [],
        (3, 4, 37): [f"k_stencil_plane<{t}, {vec},"],
        (4, 5, 136): [f"k_stencil_row_vec<{t}, {vec},"],
        (2, 3, 7): [f"k_stencil_row_scalar<{t},"],
        (3, 300, 117): [f"k_stencil_plane<{t}, {vec},", f"k_scan_strided<{t}, {vec}, true,",
                        f"k_reduce_strided<{t}, {vec}, true,"],
    }
    for shape, kernels in expect.items():
        rng = np.random.default_rng(sum(shape))
        xh = rng.standard_normal(shape).astype(dtype)
        x = _dev(xh)
        with _Kernels() as k:
            _strided_sweep(ops, tdt, dtype, shape, x, xh)
        for prefix in kernels:
            k.ran(prefix)


def _strided_sweep(ops, tdt, dtype, shape, x, xh):
    """One shape of test_strided_operands_against_oracle, every view and op."""
    for name, m, mh in _views(dtype, shape[2], shape):
        ctx = f"{np.dtype(dtype).name} {shape} {name}"
        for axis in (0, 1, 2):
            for op in ("diff", "interp", "max"):
                for lo, hi, bc in ((1, 0, "fill"), (0, 1, "periodic"), (1, 1, "extend")):
                    got = ops.stencil2(x, axis, op, lo, hi, bc, 0.5, pre=m)
                    want = oracle.stencil2(op, xh, axis, lo, hi, bc, 0.5, pre=mh)
                    np.testing.assert_array_equal(_np(got), want, err_msg=f"{ctx} stencil2 {axis} {op} {lo}{hi} {bc}")
            got = ops.stencil2(x, axis, "diff", 1, 0, "fill", 0.0, post=m)
            want = oracle.stencil2("diff", xh, axis, 1, 0, "fill", 0.0, post=mh)
            np.testing.assert_array_equal(_np(got), want, err_msg=f"{ctx} stencil2 post {axis}")
        for axis_b in (0, 1):
            got = ops.stencil_pair(x, x, ("diff", 1, 0, "periodic", 0.0), (axis_b, "interp", 0, 1, "fill", 0.5),
                                   subtract=1, pre_a=m, pre_b=m, post=m)
            want = oracle.stencil_pair("diff", xh, 2, 1, 0, "periodic", 0.0, mh, "interp", xh, axis_b, 0, 1, "fill",
                                       0.5, mh, subtract=True, post=mh)
            np.testing.assert_array_equal(_np(got), want, err_msg=f"{ctx} stencil_pair {axis_b}")
        for axis in (0, 1):
            got = ops.cumscan(x, axis, False, "none", 0, 0, None, 0.0, pre=m, post=m)
            want = oracle.cumscan(xh, axis, False, "none", 0, 0, None, 0.0, pre=mh, post=mh)
            np.testing.assert_array_equal(_np(got), want, err_msg=f"{ctx} cumscan {axis}")
            for mode in ("sum", "mean"):
                got = ops.wreduce(x, axis, m, mode)
                want = ops.wreduce(x, axis, m.contiguous(), mode)
                _bits(got, want, f"{ctx} wreduce {axis} {mode}")
        # theta: cumulative metric along axis 0, so it increases in every column
        th = torch.cumsum(m.expand(shape), 0)
        th_view = th.permute(2, 0, 1).contiguous().permute(1, 2, 0)  # same values, permuted strides
        tg = torch.tensor([0.7, 1.5, 2.2], dtype=tdt, device=DEV)
        got = ops.vinterp_linear(x, th_view, tg, 0)
        _bits(got, ops.vinterp_linear(x, th_view.contiguous(), tg, 0), f"{ctx} vinterp_linear")
        bounds = torch.cat([torch.zeros_like(th[:1]), th], 0)
        b_view = bounds.permute(2, 0, 1).contiguous().permute(1, 2, 0)
        bins = torch.tensor([0.0, 0.9, 1.7, 3.0], dtype=tdt, device=DEV)
        got = ops.vinterp_conservative(x, b_view, bins, 0)
        _bits(got, ops.vinterp_conservative(x, b_view.contiguous(), bins, 0), f"{ctx} vinterp_conservative")
