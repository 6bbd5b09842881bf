"""64-bit index paths, on the host.

Most launchers pick a 32-bit index path (multiply-high divisions, ``uint32_t`` arithmetic) while a count stays below
2^31 and a 64-bit path past it, and some routes (TMA tile coordinates) refuse a size and hand the call to another
kernel.  ``test_index64_gpu.py`` runs one field per gate that an 80 GB device can flip.  Here:

* every shape of that file is checked against the launcher predicate it is meant to cross, restated from the source,
  so that a later edit of a shape or a threshold cannot silently drop a case back to the 32-bit path;
* the gates no 80 GB device can flip are listed with the arithmetic, so nobody mistakes them for covered;
* the operand descriptor (``xg_make_operand``, xg_core.cu) of a transposed metric whose elements lie more than 2^31
  apart is built by a host-only driver: a vector of such an operand may straddle two rows whose offsets differ by
  more than ``XgOperandView``'s 32-bit deltas hold, and the descriptor must keep the vector kernels away from it.
"""

import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "xgcm_b200", "csrc")
INCLUDE = os.path.join(ROOT, "include")

N30, N31 = 1 << 30, 1 << 31
VEC32 = 4  # XgVecWidth<float>
HBM = 80 * 10**9  # bytes of the largest device the suite runs on

# fp32 field shapes of test_index64_gpu.py, one per gate
SHAPE = {
    "stencil2_operand_groups": (1, 32768, 65539),   # 1a / 1b: broadcast and transposed metrics
    "stencil2_plane_strips": (N31 + 64, 1, 2),      # 2
    "wreduce_strided": (2, N31 + 5),                # 3
    "cumscan_strided": (2, N31 + 5),                # 4
    "pad_strided": (1, N31 + 5),                    # 5
    "pad_rows": (268435457, 7),                     # 5, last axis
    "binary": (2, N30 + 3),                         # 6
    "vinterp_linear": (2, N31 + 5),                 # 7
    "vinterp_conservative": (1, N31 + 5),           # 8
    "stencil_pair_inner": (1, 32768, 65540),        # 9
    "stencil_pair_units": (N31 + 8, 1, 1),          # 9b
    "stencil2_row_zb": (2, N30 + 512),              # 10
    "stencil2_tile_refused": (2, 1, N30 + 512),     # 11
    "grid_fold_y": (9, 16384, 16400),               # 12: Grid.diff / interp along Y across the north fold
}


def _prod(s):
    r = 1
    for v in s:
        r *= v
    return r


def _cdiv(a, b):
    return -(-a // b)


def _collapse(shape, axis):
    """xg_collapse_view (xg_core.cu:53-67): (outer, n, inner)."""
    return _prod(shape[:axis]), shape[axis], _prod(shape[axis + 1:])


def _groups(shape, strides, d0, d1):
    """collapse_groups (xg_core.cu:71-118): [(size, stride)] and the `small` flag."""
    g = []
    for d in range(d0, d1):
        if shape[d] == 1:
            continue
        if g and g[-1][1] == strides[d] * shape[d]:
            g[-1] = (g[-1][0] * shape[d], strides[d])
            continue
        g.append((shape[d], strides[d]))
    small, total = True, 1
    for size, _ in g:
        if size >= N31 or total > N31 // max(size, 1):
            small = False
        total *= size
    extent = 1
    for d in range(d0, d1):
        if shape[d] > 0 and extent > N31 // shape[d]:
            small = False
        extent *= max(shape[d], 1)
    return g, small


def _bcast_strides(mshape, fshape):
    """Element strides of a contiguous operand of shape ``mshape`` broadcast to ``fshape`` (ops._operand)."""
    st, acc = [0] * len(fshape), 1
    for d in range(len(fshape) - 1, -1, -1):
        st[d] = 0 if mshape[d] == 1 else acc
        acc *= mshape[d]
    return st


# ---------------------------------------------------------------------------------------------- gates the cases flip
def test_stencil2_operand_groups_are_wide():
    """1a / 1b: stencil2 along axis 0 of (1, 32768, 65539).  The metrics' inner index groups (xg_core.cu:103-115) are
    not `small`, the TMA tile route declines them (`inner_split`, xg_stencil2.cu:983-996: one inner group at most),
    and the field's inner extent is a multiple of the vector width, so k_stencil_plane<float, 4> runs for 1a."""
    shape = SHAPE["stencil2_operand_groups"]
    outer, n, inner = _collapse(shape, 0)
    assert (outer, n) == (1, 1) and inner % VEC32 == 0 and inner > N31
    for mshape in ((1, 32768, 1), (1, 1, 65539)):  # pre, post of 1a
        g, small = _groups(shape, _bcast_strides(mshape, shape), 1, 3)
        assert len(g) == 2 and not small, (mshape, g)
    # 1b: m = w.T[None] of a contiguous (65539, 32768) w: strides (0, 1, 32768)
    g, small = _groups(shape, (0, 1, 32768), 1, 3)
    assert g == [(32768, 1), (65539, 32768)] and not small
    assert shape[2] % VEC32 != 0  # vectors straddle the rows of the innermost dim


def test_stencil2_plane_strips_past_2_31():
    """2: no metric, inner = 2 (not a multiple of 4): k_stencil_plane<float, 1>; xg_plane_plan (xg_plane.cuh:31-41)
    with LPL = 32 lanes x 1 element per line and J = n_out (n_out <= 96, xg_stencil2.cu:726) gives nstrips = outer."""
    outer, n, inner = _collapse(SHAPE["stencil2_plane_strips"], 1)
    assert inner % VEC32 != 0
    n_out = n + 1 + 0 - 1  # lo = 1, hi = 0
    nlines, J = _cdiv(inner, 32), n_out
    nstrips = outer * _cdiv(n_out, J) * nlines
    assert nstrips >= N31  # XgPlanePlan.small = 0


@pytest.mark.parametrize("case", ["wreduce_strided", "cumscan_strided"])
def test_strided_scan_and_reduce_index_past_2_31(case):
    """3 / 4: an odd inner extent takes the VEC = 1 instance (xg_wreduce.cu:148, xg_cumscan.cu:524) and
    outer * nvec_inner >= 2^31 clears `small_index` (xg_wreduce.cu:152, xg_cumscan.cu:538)."""
    outer, n, inner = _collapse(SHAPE[case], 0)
    assert n == 2 and inner % VEC32 != 0
    assert outer * inner >= N31
    g, _ = _groups(SHAPE[case], _bcast_strides((2, 1), SHAPE[case]), 1, 2)  # weight / pre (2, 1): inner broadcast
    assert g == [(N31 + 5, 0)]


def test_pad_index_past_2_31():
    """5: k_pad (xg_elementwise.cu:157-160): total = outer * n_out * nvec_inner >= 2^31 with VEC = 1;
    k_pad_rows (xg_elementwise.cu:145-149): inner == 1, n_out >= 8, total = outer * n_out >= 2^31."""
    outer, n, inner = _collapse(SHAPE["pad_strided"], 0)
    assert inner % VEC32 != 0 and outer * (n + 1) * inner >= N31
    outer, n, inner = _collapse(SHAPE["pad_rows"], 1)
    assert inner == 1 and n + 1 == 8 and outer * (n + 1) >= N31


def test_binary_index_past_2_31():
    """6: k_binary (xg_elementwise.cu:224-227, 256): a row length that is not a multiple of 4 gives VEC = 1 and
    rows * n >= 2^31 clears `small`."""
    rows, n, _ = _collapse(SHAPE["binary"], 1)
    assert n % VEC32 != 0 and rows * n >= N31


def test_vinterp_columns_past_2_31():
    """7 / 8: ncols = outer * inner >= 2^31 clears `small_cols` (xg_vinterp.cu:513, xg_vconserv.cu:164); for 7 the TMA
    route refuses inner >= 2^31 (xg_vinterp_tma.cu:528), so k_vinterp_shared runs (theta and target broadcast)."""
    for case in ("vinterp_linear", "vinterp_conservative"):
        outer, n, inner = _collapse(SHAPE[case], 0)
        assert outer * inner >= N31
    assert _collapse(SHAPE["vinterp_linear"], 0)[2] >= N31


def test_stencil_pair_index_past_2_31():
    """9: `small_inner` = inner < 2^31 (xg_stencil_pair.cu:235) with nx % 4 == 0 (the vector instance) and
    inner != nx (no tile route, xg_stencil_pair.cu:302).  9b: nunits = outer * nseg * nwc >= 2^31
    (xg_stencil_pair.cu:229-234) with nx = 1: one warp unit per row of one cell."""
    shape = SHAPE["stencil_pair_inner"]
    outer, nb, inner = _collapse(shape, 0)
    assert inner >= N31 and shape[-1] % VEC32 == 0 and inner != shape[-1]
    outer, nb, inner = _collapse(SHAPE["stencil_pair_units"], 1)
    J = nb if nb <= 96 else 32
    nunits = outer * _cdiv(nb, J) * _cdiv(_cdiv(inner, 1), 32)
    assert nunits >= N31


def test_row_tma_and_tile_routes_refuse():
    """10: stencil2 along the last axis with level-shared (1, n) metrics: k_stencil_row_tma refuses n >= 2^30
    (xg_stencil2.cu:819), and k_stencil_row_zb takes the call (Zn = 2 levels, P = 1 row, pre shared).
    11: stencil2 along a unit axis with a (1, 1, n) divisor: the tile kernel refuses n >= 2^30
    (xg_stencil_tile.cu:417) and k_stencil_plane runs."""
    outer, n, inner = _collapse(SHAPE["stencil2_row_zb"], 1)
    assert inner == 1 and n >= N30 and n % VEC32 == 0 and n // VEC32 >= 32 and outer == 2
    g, _ = _groups(SHAPE["stencil2_row_zb"], _bcast_strides((1, n), SHAPE["stencil2_row_zb"]), 0, 1)
    assert g == [(2, 0)]  # one broadcast level group: Zn = 2
    outer, n, inner = _collapse(SHAPE["stencil2_tile_refused"], 1)
    assert outer == 2 and inner >= N30 and inner % VEC32 == 0


def test_fold_rows_read_past_2_31():
    """12: k_fold_rows (xg_fold.cu:33-58) has no 32-bit path; its source offsets, (z, n - 1 - skip - r, mirror - k)
    in the input's strides, pass 2^31 for the last levels of a (9, 16384, 16400) field (skip = 1: a `left` field under
    a corner pivot), and the stencil that takes the folded row as its upper halo plane
    (k_stencil_plane<float, 4, ...>, plane strips well below 2^31) writes output past 2^31."""
    nz, ny, nx = SHAPE["grid_fold_y"]
    assert nz * ny * nx > N31
    top_src_last_level = ((nz - 1) * ny + ny - 1 - 1) * nx  # first source cell of the folded row of the last level
    assert top_src_last_level > N31
    outer, n, inner = _collapse(SHAPE["grid_fold_y"], 1)
    assert inner % VEC32 == 0 and outer * _cdiv(n, 4) * _cdiv(inner, 32) < N31  # J = 4, 32 fp32 cells per line


# ---------------------------------------------------------------------------------------------- unreachable gates
def _min_bytes_row_vec():
    # k_stencil_row_vec (xg_stencil2.cu:735-746): rows of n >= 128 cells (n / VEC >= 32); nwc = ceil(n / 512) <= n / 128,
    # so nunits = outer * nwc <= cells / 128: 2^31 units need 2^38 cells, read and written
    return N31 * 128 * 4 * 2


def _min_bytes_row_zb():
    # k_stencil_row_zb (xg_stencil2.cu:779-781): nunits = ceil(Zn / 4) * P * ceil(n / 128) with n >= 128, Zn >= 2, so
    # nunits <= Zn * P * n / 64 = cells / 64
    return N31 * 64 * 4 * 2


def _min_bytes_tiles():
    # TMA tile kernels (xg_stencil2.cu:888, xg_stencil_tile.cu:490, xg_stencil_multi_tma.cu:346): a tile holds U = 4
    # levels x TY rows x TXE = 224 fp32 cells; rows >= 2 * TXE long, so a tile averages >= 2 * 224 / 3 cells of a row,
    # and at least one row of half its levels (Zn >= 2 of U = 4)
    return N31 * (2 * 224 // 3) * 2 * 4 * 2


def _min_bytes_vinterp_tma():
    # k_vinterp_shared_tma / k_vinterp_columns_tma (xg_vinterp_tma.cu:452, 490, 889-890): ntiles = outer *
    # ceil(inner / TC) with TC >= 32 and inner >= 32 (xg_vinterp_tma.cu:528), so ntiles <= outer * inner / 16; with
    # n >= 2 levels the input holds >= 32 cells per tile: 2^31 tiles need 2^36 fp32 cells of phi alone
    return N31 * 32 * 4


UNREACHABLE = {
    "k_stencil_row_vec small_units": _min_bytes_row_vec,
    "k_stencil_row_zb small_units": _min_bytes_row_zb,
    "TMA tile kernels ntiles >= 2^31": _min_bytes_tiles,
    "vinterp TMA kernels ntiles >= 2^31": _min_bytes_vinterp_tma,
}


@pytest.mark.parametrize("gate", sorted(UNREACHABLE))
def test_unreachable_gates_need_more_than_a_device(gate):
    """The 64-bit branches of these gates stay unexercised: the smallest fp32 input and output that flip them exceed
    80 GB.  (k_stencil_pair's `small_units` is not among them: rows of one cell flip it, case 9b.)"""
    assert UNREACHABLE[gate]() > HBM


# ---------------------------------------------------------------------------------------------- operand descriptor
DRIVER = r"""
#include "xg_common.cuh"
#include <stdio.h>
#include <stdlib.h>

// argv: ndim shape[ndim] strides[ndim] axis vec
// prints: inner_mode small wide_span vec_view_ok max_abs_delta overflows worst_x0
int main(int argc, char** argv) {
  const int ndim = atoi(argv[1]);
  if (argc != 2 + 2 * ndim + 2) return 2;
  int64_t shape[8], strides[8];
  for (int d = 0; d < ndim; ++d) {
    shape[d] = atoll(argv[2 + d]);
    strides[d] = atoll(argv[2 + ndim + d]);
  }
  const int axis = atoi(argv[2 + 2 * ndim]), vec = atoi(argv[3 + 2 * ndim]);
  XgOperand op;
  // the descriptor never dereferences the pointer: any 16-byte aligned value
  if (xg_make_operand((const void*)(uintptr_t)4096, strides, ndim, shape, axis, vec, sizeof(float), &op, "pre"))
    return 3;
  XgView v;
  if (xg_collapse_view(ndim, shape, axis, &v)) return 4;
  // the deltas XgOperandView<float, vec> would store (xg_common.cuh) for every vector that holds the last element of a
  // row of the innermost dim, i.e. every vector that can straddle two rows, plus the first one
  const int64_t nx = shape[ndim - 1];
  long long overflows = 0;
  int64_t max_abs = 0, worst_x0 = -1;
  for (int64_t r = -1; r < v.inner / nx; ++r) {
    const int64_t i = r < 0 ? 0 : (r * nx + nx - 1) / vec * vec;
    if (i + vec > v.inner) continue;
    const int64_t o0 = xg_groups_offset(op.inner, i);
    for (int k = 1; k < vec; ++k) {
      const int64_t d = xg_groups_offset(op.inner, i + k) - o0;
      if ((int64_t)(int)d != d) ++overflows;
      const int64_t a = d < 0 ? -d : d;
      if (a > max_abs) {
        max_abs = a;
        worst_x0 = i % nx;
      }
    }
  }
  printf("%d %d %d %d %lld %lld %lld\n", op.inner_mode, op.inner.small, op.wide_span, (int)xg_vec_view_ok(op),
         (long long)max_abs, overflows, (long long)worst_x0);
  return 0;
}
"""


@pytest.fixture(scope="module")
def operand_driver(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):  # pragma: no cover
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("operand")
    src = d / "operand.cu"
    src.write_text(DRIVER)
    exe = d / "operand"
    subprocess.run([nvcc, "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-I", INCLUDE, "-I", CSRC,
                    str(src), os.path.join(CSRC, "xg_core.cu"), "-cudart", "static", "-o", str(exe)], check=True)
    return str(exe)


def _describe(driver, shape, strides, axis, vec=VEC32):
    args = [driver, str(len(shape)), *map(str, shape), *map(str, strides), str(axis), str(vec)]
    out = subprocess.run(args, check=True, capture_output=True, text=True).stdout.split()
    keys = ("mode", "small", "wide_span", "vec_view_ok", "max_abs_delta", "overflows", "worst_x0")
    return dict(zip(keys, map(int, out)))


def test_transposed_metric_past_2_31_refuses_vectors(operand_driver):
    """Case 1b: m = w.T[None] for a contiguous (65539, 32768) w against a (1, 32768, 65539) field, axis 0.  The
    vector starting at x0 = 65537 of row y holds (y, 65537), (y, 65538), (y + 1, 0), (y + 1, 1): offsets
    65537 * 32768 + y and y + 1, 2147516415 apart, more than an int holds (one starting at x0 = 65538: 2147549183).  The descriptor marks the operand
    wide, and every launcher that would vectorise over it takes its VEC = 1 instance instead."""
    r = _describe(operand_driver, (1, 32768, 65539), (0, 1, 32768), 0)
    print(f"\ntransposed (65539, 32768) metric: {r}")
    assert r["mode"] == 2 and r["small"] == 0  # XG_IM_GENERIC, 64-bit group offsets
    assert r["max_abs_delta"] == 65538 * 32768 - 1 and r["worst_x0"] == 65538
    assert r["overflows"] > 0  # what 32-bit deltas would have stored wrongly
    assert r["wide_span"] == 1 and r["vec_view_ok"] == 0


def test_operand_span_threshold(operand_driver):
    """Spans up to 2^31 - 1 keep the vector instances; 2^31 and more do not.  A (2, 3) inner block with strides
    (1, s) spans 1 + 2 s: s = 2^30 - 1 gives 2^31 - 1, s = 2^30 gives 2^31 + 1."""
    ok = _describe(operand_driver, (1, 2, 3), (0, 1, N30 - 1), 0)
    assert ok["mode"] == 2 and ok["wide_span"] == 0 and ok["vec_view_ok"] == 1 and ok["overflows"] == 0
    wide = _describe(operand_driver, (1, 2, 3), (0, 1, N30), 0)
    assert wide["wide_span"] == 1 and wide["vec_view_ok"] == 0


def test_small_transposed_and_broadcast_metrics_keep_vectors(operand_driver):
    """The layouts the library meets every day are untouched: a transposed (37, 1000) metric, a broadcast one, a
    contiguous one."""
    for shape, strides in (((5, 1000, 37), (0, 1, 1000)), ((5, 1000, 37), (0, 1, 0)), ((5, 1000, 36), (0, 36, 1))):
        r = _describe(operand_driver, shape, strides, 0)
        assert r["wide_span"] == 0 and r["vec_view_ok"] == 1 and r["overflows"] == 0, (shape, strides, r)
