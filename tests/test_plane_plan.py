"""The work decomposition of the plane-strided stencil (xgcm_b200/csrc/xg_plane.cuh), compiled as plain C++ on
the host: for every warp and lane of a launch, the (plane, output row, element) cells it writes are counted, and
every cell of the output must be written exactly once.  Tiling errors show up here instead of as an
out-of-bounds access on the GPU."""

import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "xgcm_b200", "csrc")

DRIVER = r"""
#include "xg_plane.cuh"
#include <stdio.h>
#include <stdlib.h>
#include <vector>

// argv: outer inner n_out elem_size vec J
int main(int argc, char** argv) {
  if (argc != 7) return 2;
  const int64_t outer = atoll(argv[1]), inner = atoll(argv[2]), n_out = atoll(argv[3]);
  const int es = atoi(argv[4]), vec = atoi(argv[5]);
  const int lpl = 128 / (vec * es), lpw = 32 / lpl;  // as PlaneGeo in xg_stencil2.cu
  const XgPlanePlan p = xg_plane_plan(outer, inner, n_out, lpl * vec, lpw, atoll(argv[6]));
  if (p.nwarps < 1) return 3;
  std::vector<unsigned char> hits((size_t)(outer * n_out * inner), 0);
  long long bad = 0, calls = 0;
  for (int64_t w = 0; w < p.nwarps; ++w)
    for (int lane = 0; lane < 32; ++lane)
      xg_plane_walk(p, inner, n_out, lpl, lpw, vec, w, lane, [&](int64_t o, int64_t i, int64_t j0, int64_t j1) {
        ++calls;
        if (o < 0 || o >= outer || i < 0 || i + vec > inner || j0 < 0 || j1 > n_out || j0 >= j1) {
          ++bad;
          return;
        }
        for (int64_t j = j0; j < j1; ++j)
          for (int k = 0; k < vec; ++k) ++hits[(size_t)((o * n_out + j) * inner + i + k)];
      });
  long long zero = 0, multi = 0;
  for (unsigned char h : hits) {
    zero += h == 0;
    multi += h > 1;
  }
  printf("%lld %lld %lld %lld %lld\n", (long long)p.nwarps, bad, zero, multi, calls);
  return 0;
}
"""

# inner widths that end mid-line (4, 36 fp32 elements), mid-warp (900 + 4) and on a warp boundary (3600), the fp64
# analogues, and VEC = 1 (rows not a multiple of the vector width)
INNER = {(4, 4): [4, 36, 904, 3600], (8, 2): [2, 18, 452, 1800], (4, 1): [1, 3, 37, 905], (8, 1): [1, 7, 451]}
SHAPES = [(1, 1), (1, 75), (3, 2), (7, 33), (5, 240)]  # (outer, n_out)
CASES = [
    (es, vec, outer, inner, n_out, J)
    for (es, vec), inners in INNER.items()
    for inner in inners
    for outer, n_out in SHAPES
    for J in (1, 3, 8, 32, 1000)
]


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:  # pragma: no cover
        pytest.skip("no C++ compiler")
    d = tmp_path_factory.mktemp("plane_plan")
    src = d / "plane_plan.cpp"
    src.write_text(DRIVER)
    exe = d / "plane_plan"
    subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-Werror", "-I", CSRC, str(src), "-o", str(exe)], check=True)
    return str(exe)


@pytest.mark.parametrize("es,vec,outer,inner,n_out,J", CASES)
def test_plane_walk_writes_every_cell_once(driver, es, vec, outer, inner, n_out, J):
    out = subprocess.run([driver, str(outer), str(inner), str(n_out), str(es), str(vec), str(J)],
                         check=True, capture_output=True, text=True).stdout.split()
    nwarps, bad, zero, multi, calls = map(int, out)
    assert bad == 0 and zero == 0 and multi == 0, out
    assert nwarps >= 1 and calls > 0


def test_c3_y_plan_shape(driver):
    """The flagship Y launch (75, 2400, 3600) fp32 with J = 8: 113 lines per row (the last one half used), every
    cell once, and no warp idle — 112.5 / 113 of the lanes at work instead of 28.125 / 29 warps."""
    out = subprocess.run([driver, "75", "3600", "2400", "4", "4", "8"], check=True,
                         capture_output=True, text=True).stdout.split()
    nwarps, bad, zero, multi, calls = map(int, out)
    assert (bad, zero, multi) == (0, 0, 0)
    assert nwarps == -(-75 * 300 * 113 // 4)
    assert calls == 75 * 300 * (112 * 8 + 4)
