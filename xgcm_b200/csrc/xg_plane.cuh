// xg_plane.cuh — work decomposition of the plane-strided stencil (k_stencil_plane, xg_stencil2.cu).
//
// The field is (outer, n, inner) with inner > 1.  Each plane row of `inner` elements is cut into 128-byte
// *lines* (LPL lanes x VEC elements; the last line of a row may be partly empty), and the output rows of a plane
// into segments of J rows.  A *strip* is one line of one segment: LPL lanes march its J rows carrying the
// previous row in registers.  Strips are numbered (plane, segment, line) with the line fastest and a warp takes
// LPW = 32 / LPL consecutive strips, so a row ending mid-warp costs a few idle lanes, not an idle warp, and
// warps adjacent in launch order (resident at the same time) read and write neighbouring addresses.
//
// Plain C++ as well as CUDA: tests/test_plane_plan.py compiles it on the host and checks that the strips and
// lanes cover every (plane, row, element) of the output exactly once.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define XG_PLANE_HD __host__ __device__ __forceinline__
#else
#define XG_PLANE_HD inline
#endif

struct XgPlanePlan {
  int64_t nlines;   // 128-byte lines per plane row
  int64_t J;        // output rows per segment
  int64_t nseg;     // segments per plane
  int64_t nstrips;  // outer * nseg * nlines
  int64_t nwarps;   // ceil(nstrips / LPW)
  bool small;       // nstrips < 2^31: 32-bit index arithmetic
};

// elems_per_line = LPL * VEC, lpw = LPW
inline XgPlanePlan xg_plane_plan(int64_t outer, int64_t inner, int64_t n_out, int elems_per_line, int lpw,
                                 int64_t J) {
  XgPlanePlan p;
  p.nlines = (inner + elems_per_line - 1) / elems_per_line;
  p.J = J < n_out ? J : n_out;
  p.nseg = (n_out + p.J - 1) / p.J;
  p.nstrips = outer * p.nseg * p.nlines;
  p.nwarps = (p.nstrips + lpw - 1) / lpw;
  p.small = p.nstrips < (int64_t(1) << 31);
  return p;
}

// what lane `lane` of warp w computes: f(o, i, j0, j1) for output rows [j0, j1) of the `vec` elements starting at
// inner index i of plane o; lanes past the end of a row or of the last strip do nothing
template <class F>
XG_PLANE_HD void xg_plane_walk(const XgPlanePlan& p, int64_t inner, int64_t n_out, int lpl, int lpw, int vec,
                               int64_t w, int lane, F&& f) {
  const int q = lane / lpl, sub = lane - q * lpl;
  const int64_t s = w * lpw + q;
  if (s >= p.nstrips) return;
  int64_t t, o, seg;
  if (p.small) {
    const uint32_t t32 = (uint32_t)s / (uint32_t)p.nlines, o32 = t32 / (uint32_t)p.nseg;
    t = t32;
    o = o32;
    seg = t32 - o32 * (uint32_t)p.nseg;
  } else {
    t = s / p.nlines;
    o = t / p.nseg;
    seg = t - o * p.nseg;
  }
  const int64_t l = s - t * p.nlines;
  const int64_t i = (l * lpl + sub) * vec;
  if (i >= inner) return;
  const int64_t j0 = seg * p.J;
  f(o, i, j0, (n_out - j0 < p.J) ? n_out : j0 + p.J);
}
