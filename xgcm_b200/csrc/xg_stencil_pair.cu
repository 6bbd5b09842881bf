// xg_stencil_pair — a two-FIELD composite in one pass over HBM (SURVEY 8f row N1, second half):
//
//     out = ( OPa(pad_a(A x ma)) along the innermost dim   (+|-)   OPb(pad_b(B x mb)) along another dim ) / post
//
// e.g. the C-grid divergence (diff(u dyG, 'X') + diff(v dxG, 'Y')) / rA and the vorticity
// (diff(v dyC, 'X') - diff(u dxC, 'Y')) / rAz that users chain from Grid.diff calls and xarray arithmetic
// (xgcm docs/ufunc_examples.md:105-153; the per-axis loop of xgcm/grid.py:796-832 plus one full pass per
// arithmetic operator: ~9 passes and 5 temporaries in the reference, 3 array streams here: read A, read B,
// write out = 3 * sizeof(T) bytes per cell).
//
// Rounding is that of the sequential chain, operator by operator (--fmad=false, IEEE division):
//     ta = OPa(A x ma), tb = OPb(B x mb), s = ta +- tb, out = s / post   — each rounded to the field dtype.
// Both stencils are length preserving (lo + hi == 1: center <-> left / right), so A, B and out share one shape.
//
// xg_stencil_pair_halo takes optional halo planes of the B term (the folded north row of a tripolar grid): padB
// reads them instead of the boundary rule on their side, here and in the tile kernel (XgTileSpec::halo_lo / hi).
//
// Work split: a warp owns 32 x VEC contiguous cells of the innermost dim and marches J
// cells along axis b keeping B's previous row in registers; the x-neighbour of A comes from a warp shuffle,
// only the lanes at a warp or row edge do one extra scalar load (or take the boundary value).
#include <stdlib.h>

#include "xg_common.cuh"
#include "xg_stencil_tile.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarpsPerBlock = kThreads / 32;

template <typename T>
struct PairArgs {
  const T* a;
  const T* b;
  T* out;
  int64_t outer, nb, inner, nx;  // collapsed around axis b; inner = (dims between b and x) * nx
  int op_a, lo_a, bc_a;          // hi_a = 1 - lo_a
  int op_b, lo_b, bc_b;
  T fill_a, fill_b;
  const T* halo_lo;  // optional planes (outer, inner) of B x mb replacing bc_b below row 0 / above row nb - 1
  const T* halo_hi;
  int subtract;
  XgOperand ma, mb, post;  // broadcast operands laid out against the common shape, collapsed around axis b
  int J;
  int64_t nseg, nwc, nunits;
  bool small_units, small_inner;
  XgFastDiv fd_nseg, fd_nwc, fd_nx;  // multiply-high forms (valid with the small_* flags)
};

template <typename T>
__device__ __forceinline__ T apply_rt(int op, T lo_v, T hi_v) {
  switch (op) {
    case XG_OP_DIFF: return xg_apply_op<T, XG_OP_DIFF>(lo_v, hi_v);
    case XG_OP_INTERP: return xg_apply_op<T, XG_OP_INTERP>(lo_v, hi_v);
    case XG_OP_MIN: return xg_apply_op<T, XG_OP_MIN>(lo_v, hi_v);
    default: return xg_apply_op<T, XG_OP_MAX>(lo_v, hi_v);
  }
}

// element offset of a broadcast operand at (outer offset already applied) row j, flat inner index ii
__device__ __forceinline__ int64_t operand_inner_off(const XgOperand& m, int64_t ii) {
  if (m.inner_mode == XG_IM_CONTIG) return ii;
  if (m.inner_mode == XG_IM_GENERIC) return xg_groups_offset(m.inner, ii);
  return 0;
}

// OPS >= 0: both operators known at compile time (OPS = op_a * 4 + op_b), the common diff / interp pairs;
// OPS < 0: operators read from the arguments (min / max combinations)
template <typename T, int OPS>
__device__ __forceinline__ T op_first(const int op_rt, T lo_v, T hi_v) {
  if constexpr (OPS >= 0) return xg_apply_op<T, OPS / 4>(lo_v, hi_v);
  else return apply_rt<T>(op_rt, lo_v, hi_v);
}
template <typename T, int OPS>
__device__ __forceinline__ T op_second(const int op_rt, T lo_v, T hi_v) {
  if constexpr (OPS >= 0) return xg_apply_op<T, OPS % 4>(lo_v, hi_v);
  else return apply_rt<T>(op_rt, lo_v, hi_v);
}

template <typename T, int VEC, bool MET, int U, int OPS>
__global__ void __launch_bounds__(kThreads, 3) k_stencil_pair(const PairArgs<T> p) {
  typedef XgPack<T, VEC> Pack;
  const unsigned FULL = 0xffffffffu;
  const int64_t unit = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (unit >= p.nunits) return;  // warp-uniform
  const int lane = threadIdx.x & 31;
  int64_t wc, t, seg, o;
  xg_divmod(unit, p.nwc, p.fd_nwc, p.small_units, t, wc);
  xg_divmod(t, p.nseg, p.fd_nseg, p.small_units, o, seg);
  int64_t i = (wc * 32 + lane) * VEC;
  const bool valid = i < p.inner;
  if (!valid) i = p.inner - VEC;  // spare lanes shadow the last vector: all 32 lanes stay in the shuffles
  int64_t row_i, x0;
  xg_divmod(i, p.nx, p.fd_nx, p.small_inner, row_i, x0);
  const bool row_first = x0 == 0, row_last = x0 + VEC == p.nx;

  const int64_t j0 = seg * p.J;
  const int64_t j1 = (j0 + p.J < p.nb) ? (j0 + p.J) : p.nb;
  const T* abase = p.a + o * p.nb * p.inner + i;
  const T* bbase = p.b + o * p.nb * p.inner + i;
  T* obase = p.out + o * p.nb * p.inner + i;
  const bool has_ma = MET && p.ma.ptr != nullptr, has_mb = MET && p.mb.ptr != nullptr;
  const bool has_post = MET && p.post.ptr != nullptr;
  XgOperandView<T, VEC> ma_v, mb_v, post_v;
  int64_t ma_outer = 0;
  if (MET) {
    if (has_ma) {
      ma_outer = xg_groups_offset(p.ma.outer, o);
      ma_v = xg_operand_view<T, VEC>(p.ma, ma_outer, i);
    }
    if (has_mb) mb_v = xg_operand_view<T, VEC>(p.mb, xg_groups_offset(p.mb.outer, o), i);
    if (has_post) post_v = xg_operand_view<T, VEC>(p.post, xg_groups_offset(p.post.outer, o), i);
  }
  // A x ma at one cell of row j (flat inner index ii): the warp-edge neighbour and the periodic wrap
  auto scalarA = [&](int64_t j, int64_t ii) -> T {
    T v = __ldg(p.a + (o * p.nb + j) * p.inner + ii);
    if (has_ma)
      v = v * __ldg(reinterpret_cast<const T*>(p.ma.ptr) + ma_outer + j * p.ma.axis_stride +
                    operand_inner_off(p.ma, ii));
    return v;
  };
  // A x ma, row j (the thread's own vector)
  auto loadA = [&](int64_t j) -> Pack {
    Pack va = xg_ld_stream<T, VEC>(abase + j * p.inner);
    if (has_ma) {
      const Pack m = xg_ld_view<T, VEC>(ma_v, j * p.ma.axis_stride);
#pragma unroll
      for (int k = 0; k < VEC; ++k) va.v[k] = va.v[k] * m.v[k];
    }
    return va;
  };
  // the stencil along x on a loaded row: neighbour from the adjacent lane, the warp / row edges on their own
  auto termA = [&](int64_t j, const Pack& va) -> Pack {
    Pack r;
    if (p.lo_a) {  // out[x] = OP(P[x-1], P[x])
      T left = __shfl_up_sync(FULL, va.v[VEC - 1], 1);
      if (row_first) {
        if (p.bc_a == XG_BC_FILL) left = p.fill_a;
        else if (p.bc_a == XG_BC_PERIODIC) left = scalarA(j, i + p.nx - 1);
        else left = va.v[0];  // extend
      } else if (lane == 0) {
        left = scalarA(j, i - 1);
      }
#pragma unroll
      for (int k = 0; k < VEC; ++k) r.v[k] = op_first<T, OPS>(p.op_a, k == 0 ? left : va.v[k > 0 ? k - 1 : 0], va.v[k]);
    } else {  // out[x] = OP(P[x], P[x+1])
      T right = __shfl_down_sync(FULL, va.v[0], 1);
      if (row_last) {
        if (p.bc_a == XG_BC_FILL) right = p.fill_a;
        else if (p.bc_a == XG_BC_PERIODIC) right = scalarA(j, i + VEC - p.nx);
        else right = va.v[VEC - 1];
      } else if (lane == 31) {
        right = scalarA(j, i + VEC);
      }
#pragma unroll
      for (int k = 0; k < VEC; ++k)
        r.v[k] = op_first<T, OPS>(p.op_a, va.v[k], k == VEC - 1 ? right : va.v[k < VEC - 1 ? k + 1 : k]);
    }
    return r;
  };
  // B x mb, row s of the source (0 <= s < nb)
  auto loadB = [&](int64_t s) -> Pack {
    Pack v = xg_ld_stream<T, VEC>(bbase + s * p.inner);
    if (has_mb) {
      const Pack m = xg_ld_view<T, VEC>(mb_v, s * p.mb.axis_stride);
#pragma unroll
      for (int k = 0; k < VEC; ++k) v.v[k] = v.v[k] * m.v[k];
    }
    return v;
  };
  // padded row k of B (k in [0, nb]): source row k - lo_b, with the halo plane or the boundary rule at the two ends
  auto padB = [&](int64_t k) -> Pack {
    const int64_t s = k - p.lo_b;
    if (s >= 0 && s < p.nb) return loadB(s);
    const T* halo = s < 0 ? p.halo_lo : p.halo_hi;
    if (halo) return xg_ld_cached<T, VEC>(halo + o * p.inner + i);
    if (p.bc_b == XG_BC_FILL) {
      Pack r;
#pragma unroll
      for (int q = 0; q < VEC; ++q) r.v[q] = p.fill_b;
      return r;
    }
    if (p.bc_b == XG_BC_PERIODIC) return loadB(s < 0 ? s + p.nb : s - p.nb);
    return loadB(s < 0 ? 0 : p.nb - 1);
  };

  auto emit = [&](int64_t j, const Pack& prev_b, const Pack& cur_b, const Pack& va) {
    const Pack ta = termA(j, va);
    Pack r;
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      const T tb = op_second<T, OPS>(p.op_b, prev_b.v[k], cur_b.v[k]);
      r.v[k] = p.subtract == 0 ? ta.v[k] + tb : (p.subtract == 1 ? ta.v[k] - tb : tb - ta.v[k]);
    }
    if (has_post) {
      const Pack m = xg_ld_view<T, VEC>(post_v, j * p.post.axis_stride);
#pragma unroll
      for (int k = 0; k < VEC; ++k) r.v[k] = r.v[k] / m.v[k];
    }
    if (valid) xg_st_stream<T, VEC>(obase + j * p.inner, r);
  };
  Pack prev = padB(j0);
  // rows whose upper B operand is an ordinary source row: U rows of both fields in flight per thread
  const int64_t jm = (j1 < p.nb + p.lo_b - 1) ? j1 : (p.nb + p.lo_b - 1);
  int64_t j = j0;
  for (; j + U <= jm; j += U) {
    Pack cb[U], va[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      cb[u] = loadB(j + u + 1 - p.lo_b);
      va[u] = loadA(j + u);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      emit(j + u, prev, cb[u], va[u]);
      prev = cb[u];
    }
  }
#pragma unroll 1
  for (; j < j1; ++j) {
    const Pack cur = padB(j + 1);
    emit(j, prev, cur, loadA(j));
    prev = cur;
  }
}

template <typename T, int VEC>
int launch_pair(PairArgs<T>& p, cudaStream_t st) {
  const int64_t nvec = xg_ceil_div(p.inner, VEC);
  p.nwc = xg_ceil_div(nvec, 32);
  p.J = (p.nb <= 96) ? (int)p.nb : 32;
  p.nseg = xg_ceil_div(p.nb, p.J);
  p.nunits = p.outer * p.nseg * p.nwc;
  p.small_units = p.nunits < (1ll << 31);
  p.small_inner = p.inner < (1ll << 31);
  p.fd_nseg = xg_fastdiv_make(p.small_units ? p.nseg : 1);
  p.fd_nwc = xg_fastdiv_make(p.small_units ? p.nwc : 1);
  p.fd_nx = xg_fastdiv_make(p.small_inner ? p.nx : 1);
  const int64_t blocks = xg_ceil_div(p.nunits, kWarpsPerBlock);
  if (blocks > 0x7fffffffLL) return xg_fail(XG_EINVAL, "xg_stencil_pair: grid too large");
  const bool met = p.ma.ptr || p.mb.ptr || p.post.ptr;
  const bool ct = p.op_a <= XG_OP_INTERP && p.op_b <= XG_OP_INTERP;  // diff / interp pairs: compile-time operators
  const int ops = ct ? p.op_a * 4 + p.op_b : -1;
#define XG_PAIR_LAUNCH(MET_, U_, OPS_) k_stencil_pair<T, VEC, MET_, U_, OPS_><<<(unsigned)blocks, kThreads, 0, st>>>(p)
#define XG_PAIR_OPS(MET_, U_)                                         \
  switch (ops) {                                                      \
    case XG_OP_DIFF * 4 + XG_OP_DIFF: XG_PAIR_LAUNCH(MET_, U_, XG_OP_DIFF * 4 + XG_OP_DIFF); break;       \
    case XG_OP_DIFF * 4 + XG_OP_INTERP: XG_PAIR_LAUNCH(MET_, U_, XG_OP_DIFF * 4 + XG_OP_INTERP); break;   \
    case XG_OP_INTERP * 4 + XG_OP_DIFF: XG_PAIR_LAUNCH(MET_, U_, XG_OP_INTERP * 4 + XG_OP_DIFF); break;   \
    case XG_OP_INTERP * 4 + XG_OP_INTERP: XG_PAIR_LAUNCH(MET_, U_, XG_OP_INTERP * 4 + XG_OP_INTERP); break; \
    default: XG_PAIR_LAUNCH(MET_, U_, -1); break;                     \
  }
  if (met) {
    XG_PAIR_OPS(true, 2)
  } else {
    XG_PAIR_OPS(false, 4)
  }
#undef XG_PAIR_OPS
#undef XG_PAIR_LAUNCH
  return xg_check_launch("xg_stencil_pair");
}

template <typename T>
int pair_typed(const void* a, const void* b, void* out, int ndim, const int64_t* shape, int op_a, int lo_a, int bc_a,
               double fill_a, const void* pre_a, const int64_t* pre_a_strides, int axis_b, int op_b, int lo_b, int bc_b,
               double fill_b, const void* pre_b, const int64_t* pre_b_strides, int subtract, const void* post,
               const int64_t* post_strides, const void* halo_lo_b, const void* halo_hi_b, cudaStream_t st) {
  constexpr int VEC = XgVecWidth<T>::value;
  XgView v;
  int rc = xg_collapse_view(ndim, shape, axis_b, &v);
  if (rc) return rc;
  PairArgs<T> p;
  p.a = static_cast<const T*>(a);
  p.b = static_cast<const T*>(b);
  p.out = static_cast<T*>(out);
  p.outer = v.outer;
  p.nb = v.n;
  p.inner = v.inner;
  p.nx = shape[ndim - 1];
  p.op_a = op_a;
  p.lo_a = lo_a;
  p.bc_a = bc_a;
  p.op_b = op_b;
  p.lo_b = lo_b;
  p.bc_b = bc_b;
  p.fill_a = static_cast<T>(fill_a);
  p.fill_b = static_cast<T>(fill_b);
  p.halo_lo = static_cast<const T*>(halo_lo_b);
  p.halo_hi = static_cast<const T*>(halo_hi_b);
  p.subtract = subtract;
  if (v.n == 0 || p.nx == 0) return xg_fail(XG_EINVAL, "xg_stencil_pair: empty operated axis");
  if (v.outer == 0 || v.inner == 0) return XG_OK;
  bool vec_ok = p.nx % VEC == 0 &&
                (((uintptr_t)a | (uintptr_t)b | (uintptr_t)out | (uintptr_t)halo_lo_b | (uintptr_t)halo_hi_b) % 16 == 0);
  const int vec = vec_ok ? VEC : 1;
  rc = xg_make_operand(pre_a, pre_a_strides, ndim, shape, axis_b, vec, sizeof(T), &p.ma, "xg_stencil_pair(pre_a)");
  if (rc) return rc;
  rc = xg_make_operand(pre_b, pre_b_strides, ndim, shape, axis_b, vec, sizeof(T), &p.mb, "xg_stencil_pair(pre_b)");
  if (rc) return rc;
  rc = xg_make_operand(post, post_strides, ndim, shape, axis_b, vec, sizeof(T), &p.post, "xg_stencil_pair(post)");
  if (rc) return rc;
  if (vec_ok && p.inner == p.nx) {
    // axis b is the dim next to x and (typically) the metrics are shared between levels: the TMA-staged tile kernel
    XgTileSpec<T> ts;
    ts.Zn = p.outer;
    ts.Pb = ts.Po = p.nb;
    ts.n = p.nx;
    ts.f_sp = p.nx;
    ts.b_sz = ts.o_sz = p.nb * p.nx;
    ts.a = p.a;
    ts.op_a = p.op_a;
    ts.lo_a = p.lo_a;
    ts.bc_a = p.bc_a;
    ts.fill_a = p.fill_a;
    ts.b = p.b;
    ts.op_b = p.op_b;
    ts.lo_b = p.lo_b;
    ts.hi_b = 1 - p.lo_b;
    ts.bc_b = p.bc_b;
    ts.fill_b = p.fill_b;
    ts.halo_lo = p.halo_lo;
    ts.halo_hi = p.halo_hi;
    ts.subtract = p.subtract;
    ts.out = p.out;
    if (xg_tile_operand_from<T>(p.ma, p.outer, p.inner, &ts.ma) && xg_tile_operand_from<T>(p.mb, p.outer, p.inner, &ts.mb) &&
        xg_tile_operand_from<T>(p.post, p.outer, p.inner, &ts.post)) {
      bool launched = false;
      rc = xg_tile_stencil<T>(ts, st, &launched, "xg_stencil_pair(tile_tma)");
      if (rc || launched) return rc;
    }
  }
  if (vec_ok && xg_vec_view_ok(p.ma) && xg_vec_view_ok(p.mb) && xg_vec_view_ok(p.post))
    return launch_pair<T, VEC>(p, st);
  return launch_pair<T, 1>(p, st);
}

// the checks and dtype dispatch of both entry points
int pair_entry(int dtype, const void* a, const void* b, void* out, int ndim, const int64_t* shape, int op_a, int lo_a,
               int hi_a, int bc_a, double fill_a, const void* pre_a, const int64_t* pre_a_strides, int axis_b, int op_b,
               int lo_b, int hi_b, int bc_b, double fill_b, const void* pre_b, const int64_t* pre_b_strides,
               int subtract, const void* post, const int64_t* post_strides, const void* halo_lo_b,
               const void* halo_hi_b, void* stream) {
  if (!a || !b || !out || !shape) return xg_fail(XG_EINVAL, "xg_stencil_pair: null pointer");
  if (ndim < 2 || ndim > XG_MAX_NDIM) return xg_fail(XG_EINVAL, "xg_stencil_pair: needs 2 <= ndim <= XG_MAX_NDIM");
  if (axis_b < 0 || axis_b >= ndim - 1)
    return xg_fail(XG_EINVAL, "xg_stencil_pair: axis_b must be a dimension other than the innermost one");
  if (lo_a < 0 || hi_a < 0 || lo_a + hi_a != 1 || lo_b < 0 || hi_b < 0 || lo_b + hi_b != 1)
    return xg_fail(XG_ENOTIMPL, "xg_stencil_pair: both stencils must be length preserving (lo + hi == 1)");
  for (int bc : {bc_a, bc_b})
    if (bc < XG_BC_PERIODIC || bc > XG_BC_EXTEND)
      return xg_fail(XG_EINVAL, "xg_stencil_pair: boundary must be periodic, fill or extend");
  for (int op : {op_a, op_b})
    if (op < XG_OP_DIFF || op > XG_OP_MAX) return xg_fail(XG_EINVAL, "xg_stencil_pair: unknown op");
  if ((pre_a && !pre_a_strides) || (pre_b && !pre_b_strides) || (post && !post_strides))
    return xg_fail(XG_EINVAL, "xg_stencil_pair: metric strides missing");
  if (subtract < 0 || subtract > 2) return xg_fail(XG_EINVAL, "xg_stencil_pair: subtract must be 0, 1 or 2");
  if (a == out || b == out) return xg_fail(XG_EINVAL, "xg_stencil_pair: in-place operation is not supported");
  if ((halo_lo_b && halo_lo_b == out) || (halo_hi_b && halo_hi_b == out))
    return xg_fail(XG_EINVAL, "xg_stencil_pair: a halo plane may not be the output");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == XG_F32)
    return pair_typed<float>(a, b, out, ndim, shape, op_a, lo_a, bc_a, fill_a, pre_a, pre_a_strides, axis_b, op_b, lo_b,
                             bc_b, fill_b, pre_b, pre_b_strides, subtract, post, post_strides, halo_lo_b, halo_hi_b, st);
  if (dtype == XG_F64)
    return pair_typed<double>(a, b, out, ndim, shape, op_a, lo_a, bc_a, fill_a, pre_a, pre_a_strides, axis_b, op_b, lo_b,
                              bc_b, fill_b, pre_b, pre_b_strides, subtract, post, post_strides, halo_lo_b, halo_hi_b, st);
  return xg_fail(XG_EINVAL, "xg_stencil_pair: dtype must be XG_F32 or XG_F64");
}

}  // namespace

extern "C" int xg_stencil_pair(int dtype, const void* a, const void* b, void* out, int ndim, const int64_t* shape,
                               int op_a, int lo_a, int hi_a, int bc_a, double fill_a, const void* pre_a,
                               const int64_t* pre_a_strides, int axis_b, int op_b, int lo_b, int hi_b, int bc_b,
                               double fill_b, const void* pre_b, const int64_t* pre_b_strides, int subtract,
                               const void* post, const int64_t* post_strides, void* stream) {
  return pair_entry(dtype, a, b, out, ndim, shape, op_a, lo_a, hi_a, bc_a, fill_a, pre_a, pre_a_strides, axis_b, op_b,
                    lo_b, hi_b, bc_b, fill_b, pre_b, pre_b_strides, subtract, post, post_strides, nullptr, nullptr,
                    stream);
}

extern "C" int xg_stencil_pair_halo(int dtype, const void* a, const void* b, void* out, int ndim, const int64_t* shape,
                                    int op_a, int lo_a, int hi_a, int bc_a, double fill_a, const void* pre_a,
                                    const int64_t* pre_a_strides, int axis_b, int op_b, int lo_b, int hi_b, int bc_b,
                                    double fill_b, const void* pre_b, const int64_t* pre_b_strides, int subtract,
                                    const void* post, const int64_t* post_strides, const void* halo_lo_b,
                                    const void* halo_hi_b, void* stream) {
  return pair_entry(dtype, a, b, out, ndim, shape, op_a, lo_a, hi_a, bc_a, fill_a, pre_a, pre_a_strides, axis_b, op_b,
                    lo_b, hi_b, bc_b, fill_b, pre_b, pre_b_strides, subtract, post, post_strides, halo_lo_b, halo_hi_b,
                    stream);
}
