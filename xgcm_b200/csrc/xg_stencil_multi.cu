// xg_stencil_multi — 2 or 3 single-axis stencils fused into ONE pass over HBM.
//
// `Grid.interp(da, ['X', 'Y'])` (and diff / min / max over several axes) is, in the reference,
// one full pad + ufunc pass per axis (xgcm/grid.py:798-832; its own TODO notes the waste).  Here
// the chain  op_K(pad_K( ... op_1(pad_1(a)) ... ))  is evaluated per output cell straight from the
// input: 2^K neighbour loads (absorbed by L1 / L2: DRAM sees one read and one write per cell),
// every intermediate rounded to the field dtype exactly where the sequential passes would round,
// each axis with its own halo rule applied to ITS intermediate (fill is a constant of that level,
// periodic / extend re-index the source).  Bit-identical to K consecutive xg_stencil2 calls at
// 1/K of their traffic.
//
// Work split: a block owns one output row along the innermost dim; threads take 16-byte vectors
// of it.  The recursion is resolved at compile time (K ops, position LAST of the op acting on the
// innermost dim, or -1): row ops combine two windows of W values; the innermost op consumes a
// window of W + 1 consecutive source positions (one aligned vector + one neighbour element).
//
// Roofline: HBM, 2 * sizeof(T) bytes per output cell.
#include <stdlib.h>

#include "xg_common.cuh"
#include "xg_stencil_tile.cuh"

namespace {

constexpr int kMaxAx = 3;
constexpr int kMaxGroups = 2 * kMaxAx;  // row groups (everything but the innermost group)

template <typename T>
struct AxisOp {
  int op, lo, hi, bc;
  T fill;
  int64_t n;          // input (and intermediate) length along this axis
  int64_t in_stride;  // element stride of this axis in the INPUT (1 for the innermost dim)
};

template <typename T>
struct MultiArgs {
  const T* in;
  T* out;
  AxisOp<T> ax[kMaxAx];  // in application order
  int nrow_groups;
  int64_t row_size[kMaxGroups];        // extent in the OUTPUT, outermost first
  int64_t row_in_stride[kMaxGroups];   // input element stride (non-operated groups)
  int64_t row_out_stride[kMaxGroups];  // output element stride
  int row_axis[kMaxGroups];            // application index of the operated axis, or -1
  int64_t last_n_out;                  // output extent of the innermost group
  // the march axis (last applied row-axis op): not part of the row groups
  int64_t march_n_out, march_out_stride;
  int J;
  int64_t nseg;
};

template <typename T>
__device__ __forceinline__ T apply_rt(int op, T a, T b) {
  switch (op) {
    case XG_OP_DIFF: return xg_apply_op<T, XG_OP_DIFF>(a, b);
    case XG_OP_INTERP: return xg_apply_op<T, XG_OP_INTERP>(a, b);
    case XG_OP_MIN: return xg_apply_op<T, XG_OP_MIN>(a, b);
    default: return xg_apply_op<T, XG_OP_MAX>(a, b);
  }
}

// source index of padded position idx along an axis; false when the halo is the fill constant
template <typename T>
__device__ __forceinline__ bool resolve(const AxisOp<T>& a, int64_t idx, int64_t& s) {
  s = idx - a.lo;
  if (s < 0) {
    if (a.bc == XG_BC_FILL) { s = 0; return false; }
    s = (a.bc == XG_BC_PERIODIC) ? s + a.n : 0;
  } else if (s >= a.n) {
    if (a.bc == XG_BC_FILL) { s = a.n - 1; return false; }
    s = (a.bc == XG_BC_PERIODIC) ? s - a.n : a.n - 1;
  }
  return true;
}

template <typename T, int W>
struct Win {
  T v[W];
};

// W consecutive input elements along the innermost dim starting at source position xs (which may
// be -1, and xs + W - 1 may be n, only when the innermost dim is operated: those ends follow the
// halo rule of that op; a fill halo is patched by the caller, here it just reads a valid cell).
template <typename T, int VEC, int W, int LAST>
__device__ __forceinline__ Win<T, W> load_window(const MultiArgs<T>& a, int64_t off, int64_t xs) {
  Win<T, W> r;
  const T* p = a.in + off;
  if constexpr (LAST < 0) {
    static_assert(W == VEC, "window == vector when the innermost dim is not operated");
    XgPack<T, VEC> pk = xg_ld_cached<T, VEC>(p + xs);
#pragma unroll
    for (int q = 0; q < VEC; ++q) r.v[q] = pk.v[q];
  } else {
    const AxisOp<T>& ax = a.ax[LAST];
    auto scalar_at = [&](int64_t pos) -> T {
      if (pos < 0) pos = (ax.bc == XG_BC_PERIODIC) ? pos + ax.n : 0;
      else if (pos >= ax.n) pos = (ax.bc == XG_BC_PERIODIC) ? pos - ax.n : ax.n - 1;
      return __ldg(p + pos);
    };
    if constexpr (VEC > 1 && W == VEC + 1) {
      // exactly one aligned vector plus one neighbour: xs = x0 - lo with x0 a multiple of VEC
      const bool lead = (xs & (VEC - 1)) != 0;  // lo == 1: the neighbour comes first
      const int64_t xv = lead ? xs + 1 : xs;
      XgPack<T, VEC> pk = xg_ld_cached<T, VEC>(p + xv);
      const T extra = scalar_at(lead ? xs : xs + VEC);
      // static indices only (a runtime-indexed window would live in local memory)
#pragma unroll
      for (int q = 0; q <= VEC; ++q) {
        const T from_lead = (q == 0) ? extra : pk.v[q > 0 ? q - 1 : 0];
        const T from_tail = (q < VEC) ? pk.v[q < VEC ? q : 0] : extra;
        r.v[q] = lead ? from_lead : from_tail;
      }
    } else {
#pragma unroll
      for (int q = 0; q < W; ++q) r.v[q] = scalar_at(xs + q);
    }
  }
  return r;
}

// Window of W values of the intermediate after the first k ops, at row coordinates j (axes < k
// in their output space; axes >= k already folded into `off`), innermost coordinate x.
template <typename T, int VEC, int K, int LAST, int OP>
struct Eval {
  template <int k, int W>
  static __device__ __forceinline__ Win<T, W> run(const MultiArgs<T>& a, const int64_t* j, int64_t off,
                                                   int64_t x) {
    if constexpr (k == 0) {
      return load_window<T, VEC, W, LAST>(a, off, x);
    } else {
      constexpr int m = k - 1;  // the op applied at this level
      const AxisOp<T>& ax = a.ax[m];
      Win<T, W> r;
      if constexpr (m == LAST) {
        // innermost op: padded positions x .. x+W  <-  sources x-lo .. x-lo+W
        const int64_t xs = x - ax.lo;
        Win<T, W + 1> w = run<k - 1, W + 1>(a, j, off, xs);
        if (ax.bc == XG_BC_FILL) {  // the ends of the window may be halo cells of THIS level
          if (xs < 0) w.v[0] = ax.fill;
          if (xs + W >= ax.n) w.v[W] = ax.fill;
        }
#pragma unroll
        for (int q = 0; q < W; ++q) r.v[q] = xg_apply_op<T, OP>(w.v[q], w.v[q + 1]);
      } else {
        int64_t s0, s1;
        const bool ok0 = resolve(ax, j[m], s0);  // block-uniform: j is this block's row
        const bool ok1 = resolve(ax, j[m] + 1, s1);
        // branch-free: a fill halo still reads a (clamped, valid) row and is replaced afterwards,
        // so every load of the recursion can be issued before the first value is consumed
        Win<T, W> lo_v = run<k - 1, W>(a, j, off + s0 * ax.in_stride, x);
        Win<T, W> hi_v = run<k - 1, W>(a, j, off + s1 * ax.in_stride, x);
#pragma unroll
        for (int q = 0; q < W; ++q)
          r.v[q] = xg_apply_op<T, OP>(ok0 ? lo_v.v[q] : ax.fill, ok1 ? hi_v.v[q] : ax.fill);
      }
      return r;
    }
  }
};

// MARCH = application index of the LAST applied row-axis op.  A thread owns one vector position of
// the innermost dim and walks J consecutive output coordinates of that axis: the lower operand of
// step j+1 is the upper operand of step j (consecutive padded positions), so it stays in
// registers and only ONE evaluation of the levels below is needed per output — for
// interp(['X','Y']) that is one 16-byte load plus one neighbour element per 16-byte store.  The
// only level that can sit above MARCH is the op on the innermost dim (elementwise on the window).
template <typename T, int VEC, int K, int LAST, int MARCH, int OP>
__global__ void __launch_bounds__(256, 4) k_stencil_multi(const MultiArgs<T> a) {
  constexpr bool kInnerAbove = (LAST > MARCH);
  constexpr int WM = kInnerAbove ? VEC + 1 : VEC;  // window width at the march level
  constexpr int U = 4;
  // With row ops below the march level the select form wins; the plain X,Y case has a single
  // load per step and was faster with the branch.
  constexpr bool kBranchFreeMarch = !(K == 2 && LAST >= 0);
  // this block: a segment of the march axis at fixed coordinates of every other row group
  int64_t unit = blockIdx.x;
  const int64_t seg = unit % a.nseg;
  unit /= a.nseg;
  int64_t j0 = 0, j1 = 0, j2 = 0;  // separate scalars: a runtime-indexed array would live in local memory
  int64_t off_in = 0, off_out = 0;
#pragma unroll
  for (int g = kMaxGroups - 1; g >= 0; --g) {
    if (g < a.nrow_groups) {
      const int64_t q = unit / a.row_size[g];
      const int64_t c = unit - q * a.row_size[g];
      unit = q;
      off_out += c * a.row_out_stride[g];
      const int ra = a.row_axis[g];
      if (ra == 0) j0 = c;
      else if (ra == 1) j1 = c;
      else if (ra == 2) j2 = c;
      else off_in += c * a.row_in_stride[g];
    }
  }
  const int64_t j[kMaxAx] = {j0, j1, j2};
  const AxisOp<T>& mx = a.ax[MARCH];
  const int64_t jm0 = seg * a.J;
  const int64_t jm1 = (jm0 + a.J < a.march_n_out) ? jm0 + a.J : a.march_n_out;
  const int64_t nvec = (a.last_n_out + VEC - 1) / VEC;  // exact when VEC > 1 (host guarantees it)

  for (int64_t v = threadIdx.x; v < nvec; v += blockDim.x) {
    const int64_t x0 = v * VEC;
    int64_t xw = x0;  // innermost coordinate of the window at the march level
    if constexpr (kInnerAbove) xw = x0 - a.ax[LAST].lo;
    // padded intermediate below the march op at padded position p of the march axis
    auto below = [&](int64_t p) -> Win<T, WM> {
      int64_t sidx;
      const bool ok = resolve(mx, p, sidx);
      if constexpr (kBranchFreeMarch) {
        // a fill halo reads the clamped row and is replaced, so the U loads batch ahead of use
        Win<T, WM> r = Eval<T, VEC, K, LAST, OP>::template run<MARCH, WM>(a, j, off_in + sidx * mx.in_stride, xw);
#pragma unroll
        for (int q = 0; q < WM; ++q) r.v[q] = ok ? r.v[q] : mx.fill;
        return r;
      } else {
        if (ok) return Eval<T, VEC, K, LAST, OP>::template run<MARCH, WM>(a, j, off_in + sidx * mx.in_stride, xw);
        Win<T, WM> r;
#pragma unroll
        for (int q = 0; q < WM; ++q) r.v[q] = mx.fill;
        return r;
      }
    };
    auto finish = [&](int64_t jm, const Win<T, WM>& lo_w, const Win<T, WM>& hi_w) {
      Win<T, WM> r;
#pragma unroll
      for (int q = 0; q < WM; ++q) r.v[q] = xg_apply_op<T, OP>(lo_w.v[q], hi_w.v[q]);
      XgPack<T, VEC> res;
      if constexpr (kInnerAbove) {
        const AxisOp<T>& ix = a.ax[LAST];
        if (ix.bc == XG_BC_FILL) {  // halo cells of the innermost op's own level
          if (xw < 0) r.v[0] = ix.fill;
          if (xw + VEC >= ix.n) r.v[VEC] = ix.fill;
        }
#pragma unroll
        for (int q = 0; q < VEC; ++q) res.v[q] = xg_apply_op<T, OP>(r.v[q], r.v[q + 1]);
      } else {
#pragma unroll
        for (int q = 0; q < VEC; ++q) res.v[q] = r.v[q];
      }
      xg_st_stream<T, VEC>(a.out + off_out + jm * a.march_out_stride + x0, res);
    };
    Win<T, WM> prev = below(jm0);
    int64_t jm = jm0;
    for (; jm + U <= jm1; jm += U) {
      Win<T, WM> cur[U];
#pragma unroll
      for (int u = 0; u < U; ++u) cur[u] = below(jm + u + 1);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        finish(jm + u, prev, cur[u]);
        prev = cur[u];
      }
    }
    for (; jm < jm1; ++jm) {
      Win<T, WM> cur = below(jm + 1);
      finish(jm, prev, cur);
      prev = cur;
    }
  }
}

template <typename T, int VEC, int K, int LAST, int MARCH>
int launch_op(int op, const MultiArgs<T>& a, int64_t nblocks, int threads, cudaStream_t st) {
  const unsigned grid = (unsigned)nblocks;
  switch (op) {
    case XG_OP_DIFF: k_stencil_multi<T, VEC, K, LAST, MARCH, XG_OP_DIFF><<<grid, threads, 0, st>>>(a); break;
    case XG_OP_INTERP: k_stencil_multi<T, VEC, K, LAST, MARCH, XG_OP_INTERP><<<grid, threads, 0, st>>>(a); break;
    case XG_OP_MIN: k_stencil_multi<T, VEC, K, LAST, MARCH, XG_OP_MIN><<<grid, threads, 0, st>>>(a); break;
    default: k_stencil_multi<T, VEC, K, LAST, MARCH, XG_OP_MAX><<<grid, threads, 0, st>>>(a); break;
  }
  return xg_check_launch("xg_stencil_multi");
}

template <typename T, int VEC, int K, int LAST>
int launch_march(int march, const MultiArgs<T>& a, int64_t nblocks, int threads, cudaStream_t st) {
  const int op = a.ax[0].op;  // the fused kernel applies one operator along all axes
  // multi_typed marches along the highest application index other than LAST; only that MARCH is
  // instantiated for each (K, LAST)
  constexpr int MARCH = LAST == K - 1 ? K - 2 : K - 1;
  if (march != MARCH) return xg_fail(XG_EINVAL, "xg_stencil_multi: bad march axis");
  return launch_op<T, VEC, K, LAST, MARCH>(op, a, nblocks, threads, st);
}

template <typename T, int VEC, int K>
int launch_last(int last, int march, const MultiArgs<T>& a, int64_t nblocks, int threads, cudaStream_t st) {
  switch (last) {
    case -1: return launch_march<T, VEC, K, -1>(march, a, nblocks, threads, st);
    case 0: return launch_march<T, VEC, K, 0>(march, a, nblocks, threads, st);
    case 1: return launch_march<T, VEC, K, 1>(march, a, nblocks, threads, st);
    case 2:
      if constexpr (K == 3) return launch_march<T, VEC, K, 2>(march, a, nblocks, threads, st);
    default: return xg_fail(XG_EINVAL, "xg_stencil_multi: bad innermost op index");
  }
}

template <typename T>
int multi_typed(const void* in, void* out, int ndim, const int64_t* shape, int naxes, const int* axes,
                const int* ops, const int* lo, const int* hi, const int* bc, const double* fill,
                cudaStream_t st) {
  constexpr int VEC = XgVecWidth<T>::value;
  MultiArgs<T> a;
  a.in = static_cast<const T*>(in);
  a.out = static_cast<T*>(out);
  int64_t out_shape[XG_MAX_NDIM], in_stride[XG_MAX_NDIM], out_stride[XG_MAX_NDIM];
  int app_index[XG_MAX_NDIM];
  for (int d = 0; d < ndim; ++d) {
    out_shape[d] = shape[d];
    app_index[d] = -1;
  }
  for (int k = 0; k < naxes; ++k) {
    const int d = axes[k];
    if (d < 0 || d >= ndim) return xg_fail(XG_EINVAL, "xg_stencil_multi: axis out of range");
    if (app_index[d] >= 0) return xg_fail(XG_EINVAL, "xg_stencil_multi: an axis may appear only once");
    if (lo[k] < 0 || lo[k] > 1 || hi[k] < 0 || hi[k] > 1)
      return xg_fail(XG_EINVAL, "xg_stencil_multi: halo widths must be 0 or 1");
    if ((lo[k] || hi[k]) && (bc[k] < XG_BC_PERIODIC || bc[k] > XG_BC_EXTEND))
      return xg_fail(XG_EINVAL,
                     "xg_stencil_multi: each padded axis needs a periodic / fill / extend boundary");
    if (shape[d] == 0) return xg_fail(XG_EINVAL, "xg_stencil_multi: empty operated axis");
    app_index[d] = k;
    out_shape[d] = shape[d] + lo[k] + hi[k] - 1;
  }
  int64_t total_out = 1;
  {
    int64_t si = 1, so = 1;
    for (int d = ndim - 1; d >= 0; --d) {
      in_stride[d] = si;
      out_stride[d] = so;
      si *= shape[d];
      so *= out_shape[d];
      total_out *= out_shape[d];
    }
  }
  if (total_out == 0) return XG_OK;
  for (int k = 0; k < naxes; ++k) {
    const int d = axes[k];
    a.ax[k].op = ops[k];
    a.ax[k].lo = lo[k];
    a.ax[k].hi = hi[k];
    a.ax[k].bc = bc[k];
    a.ax[k].fill = static_cast<T>(fill[k]);
    a.ax[k].n = shape[d];
    a.ax[k].in_stride = in_stride[d];
  }
  // the common chain — innermost axis first over the last two / three dims, every op length preserving —
  // has a TMA-staged form (xg_stencil_multi_tma.cu); everything else runs the kernel below
  {
    bool ok = ndim >= 2;
    for (int k = 0; k < naxes && ok; ++k) {
      ok = lo[k] + hi[k] == 1 && axes[k] >= ndim - 3 && (k == 0 || axes[k] < axes[k - 1]);
    }
    if (ok) {
      XgMultiTileSpec<T> ms;
      ms.in = a.in;
      ms.out = a.out;
      ms.op = ops[0];
      for (int q = 0; q < 3; ++q) {
        ms.has[q] = 0;
        ms.lo[q] = 0;
        ms.bc[q] = XG_BC_FILL;
        ms.fill[q] = T(0);
      }
      for (int k = 0; k < naxes; ++k) {
        const int q = ndim - 1 - axes[k];  // 0 = x, 1 = rows, 2 = levels
        ms.has[q] = 1;
        ms.lo[q] = lo[k];
        ms.bc[q] = bc[k];
        ms.fill[q] = static_cast<T>(fill[k]);
      }
      ms.n = shape[ndim - 1];
      ms.P = shape[ndim - 2];
      ms.L = 1;
      for (int d = 0; d < ndim - 2; ++d) ms.L *= shape[d];
      // an operated level axis must be the only level dim (the dims before it have extent 1)
      if (ms.has[2]) ok = ndim >= 3 && ms.L == shape[ndim - 3];
      if (ok) {
        bool launched = false;
        const int rc = xg_multi_tile<T>(ms, st, &launched);
        if (rc || launched) return rc;
      }
    }
  }
  // innermost group: the last dim if it is operated, else the run of trailing non-operated dims
  int last = app_index[ndim - 1];
  int d_end = ndim - 1;  // dims [0, d_end) form the row space
  int64_t last_n_out = out_shape[ndim - 1];
  if (last < 0) {
    while (d_end > 0 && app_index[d_end - 1] < 0) {
      --d_end;
      last_n_out *= out_shape[d_end];
    }
  }
  a.last_n_out = last_n_out;
  // the march axis: the last applied op that is not on the innermost dim
  int march = -1;
  for (int k = naxes - 1; k >= 0; --k)
    if (k != last) { march = k; break; }
  const int march_dim = axes[march];
  a.march_n_out = out_shape[march_dim];
  a.march_out_stride = out_stride[march_dim];
  a.J = a.march_n_out <= 16 ? (int)a.march_n_out : 16;  // flat optimum of a sweep (not repeated on H100)
  if (const char* e = getenv("XG_MULTI_J")) {  // tuning knob (benchmarks only)
    const int tj = atoi(e);
    if (tj > 0) a.J = tj < a.march_n_out ? tj : (int)a.march_n_out;
  }
  a.nseg = xg_ceil_div(a.march_n_out, a.J);
  // row groups: operated dims alone, runs of non-operated dims merged
  a.nrow_groups = 0;
  int64_t nrows = 1;
  for (int d = 0; d < d_end; ++d) {
    if (d == march_dim) continue;
    if (out_shape[d] == 1 && app_index[d] < 0) continue;
    const bool merge = a.nrow_groups > 0 && app_index[d] < 0 && a.row_axis[a.nrow_groups - 1] < 0 &&
                       a.row_in_stride[a.nrow_groups - 1] == in_stride[d] * shape[d] &&
                       a.row_out_stride[a.nrow_groups - 1] == out_stride[d] * out_shape[d];
    if (merge) {
      const int g = a.nrow_groups - 1;
      a.row_size[g] *= out_shape[d];
      a.row_in_stride[g] = in_stride[d];
      a.row_out_stride[g] = out_stride[d];
    } else {
      if (a.nrow_groups == kMaxGroups)
        return xg_fail(XG_ENOTIMPL, "xg_stencil_multi: too many interleaved dimensions");
      const int g = a.nrow_groups++;
      a.row_size[g] = out_shape[d];
      a.row_in_stride[g] = in_stride[d];
      a.row_out_stride[g] = out_stride[d];
      a.row_axis[g] = app_index[d];
    }
    nrows *= out_shape[d];
  }
  const int64_t nblocks = nrows * a.nseg;
  if (nblocks > 0x7fffffffLL) return xg_fail(XG_ENOTIMPL, "xg_stencil_multi: more than 2^31 blocks");
  // vector path: aligned rows whose length the vector width divides; an operated innermost dim must
  // keep its length (lo + hi == 1) so input and output rows stay aligned with each other
  bool vec_ok = ((uintptr_t)in % 16 == 0) && ((uintptr_t)out % 16 == 0) && (last_n_out % VEC == 0);
  if (last >= 0) vec_ok = vec_ok && (lo[last] + hi[last] == 1) && (shape[ndim - 1] % VEC == 0) && shape[ndim - 1] >= 2 * VEC;
  for (int d = 0; d < ndim - 1 && vec_ok; ++d)
    if (shape[d] > 1 && in_stride[d] % VEC != 0) vec_ok = false;
  for (int d = 0; d < ndim - 1 && vec_ok; ++d)
    if (out_shape[d] > 1 && out_stride[d] % VEC != 0) vec_ok = false;
  const int64_t nvec = vec_ok ? last_n_out / VEC : last_n_out;
  int threads = 256;
  while (threads > 32 && threads / 2 >= nvec) threads /= 2;
  if (naxes == 2) {
    if (vec_ok) return launch_last<T, VEC, 2>(last, march, a, nblocks, threads, st);
    return launch_last<T, 1, 2>(last, march, a, nblocks, threads, st);
  }
  if (vec_ok) return launch_last<T, VEC, 3>(last, march, a, nblocks, threads, st);
  return launch_last<T, 1, 3>(last, march, a, nblocks, threads, st);
}

}  // namespace

extern "C" int xg_stencil_multi(int dtype, const void* in, void* out, int ndim, const int64_t* shape,
                                int naxes, const int* axes, const int* ops, const int* lo, const int* hi,
                                const int* bc, const double* fill_value, void* stream) {
  if (!in || !out || !shape || !axes || !ops || !lo || !hi || !bc || !fill_value)
    return xg_fail(XG_EINVAL, "xg_stencil_multi: null pointer");
  if (ndim < 1 || ndim > XG_MAX_NDIM) return xg_fail(XG_EINVAL, "xg_stencil_multi: bad ndim");
  if (naxes < 2 || naxes > kMaxAx)
    return xg_fail(XG_EINVAL, "xg_stencil_multi: 2 or 3 axes (use xg_stencil2 for one)");
  for (int k = 0; k < naxes; ++k) {
    if (ops[k] < XG_OP_DIFF || ops[k] > XG_OP_MAX) return xg_fail(XG_EINVAL, "xg_stencil_multi: unknown op");
    if (ops[k] != ops[0])
      return xg_fail(XG_ENOTIMPL, "xg_stencil_multi: the fused kernel applies ONE operator along all axes "
                                  "(what Grid.diff / interp / min / max do); chain xg_stencil2 for mixed ones");
  }
  if (in == out) return xg_fail(XG_EINVAL, "xg_stencil_multi: in-place operation is not supported");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == XG_F32)
    return multi_typed<float>(in, out, ndim, shape, naxes, axes, ops, lo, hi, bc, fill_value, st);
  if (dtype == XG_F64)
    return multi_typed<double>(in, out, ndim, shape, naxes, axes, ops, lo, hi, bc, fill_value, st);
  return xg_fail(XG_EINVAL, "xg_stencil_multi: dtype must be XG_F32 or XG_F64");
}
