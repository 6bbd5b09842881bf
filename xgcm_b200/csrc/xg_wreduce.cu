// xg_wreduce — metric-weighted reduction along one axis, one HBM pass.
//
// Replaces xgcm/grid.py:1598-1605 (integrate: (da * metric).sum(dim), a full-size
// product temp plus a reduction read in the reference) and :1680-1685
// (average: da.weighted(metric).mean(dim)).
//
// Order of summation:
//   strided axis (inner > 1): sequential per column in the field dtype — exactly
//       what np.add.reduce does along a non-contiguous axis (SURVEY H4-ii);
//   innermost axis (inner == 1): numpy uses pairwise summation there, which is
//       close to the exact sum; we accumulate in fp64 (lane-strided partials +
//       shuffle tree) and round once, well inside the 1e-6 / 1e-12 budgets.
//
// Roofline: HBM, sizeof(T) * (1 + metric fraction) bytes per input cell.
#include "xg_common.cuh"

namespace {

constexpr int kThreads = 128;

template <typename T>
struct ReduceArgs {
  const T* in;
  T* out;
  int64_t outer, n, inner;
  int mode, skipna;
  XgOperand w;
  int64_t nvec_inner;
  bool small_index;
  XgFastDiv fd_nvi;  // multiply-high form of nvec_inner (valid with small_index)
};

template <typename T, int VEC, bool HASW, int U>
__global__ void __launch_bounds__(kThreads) k_reduce_strided(const ReduceArgs<T> a) {
  typedef XgPack<T, VEC> Pack;
  const int64_t g = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (g >= a.outer * a.nvec_inner) return;
  int64_t o, iv;
  xg_divmod(g, a.nvec_inner, a.fd_nvi, a.small_index, o, iv);
  const int64_t i = iv * VEC;
  const T* ibase = a.in + o * a.n * a.inner + i;
  XgOperandView<T, VEC> w_v;
  if (HASW) w_v = xg_operand_view<T, VEC>(a.w, xg_groups_offset(a.w.outer, o), i);
  Pack num, den;
#pragma unroll
  for (int q = 0; q < VEC; ++q) num.v[q] = den.v[q] = T(0);
  const bool mean = a.mode != XG_REDUCE_SUM;  // MEAN and WVALID carry the sum of valid weights

  auto step = [&](const Pack& v, const Pack& m) {
#pragma unroll
    for (int q = 0; q < VEC; ++q) {
      if (!mean) {
        T p = HASW ? v.v[q] * m.v[q] : v.v[q];  // grid.py:1599 da * weight
        if (a.skipna && xg_isnan(p)) p = T(0);   // .sum(skipna) -> nansum
        num.v[q] = num.v[q] + p;
      } else {
        // da.weighted(w).mean(skipna): NaN cells drop out together with their weights; with
        // skipna=False they stay in and the result is NaN (grid.py:1680-1685 forwards the kwarg)
        const bool valid = !a.skipna || !xg_isnan(v.v[q]);
        const T wq = HASW ? m.v[q] : T(1);
        num.v[q] = num.v[q] + (valid ? v.v[q] * wq : T(0));
        den.v[q] = den.v[q] + (valid ? wq : T(0));
      }
    }
  };
  int64_t k = 0;
  for (; k + U <= a.n; k += U) {
    Pack v[U], m[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      v[u] = xg_ld_stream<T, VEC>(ibase + (k + u) * a.inner);
      if (HASW) m[u] = xg_ld_view<T, VEC>(w_v, (k + u) * a.w.axis_stride);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) step(v[u], m[u]);
  }
  for (; k < a.n; ++k) {
    Pack v = xg_ld_stream<T, VEC>(ibase + k * a.inner), m;
    if (HASW) m = xg_ld_view<T, VEC>(w_v, k * a.w.axis_stride);
    step(v, m);
  }
  Pack r;
#pragma unroll
  for (int q = 0; q < VEC; ++q) {
    if (!mean) r.v[q] = num.v[q];
    else if (a.mode == XG_REDUCE_WVALID) r.v[q] = den.v[q];
    else r.v[q] = (den.v[q] != T(0)) ? num.v[q] / den.v[q] : T(NAN);
  }
  xg_st_stream<T, VEC>(a.out + o * a.inner + i, r);
}

// one warp per row (innermost axis); fp64 accumulation; 16-byte loads when the rows allow it.  Either way a lane
// sums the same cells in the same order (W consecutive cells every 32 W), so a row gives the same bits whether it
// is aligned or not: x[t] of a (T, Z, Y, X) field and x[t].clone() agree.
template <typename T, bool HASW, int VEC>
__global__ void __launch_bounds__(kThreads) k_reduce_rows(const ReduceArgs<T> a) {
  const int64_t r = (int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
  if (r >= a.outer) return;
  const int lane = threadIdx.x & 31;
  const T* row = a.in + r * a.n;
  const T* wp = reinterpret_cast<const T*>(a.w.ptr);
  int64_t w_base = 0;
  if (HASW) w_base = xg_groups_offset(a.w.outer, r);
  const bool mean = a.mode != XG_REDUCE_SUM;
  double num = 0.0, den = 0.0;
  constexpr int W = XgVecWidth<T>::value;
  for (int64_t x = (int64_t)lane * W; x < a.n; x += 32 * W) {
    XgPack<T, W> v;
    if constexpr (VEC == W) {
      v = xg_ld_stream<T, W>(row + x);
    } else {
#pragma unroll
      for (int q = 0; q < W; ++q)
        if (x + q < a.n) v.v[q] = xg_ld_stream<T, 1>(row + x + q).v[0];
    }
#pragma unroll
    for (int q = 0; q < W; ++q) {
      if (VEC != W && x + q >= a.n) break;
      const T w = HASW ? __ldg(wp + w_base + (x + q) * a.w.axis_stride) : T(1);
      if (!mean) {
        T p = HASW ? v.v[q] * w : v.v[q];
        if (a.skipna && xg_isnan(p)) p = T(0);
        num += (double)p;
      } else {
        const bool valid = !a.skipna || !xg_isnan(v.v[q]);
        num += valid ? (double)(v.v[q] * w) : 0.0;
        den += valid ? (double)w : 0.0;
      }
    }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    num += __shfl_xor_sync(0xffffffffu, num, s);
    den += __shfl_xor_sync(0xffffffffu, den, s);
  }
  if (lane == 0) {
    if (!mean) a.out[r] = (T)num;
    else if (a.mode == XG_REDUCE_WVALID) a.out[r] = (T)den;
    else a.out[r] = (den != 0.0) ? (T)(num / den) : T(NAN);
  }
}

template <typename T, bool HASW>
int reduce_launch(ReduceArgs<T>& a, cudaStream_t st) {
  constexpr int VEC = XgVecWidth<T>::value;
  constexpr int U = 8;
  if (a.inner > 1) {
    bool vec_ok = (a.inner % VEC == 0) && ((uintptr_t)a.in % 16 == 0) && ((uintptr_t)a.out % 16 == 0) &&
                  xg_vec_view_ok(a.w);
    if (vec_ok && a.outer * (a.inner / VEC) < XG_SMS * 64) vec_ok = false;
    a.nvec_inner = vec_ok ? a.inner / VEC : a.inner;
    if (!vec_ok) a.w.vec_ok = 0;
    a.small_index = a.outer * a.nvec_inner < (1ll << 31);
    a.fd_nvi = xg_fastdiv_make(a.small_index ? a.nvec_inner : 1);
    const int64_t blocks = xg_ceil_div(a.outer * a.nvec_inner, kThreads);
    if (blocks > 0x7fffffffLL) return xg_fail(XG_EINVAL, "xg_wreduce: grid too large");
    if (vec_ok)
      k_reduce_strided<T, VEC, HASW, U><<<(unsigned)blocks, kThreads, 0, st>>>(a);
    else
      k_reduce_strided<T, 1, HASW, U><<<(unsigned)blocks, kThreads, 0, st>>>(a);
    return xg_check_launch(vec_ok ? "xg_wreduce(strided, vec)" : "xg_wreduce(strided, scalar)");
  }
  const int64_t blocks = xg_ceil_div(a.outer, kThreads / 32);
  if (blocks > 0x7fffffffLL) return xg_fail(XG_EINVAL, "xg_wreduce: grid too large");
  const bool row_vec = a.n % VEC == 0 && ((uintptr_t)a.in & 15) == 0;
  if (row_vec)
    k_reduce_rows<T, HASW, VEC><<<(unsigned)blocks, kThreads, 0, st>>>(a);
  else
    k_reduce_rows<T, HASW, 1><<<(unsigned)blocks, kThreads, 0, st>>>(a);
  return xg_check_launch(row_vec ? "xg_wreduce(rows, vec)" : "xg_wreduce(rows, scalar)");
}

template <typename T>
int wreduce_typed(const void* in, const void* weight, const int64_t* w_strides, void* out, int ndim,
                  const int64_t* shape, int axis, int mode, int skipna, cudaStream_t st) {
  constexpr int VEC = XgVecWidth<T>::value;
  XgView v;
  int rc = xg_collapse_view(ndim, shape, axis, &v);
  if (rc) return rc;
  ReduceArgs<T> a;
  a.in = static_cast<const T*>(in);
  a.out = static_cast<T*>(out);
  a.outer = v.outer;
  a.n = v.n;
  a.inner = v.inner;
  a.mode = mode;
  a.skipna = skipna ? 1 : 0;
  a.nvec_inner = 0;
  a.small_index = false;
  a.fd_nvi = xg_fastdiv_make(1);
  rc = xg_make_operand(weight, w_strides, ndim, shape, axis, VEC, sizeof(T), &a.w,
                       "xg_wreduce(weight)");
  if (rc) return rc;
  if (v.outer == 0 || v.inner == 0) return XG_OK;
  if (weight) return reduce_launch<T, true>(a, st);
  return reduce_launch<T, false>(a, st);
}

}  // namespace

extern "C" int xg_wreduce(int dtype, const void* in, const void* weight, const int64_t* w_strides,
                          void* out, int ndim, const int64_t* shape, int axis, int mode,
                          int skipna, void* stream) {
  if (!in || !out || !shape) return xg_fail(XG_EINVAL, "xg_wreduce: null pointer");
  if (mode != XG_REDUCE_SUM && mode != XG_REDUCE_MEAN && mode != XG_REDUCE_WVALID)
    return xg_fail(XG_EINVAL, "xg_wreduce: unknown mode");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == XG_F32)
    return wreduce_typed<float>(in, weight, w_strides, out, ndim, shape, axis, mode, skipna, st);
  if (dtype == XG_F64)
    return wreduce_typed<double>(in, weight, w_strides, out, ndim, shape, axis, mode, skipna, st);
  return xg_fail(XG_EINVAL, "xg_wreduce: dtype must be XG_F32 or XG_F64");
}
