// xg_fold_rows: the north-fold halo of a tripolar grid.
//
// The fold axis (Y) of a tripolar ocean grid folds its northern edge onto itself along the bipolar
// seam: halo row r (going north) is interior row n-1-skip-r mirrored along the periodic seam axis (X)
// about the pole, seam index k reading (mirror - k) mod period, and vector components change sign.
// The mirror wraps at a point that depends on the field's position and on the pivot, so one kernel
// does the gather (and the metric product and sign in the same pass) instead of a set of host-planned
// signed-stride copies.  The rows are thin (one per level), so the kernel is plain: one thread per
// output element, flat over the output order (coalesced stores), per-dim index decomposition.
#include "xg_common.cuh"

namespace {

constexpr int kThreads = 256;

template <typename T>
struct FoldArgs {
  const T* in;
  T* out;
  const T* pre;  // nullptr = absent; read at the mirrored source cell
  int ndim;
  int fold, seam;   // dims (after collapsing)
  int64_t total;    // output elements written
  int64_t shape[XG_MAX_NDIM];  // iteration shape: `width` along fold
  int64_t ostride[XG_MAX_NDIM], istride[XG_MAX_NDIM], pstride[XG_MAX_NDIM];
  int64_t out_base;  // row0 * ostride[fold]
  int64_t src_top;   // n - 1 - skip
  int64_t mirror, period;
  int negate;
};

template <typename T>
__global__ void __launch_bounds__(kThreads) k_fold_rows(const FoldArgs<T> a) {
  for (int64_t g = (int64_t)blockIdx.x * kThreads + threadIdx.x; g < a.total;
       g += (int64_t)gridDim.x * kThreads) {
    int64_t rem = g, ooff = a.out_base, ioff = 0, poff = 0;
#pragma unroll
    for (int d = XG_MAX_NDIM - 1; d >= 0; --d) {
      if (d < a.ndim) {
        const int64_t q = rem / a.shape[d];
        const int64_t c = rem - q * a.shape[d];
        rem = q;
        int64_t src = c;
        if (d == a.fold) {
          src = a.src_top - c;
        } else if (d == a.seam) {
          src = (a.mirror - c) % a.period;
          if (src < 0) src += a.period;
        }
        ooff += c * a.ostride[d];
        ioff += src * a.istride[d];
        poff += src * a.pstride[d];
      }
    }
    T v = a.in[ioff];
    if (a.pre) v = v * __ldg(a.pre + poff);
    a.out[ooff] = a.negate ? -v : v;
  }
}

template <typename T>
int fold_typed(const void* in, void* out, int ndim, const int64_t* shape, int fold, int seam,
               int64_t out_len, int64_t row0, int width, int skip, int64_t mirror, int64_t period,
               int negate, const void* pre, const int64_t* pre_strides, cudaStream_t st) {
  FoldArgs<T> a;
  a.in = static_cast<const T*>(in);
  a.out = static_cast<T*>(out);
  a.pre = static_cast<const T*>(pre);
  a.negate = negate;
  a.src_top = shape[fold] - 1 - skip;
  a.mirror = mirror;
  a.period = period;
  // contiguous strides of the input and of the output (fold dim of length out_len)
  int64_t is[XG_MAX_NDIM], os[XG_MAX_NDIM];
  int64_t iacc = 1, oacc = 1;
  for (int d = ndim - 1; d >= 0; --d) {
    is[d] = iacc;
    os[d] = oacc;
    iacc *= shape[d];
    oacc *= (d == fold) ? out_len : shape[d];
  }
  a.out_base = row0 * os[fold];
  // merge neighbouring plain dims that are contiguous in the output, the input and `pre`
  int k = 0;
  a.total = 1;
  a.fold = a.seam = -1;
  for (int d = 0; d < ndim; ++d) {
    const int64_t n = (d == fold) ? width : shape[d];
    const int64_t ps = pre ? pre_strides[d] : 0;
    a.total *= n;
    const bool special = (d == fold || d == seam);
    const bool prev_plain = k > 0 && (k - 1) != a.fold && (k - 1) != a.seam;
    if (!special && prev_plain && a.ostride[k - 1] == os[d] * n && a.istride[k - 1] == is[d] * n &&
        a.pstride[k - 1] == ps * n) {
      a.shape[k - 1] *= n;
      a.ostride[k - 1] = os[d];
      a.istride[k - 1] = is[d];
      a.pstride[k - 1] = ps;
      continue;
    }
    if (d == fold) a.fold = k;
    if (d == seam) a.seam = k;
    a.shape[k] = n;
    a.ostride[k] = os[d];
    a.istride[k] = is[d];
    a.pstride[k] = ps;
    ++k;
  }
  a.ndim = k;
  for (int d = k; d < XG_MAX_NDIM; ++d) {
    a.shape[d] = 1;
    a.ostride[d] = a.istride[d] = a.pstride[d] = 0;
  }
  if (a.total == 0) return XG_OK;
  int64_t blocks = xg_ceil_div(a.total, kThreads);
  if (blocks > XG_SMS * 16) blocks = XG_SMS * 16;
  k_fold_rows<T><<<(unsigned)blocks, kThreads, 0, st>>>(a);
  return xg_check_launch("xg_fold_rows");
}

}  // namespace

extern "C" int xg_fold_rows(int dtype, const void* in, void* out, int ndim, const int64_t* shape,
                            int fold_axis, int seam_axis, int64_t out_len, int64_t row0, int width,
                            int skip, int64_t mirror, int64_t period, int negate, const void* pre,
                            const int64_t* pre_strides, void* stream) {
  if (!in || !out || !shape) return xg_fail(XG_EINVAL, "xg_fold_rows: null pointer");
  if (pre && !pre_strides) return xg_fail(XG_EINVAL, "xg_fold_rows: null pre_strides");
  if (ndim < 2 || ndim > XG_MAX_NDIM) return xg_fail(XG_EINVAL, "xg_fold_rows: bad ndim");
  if (fold_axis < 0 || fold_axis >= ndim || seam_axis < 0 || seam_axis >= ndim)
    return xg_fail(XG_EINVAL, "xg_fold_rows: axis out of range");
  if (fold_axis == seam_axis) return xg_fail(XG_EINVAL, "xg_fold_rows: the fold and seam axes must differ");
  if (dtype != XG_F32 && dtype != XG_F64)
    return xg_fail(XG_EINVAL, "xg_fold_rows: dtype must be XG_F32 or XG_F64");
  for (int d = 0; d < ndim; ++d)
    if (shape[d] < 0) return xg_fail(XG_EINVAL, "xg_fold_rows: negative extent");
  if (skip < 0 || skip > 1) return xg_fail(XG_EINVAL, "xg_fold_rows: skip must be 0 or 1");
  const int64_t n = shape[fold_axis];
  if (width < 1 || width > n - skip)
    return xg_fail(XG_EINVAL, "xg_fold_rows: halo width exceeds the interior rows of the fold axis");
  if (row0 < 0 || out_len < row0 + width)
    return xg_fail(XG_EINVAL, "xg_fold_rows: the halo rows do not fit into out_len");
  if (period < 1) return xg_fail(XG_EINVAL, "xg_fold_rows: period must be positive");
  const int64_t L = shape[seam_axis];
  for (int64_t k = 0; k < L; ++k) {
    int64_t src = (mirror - k) % period;
    if (src < 0) src += period;
    if (src >= L)
      return xg_fail(XG_ENOTIMPL,
                     "xg_fold_rows: seam position incompatible with the pivot: the mirror partner of a seam "
                     "index lies outside the seam dim");
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == XG_F32)
    return fold_typed<float>(in, out, ndim, shape, fold_axis, seam_axis, out_len, row0, width, skip, mirror,
                             period, negate, pre, pre_strides, st);
  return fold_typed<double>(in, out, ndim, shape, fold_axis, seam_axis, out_len, row0, width, skip, mirror,
                            period, negate, pre, pre_strides, st);
}
