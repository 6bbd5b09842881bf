// Host-buffer entry points beyond the stencils of xg_host.cu, on the same slab engine (xg_host.cuh), with
// slabs cut along a dimension that is not the outermost one (strided 2-D copies), so that every device entry point
// has a host twin:
//
//   xg_stencil_multi_host    xgcm/grid.py:798-832 (a multi-axis diff / interp / min / max): one
//                            xg_stencil_multi launch per slab
//   xg_cumscan_host          xgcm/grid.py:1306-1414 on numpy-backed fields
//   xg_wreduce_host          xgcm/grid.py:1598-1605, :1680-1685
//   xg_wreduce_host_multi    the same over several dims: the device launch sequence per slab
//   xg_vinterp_linear_host        xgcm/transform.py:233-249
//   xg_vinterp_conservative_host  xgcm/transform.py:157-198 (k_vconserv per slab)
//
// Slabs are cut along a NON-operated dimension: a slab of (Z, y0:y1, X) is Z pieces of (y1-y0)*X
// contiguous elements -> one cudaMemcpy2DAsync each way.  Lines along the operated axis stay whole, so
// no halo exchange between slabs is needed and summation order is untouched.  xg_cumscan_host and
// xg_wreduce_host cut the first non-operated dim, and upload their metric / weight whole, once.
//
// The two multi-axis twins cut the outermost dim of extent > 1 that is not operated, so every operated line is
// whole in a slab.  When every dim of extent > 1 is operated, xg_stencil_multi_host cuts the outermost one and
// reads the row next to each slab (as the stencils of xg_host.cu do along dim 0), and xg_wreduce_host_multi keeps
// one partial per index of it on the device and runs the launches along it once, at the end.
//
// The two transform twins pick the outermost non-operated dim of extent > 1 one index of which (its phi,
// theta, theta-bounds scratch and result bytes together) fits the slab budget, else the innermost one, so
// that (time_counter=1, deptht, y, x) or a short time axis does not make one huge slab; the rows per slab
// are sized from that same per-index total (the result of m >> n bins outweighs phi).  A dense theta field
// is the pipe's second streamed input: it goes up in the same slab window as phi into its own per-slot
// buffers.  A broadcast theta (a 1-D coordinate, (T, Z+1, 1, 1), ...) is uploaded whole once.  Theta given
// at cell centres (xg_vinterp_conservative_host's theta_at_centers) becomes its n + 1 bounds on the device:
// one xg_stencil2(interp, lo = hi = 1, extend) along the axis per slab into the workspace's scratch buffer
// (once, into an aux buffer, for a broadcast theta) -- the center -> outer shift of grid.interp(theta, axis,
// padding="extend"), so the bounds are the ones that call would give.
#include "xg_host.cuh"

using namespace xg_host;

namespace {

int first_free_dim(int ndim, int axis) { return (ndim == 1) ? -1 : (axis == 0 ? 1 : 0); }

// ------------------------------------------------------------------- the two transform twins (theta beside phi)
int64_t numel(int ndim, const int64_t* shape) {
  int64_t n = 1;
  for (int d = 0; d < ndim; ++d) n *= shape[d];
  return n;
}

void dense_strides(int ndim, const int64_t* shape, int64_t* strides) {  // C order
  int64_t s = 1;
  for (int d = ndim - 1; d >= 0; --d) {
    strides[d] = s;
    s *= shape[d];
  }
}

// a dense C-contiguous array of `tshape` (dims of extent 1 aside), which can stream beside the field (theta beside
// phi, a weight beside the field it reduces)
bool is_dense(int ndim, const int64_t* tshape, const int64_t* strides) {
  int64_t ds[XG_MAX_NDIM];
  dense_strides(ndim, tshape, ds);
  for (int d = 0; d < ndim; ++d)
    if (tshape[d] > 1 && strides[d] != ds[d]) return false;
  return true;
}

// the compact shape of a broadcast theta: 1 where it is broadcast (stride 0) or of extent 1
void compact_shape(int ndim, const int64_t* tshape, const int64_t* strides, int64_t* cshape) {
  for (int d = 0; d < ndim; ++d) cshape[d] = (tshape[d] > 1 && strides[d] != 0) ? tshape[d] : 1;
}

// Slab dim of the transform twins: the outermost non-operated dim of extent > 1 whose one index -- its share of
// `total_bytes` (phi, streamed theta, theta-bounds scratch and result together) -- fits the slab budget; else the
// innermost non-operated dim of extent > 1; -1 when there is none (the whole field is one slab).
int transform_slab_dim(int ndim, const int64_t* shape, int axis, int64_t total_bytes) {
  const int64_t budget = slab_budget_bytes();
  int inner = -1;
  for (int d = 0; d < ndim; ++d) {
    if (d == axis || shape[d] <= 1) continue;
    if (total_bytes / shape[d] <= budget) return d;
    inner = d;
  }
  return inner;
}

// theta of one transform-twin call: tshape = phi's shape with `tn` along the axis (n + 1 bounds, or n centres)
struct ThetaPlan {
  int dtype = XG_F32, ndim = 0, axis = 0, sd = -1;
  size_t es = 4;
  bool dense = false, centers = false;
  int64_t tshape[XG_MAX_NDIM], bshape[XG_MAX_NDIM];  // theta as given; its n + 1 bounds
  const void* d_bcast = nullptr;                     // broadcast theta's bounds on the device
  int64_t bstrides[XG_MAX_NDIM];                     // and their strides

  // bytes of the whole streamed theta and of the whole bounds scratch
  int64_t stream_bytes() const { return dense ? numel(ndim, tshape) * (int64_t)es : 0; }
  int64_t scratch_bytes() const { return dense && centers ? numel(ndim, bshape) * (int64_t)es : 0; }

  // device bounds of slab rows [j0, j1) of the slab dim, and their strides (on stream st, after the slab's upload)
  int slab(int64_t j0, int64_t j1, const SlabBufs& b, cudaStream_t st, const void** th, int64_t* strides) const {
    if (!dense) {
      for (int d = 0; d < ndim; ++d) strides[d] = bstrides[d];
      *th = static_cast<const char*>(d_bcast) + (sd >= 0 ? (size_t)(j0 * bstrides[sd]) * es : 0);
      return XG_OK;
    }
    int64_t ts[XG_MAX_NDIM], bs[XG_MAX_NDIM];
    for (int d = 0; d < ndim; ++d) {
      ts[d] = tshape[d];
      bs[d] = bshape[d];
    }
    if (sd >= 0) ts[sd] = bs[sd] = j1 - j0;
    dense_strides(ndim, bs, strides);  // a slab's own dense layout, not the host strides
    if (!centers) {
      *th = b.in2;
      return XG_OK;
    }
    *th = b.scratch;
    return xg_stencil2(XG_OP_INTERP, dtype, b.in2, b.scratch, ndim, ts, axis, 1, 1, XG_BC_EXTEND, 0.0, nullptr,
                       nullptr, nullptr, nullptr, nullptr, nullptr, st);
  }
};

// Argument checks on theta that need no device: its extent along the axis, and (at centres) a layout the
// center -> outer stencil can read.
int check_theta(const char* fn, int ndim, const int64_t* tshape, const int64_t* strides, int axis, int centers) {
  for (int d = 0; d < ndim; ++d)
    if (strides[d] < 0) return xg_fail(XG_EINVAL, std::string(fn) + ": negative theta stride");
  if (tshape[axis] > 1 && strides[axis] == 0)
    return xg_fail(XG_EINVAL, std::string(fn) + ": theta must hold " + std::to_string(tshape[axis]) +
                                  (centers ? " cell-centre values" : " cell bounds") +
                                  " along the axis; it is broadcast along it");
  if (centers && !is_dense(ndim, tshape, strides)) {
    int64_t cshape[XG_MAX_NDIM], cs[XG_MAX_NDIM];
    compact_shape(ndim, tshape, strides, cshape);
    dense_strides(ndim, cshape, cs);
    for (int d = 0; d < ndim; ++d)
      if (cshape[d] > 1 && strides[d] != cs[d])
        return xg_fail(XG_EINVAL, std::string(fn) +
                                      ": theta at cell centres must be C-contiguous in the dims it is not broadcast over");
  }
  return XG_OK;
}

// The plan, before any device is touched; theta holds `tn` values along the axis (n + 1 bounds, n centres, or the
// n levels of the linear twin).
void plan_theta(ThetaPlan* p, int dtype, const int64_t* strides, int centers, int64_t tn, int ndim,
                const int64_t* shape, int axis) {
  p->dtype = dtype;
  p->es = dtype == XG_F32 ? 4 : 8;
  p->ndim = ndim;
  p->axis = axis;
  p->centers = centers != 0;
  for (int d = 0; d < ndim; ++d) p->tshape[d] = p->bshape[d] = shape[d];
  p->tshape[axis] = tn;
  p->bshape[axis] = p->centers ? tn + 1 : tn;
  p->dense = is_dense(ndim, p->tshape, strides);
}

// On the open session: a broadcast theta goes up whole (kAuxTheta); plan_theta_bounds makes the bounds of one that
// holds centres.
int upload_theta(Session& ss, ThetaPlan* p, const void* theta, const int64_t* strides) {
  if (p->dense) return XG_OK;
  int rc = ss.upload(kAuxTheta, theta, operand_span(strides, p->tshape, p->ndim, p->es), &p->d_bcast);
  if (rc) return rc;
  for (int d = 0; d < p->ndim; ++d) p->bstrides[d] = strides[d];
  return XG_OK;
}

// the bounds of a broadcast theta held at centres, once, into kAuxThetaBounds, on the kernel stream (after the fence)
int plan_theta_bounds(Session& ss, ThetaPlan* p, const int64_t* strides) {
  if (p->dense || !p->centers) return XG_OK;
  int64_t cshape[XG_MAX_NDIM], cb[XG_MAX_NDIM];
  compact_shape(p->ndim, p->tshape, strides, cshape);
  for (int d = 0; d < p->ndim; ++d) cb[d] = cshape[d];
  cb[p->axis] = p->bshape[p->axis];
  void* bounds = nullptr;
  int rc = ss.aux(kAuxThetaBounds, (size_t)numel(p->ndim, cb) * p->es, &bounds);
  if (rc) return rc;
  rc = xg_stencil2(XG_OP_INTERP, p->dtype, p->d_bcast, bounds, p->ndim, cshape, p->axis, 1, 1, XG_BC_EXTEND,
                   0.0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, ss.kernel_stream());
  if (rc) return rc;
  dense_strides(p->ndim, cb, p->bstrides);
  for (int d = 0; d < p->ndim; ++d)
    if (cb[d] == 1) p->bstrides[d] = 0;  // broadcast again over phi's extent
  p->d_bcast = bounds;
  return XG_OK;
}

// [C][L][R] views of phi, streamed theta and the result (shape-without-axis + trailing `m_out`) around the slab
// dim of a transform twin, and the PipeExtra that streams theta and sizes the slabs
struct TransformViews {
  int sd = -1;
  View3 vin{1, 1, 1}, vout{1, 1, 1};
  PipeExtra ex;
};

TransformViews transform_views(int ndim, const int64_t* shape, int axis, int64_t m_out, const ThetaPlan& p,
                               const void* theta) {
  TransformViews t;
  const int64_t es = (int64_t)p.es;
  int64_t out_shape[XG_MAX_NDIM + 1];
  int nd_o = 0;
  for (int d = 0; d < ndim; ++d)
    if (d != axis) out_shape[nd_o++] = shape[d];
  out_shape[nd_o++] = m_out;
  const int64_t out_bytes = numel(nd_o, out_shape) * es;
  const int64_t total = numel(ndim, shape) * es + p.stream_bytes() + p.scratch_bytes() + out_bytes;
  t.sd = transform_slab_dim(ndim, shape, axis, total);
  const int64_t L = t.sd >= 0 ? shape[t.sd] : 1;
  if (t.sd >= 0) {
    t.vin = view3(ndim, shape, t.sd);
    t.vout = view3(nd_o, out_shape, t.sd < axis ? t.sd : t.sd - 1);
    t.ex.in2 = view3(ndim, p.tshape, t.sd);
  } else {
    t.vin = View3{1, 1, numel(ndim, shape)};
    t.vout = View3{1, 1, out_bytes / es};
    t.ex.in2 = View3{1, 1, numel(ndim, p.tshape)};
  }
  if (p.dense) t.ex.hin2 = theta;
  t.ex.scratch_row_bytes = (size_t)(p.scratch_bytes() / L);
  t.ex.row_bytes = total / L;
  return t;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------
namespace {

int multi_host(const char* name, int dtype, const void* in, void* out, int ndim, const int64_t* shape, int naxes,
               const int* axes, const int* ops, const int* lo, const int* hi, const int* bc, const double* fill_value,
               const void* const* pre, const int64_t* pre_strides, const void* const* post,
               const int64_t* post_strides, int device) {
  const std::string who = name;
  int rc = xg_stencil_multi_check(name, dtype, in, out, ndim, shape, naxes, axes, ops, lo, hi, bc, fill_value, pre,
                                  pre_strides, post, post_strides);
  if (rc) return rc;
  int app[XG_MAX_NDIM];  // application index of each dim, -1 where it is not operated
  int64_t out_shape[XG_MAX_NDIM];
  for (int d = 0; d < ndim; ++d) {
    app[d] = -1;
    out_shape[d] = shape[d];
  }
  for (int k = 0; k < naxes; ++k) {
    app[axes[k]] = k;
    out_shape[axes[k]] = shape[axes[k]] + lo[k] + hi[k] - 1;
  }
  // slab dim: the outermost non-operated dim of extent > 1, whose slabs hold every operated line whole; else the
  // outermost dim of extent > 1, an operated one (the dims in front of it have extent 1)
  int sd = -1;
  for (int d = 0; d < ndim && sd < 0; ++d)
    if (app[d] < 0 && shape[d] > 1) sd = d;
  for (int d = 0; d < ndim && sd < 0; ++d)
    if (shape[d] > 1) sd = d;
  if (sd < 0) sd = 0;
  const int ka = app[sd];  // the application cut into slabs, -1 when none is
  PipeExtra ex;
  if (ka >= 0) {
    // each slab reads the row next to it along the cut dim; xg_stencil_multi takes no halo planes, so only the
    // field's own ends can be padded, and a slab of result rows must read as many input rows (lo + hi == 1)
    if (lo[ka] + hi[ka] != 1)
      return xg_fail(XG_ENOTIMPL, who + ": outer / inner shift along the cut dim (every dim of extent > 1 is "
                                        "operated); use xg_stencil_multi");
    if (bc[ka] == XG_BC_PERIODIC)
      return xg_fail(XG_ENOTIMPL, who + ": periodic boundary along the cut dim (every dim of extent > 1 is "
                                        "operated); use xg_stencil_multi");
    ex.lo_rows = lo[ka];
    ex.hi_rows = hi[ka];
  }
  int64_t total_out = 1;
  for (int d = 0; d < ndim; ++d) total_out *= out_shape[d];
  if (total_out == 0) return XG_OK;
  const size_t es = dtype == XG_F32 ? 4 : 8;
  const View3 vin = view3(ndim, shape, sd), vout = view3(ndim, out_shape, sd);
  ex.row_bytes = (vin.C * vin.R + vout.C * vout.R) * (int64_t)es;
  // each stage's metric shapes: its input (pre) and output (post)
  int64_t met_shape[2 * 3][XG_MAX_NDIM];
  for (int m = 0; m < naxes; ++m)
    for (int d = 0; d < ndim; ++d) {
      met_shape[m][d] = app[d] >= 0 && app[d] < m ? out_shape[d] : shape[d];
      met_shape[3 + m][d] = app[d] >= 0 && app[d] <= m ? out_shape[d] : shape[d];
    }
  return spread(who.c_str(), device, vout.L, false, [&](int dev, int64_t r0, int64_t r1) -> int {
    Session ss;
    int rc2 = ss.open(dev);
    if (rc2) return rc2;
    const void* d_met[2 * 3] = {};  // pre[0..3), post[0..3) on this device
    for (int m = 0; m < naxes && !rc2; ++m)
      for (int w = 0; w < 2 && !rc2; ++w) {
        const void* const* h = w ? post : pre;
        const int64_t* st = (w ? post_strides : pre_strides) + m * ndim;
        if (h && h[m])
          rc2 = ss.upload((Aux)(kAuxStage0 + 3 * w + m), h[m], operand_span(st, met_shape[3 * w + m], ndim, es),
                          &d_met[3 * w + m]);
      }
    if (!rc2 && (pre || post)) rc2 = ss.fence();
    if (rc2) return rc2;
    const int64_t n = shape[sd];
    auto launch = [&](int64_t j0, int64_t j1, int64_t i0, int64_t i1, const SlabBufs& b, cudaStream_t st) -> int {
      int64_t sshape[XG_MAX_NDIM];
      int slo[3], shi[3], sbc[3];
      for (int d = 0; d < ndim; ++d) sshape[d] = shape[d];
      for (int k = 0; k < naxes; ++k) {
        slo[k] = lo[k];
        shi[k] = hi[k];
        sbc[k] = bc[k];
      }
      const char* src = static_cast<const char*>(b.in);
      int64_t s0 = j0;  // first input row of the slab along the cut dim
      if (ka >= 0) {
        // an inner slab edge reads its neighbour row, the field's own ends keep the call's boundary condition
        if (vin.C != 1) return xg_fail(XG_EINVAL, who + ": internal slab window error");
        Window w;
        const int rc3 = read_window(who.c_str(), j0, j1, lo[ka], n, i0, i1, &w);
        if (rc3) return rc3;
        slo[ka] = w.slo;
        shi[ka] = w.shi;
        if (!w.slo && !w.shi) sbc[ka] = XG_BC_NONE;
        src += (size_t)(w.s0 - i0) * vin.R * es;
        sshape[sd] = w.s1 - w.s0;
        s0 = w.s0;
      } else {
        sshape[sd] = j1 - j0;
      }
      if (!pre && !post)
        return xg_stencil_multi(dtype, src, b.out[0], ndim, sshape, naxes, axes, ops, slo, shi, sbc, fill_value, st);
      // the slab's metrics: the cut dim at input rows (s0) before the stage that operates it, at result rows after
      const void* met[2 * 3] = {};
      for (int m = 0; m < naxes; ++m)
        for (int w = 0; w < 2; ++w) {
          const int i = 3 * w + m;
          if (!d_met[i]) continue;
          const int64_t row = (ka >= 0 && (w ? m < ka : m <= ka)) ? s0 : j0;
          const int64_t stride = (w ? post_strides : pre_strides)[m * ndim + sd];
          met[i] = static_cast<const char*>(d_met[i]) + (size_t)(row * stride) * es;
        }
      return xg_stencil_multi_weighted(dtype, src, b.out[0], ndim, sshape, naxes, axes, ops, slo, shi, sbc,
                                       fill_value, met, pre_strides, met + 3, post_strides, st);
    };
    return ss.run(es, in, vin, 1, &out, &vout, launch, ex.rows(r0, r1));
  });
}

}  // namespace

extern "C" int xg_stencil_multi_host(int dtype, const void* in, void* out, int ndim, const int64_t* shape, int naxes,
                                     const int* axes, const int* ops, const int* lo, const int* hi, const int* bc,
                                     const double* fill_value, int device) {
  return multi_host("xg_stencil_multi_host", dtype, in, out, ndim, shape, naxes, axes, ops, lo, hi, bc, fill_value,
                    nullptr, nullptr, nullptr, nullptr, device);
}

extern "C" int xg_stencil_multi_weighted_host(int dtype, const void* in, void* out, int ndim, const int64_t* shape,
                                              int naxes, const int* axes, const int* ops, const int* lo, const int* hi,
                                              const int* bc, const double* fill_value, const void* const* pre,
                                              const int64_t* pre_strides, const void* const* post,
                                              const int64_t* post_strides, int device) {
  return multi_host("xg_stencil_multi_weighted_host", dtype, in, out, ndim, shape, naxes, axes, ops, lo, hi, bc,
                    fill_value, pre, pre_strides, post, post_strides, device);
}

// ---------------------------------------------------------------------------------------------------
extern "C" int xg_cumscan_host(int dtype, const void* in, void* out, int ndim, const int64_t* shape, int axis,
                               int reverse, int trim, int pad_lo, int pad_hi, int bc, double fill_value,
                               const void* pre_metric, const int64_t* pre_strides, const void* post_metric,
                               const int64_t* post_strides, int skipna, int device) {
  if (!in || !out || !shape) return xg_fail(XG_EINVAL, "xg_cumscan_host: null pointer");
  if (dtype != XG_F32 && dtype != XG_F64) return xg_fail(XG_EINVAL, "xg_cumscan_host: dtype must be XG_F32 or XG_F64");
  if (ndim < 1 || ndim > XG_MAX_NDIM) return xg_fail(XG_EINVAL, "xg_cumscan_host: bad ndim");
  if (axis < 0 || axis >= ndim) return xg_fail(XG_EINVAL, "xg_cumscan_host: axis out of range");
  if ((pre_metric && !pre_strides) || (post_metric && !post_strides))
    return xg_fail(XG_EINVAL, "xg_cumscan_host: metric strides missing");
  const size_t es = dtype == XG_F32 ? 4 : 8;
  const int64_t kept = shape[axis] - (trim != XG_TRIM_NONE ? 1 : 0);
  if (kept < 0) return xg_fail(XG_EINVAL, "xg_cumscan_host: operated axis too short to trim");
  int64_t out_shape[XG_MAX_NDIM];
  for (int d = 0; d < ndim; ++d) out_shape[d] = shape[d];
  out_shape[axis] = kept + pad_lo + pad_hi;
  const int sd = first_free_dim(ndim, axis);
  return spread("xg_cumscan_host", device, sd < 0 ? 1 : shape[sd], false,
                [&](int dev, int64_t r0, int64_t r1) -> int {
    Session ss;
    int rc = ss.open(dev);
    if (rc) return rc;
    const void* d_pre = nullptr;
    const void* d_post = nullptr;
    if (pre_metric) rc = ss.upload(kAuxPre, pre_metric, operand_span(pre_strides, shape, ndim, es), &d_pre);
    if (rc) return rc;
    if (post_metric) rc = ss.upload(kAuxPost, post_metric, operand_span(post_strides, out_shape, ndim, es), &d_post);
    if (rc) return rc;
    rc = ss.fence();
    if (rc) return rc;
    if (sd < 0) {  // 1-D: one slab = the whole line
      const View3 v{1, 1, shape[0]}, vo{1, 1, out_shape[0]};
      void* outs[1] = {out};
      auto launch = [&](int64_t, int64_t, int64_t, int64_t, const SlabBufs& b, cudaStream_t st) -> int {
        return xg_cumscan(dtype, b.in, b.out[0], ndim, shape, axis, reverse, trim, pad_lo, pad_hi, bc, fill_value,
                          d_pre, pre_strides, d_post, post_strides, skipna, st);
      };
      return ss.run(es, in, v, 1, outs, &vo, launch);
    }
    const View3 vin = view3(ndim, shape, sd), vout = view3(ndim, out_shape, sd);
    void* outs[1] = {out};
    auto launch = [&](int64_t j0, int64_t j1, int64_t, int64_t, const SlabBufs& b, cudaStream_t st) -> int {
      int64_t sshape[XG_MAX_NDIM];
      for (int d = 0; d < ndim; ++d) sshape[d] = shape[d];
      sshape[sd] = j1 - j0;
      const char* pm = static_cast<const char*>(d_pre);
      const char* qm = static_cast<const char*>(d_post);
      if (pm) pm += (size_t)(j0 * pre_strides[sd]) * es;
      if (qm) qm += (size_t)(j0 * post_strides[sd]) * es;
      return xg_cumscan(dtype, b.in, b.out[0], ndim, sshape, axis, reverse, trim, pad_lo, pad_hi, bc, fill_value, pm,
                        pre_strides, qm, post_strides, skipna, st);
    };
    return ss.run(es, in, vin, 1, outs, &vout, launch, PipeExtra().rows(r0, r1));
  });
}

// ---------------------------------------------------------------------------------------------------
extern "C" int xg_wreduce_host(int dtype, const void* in, const void* weight, const int64_t* w_strides, void* out,
                               int ndim, const int64_t* shape, int axis, int mode, int skipna, int device) {
  if (!in || !out || !shape) return xg_fail(XG_EINVAL, "xg_wreduce_host: null pointer");
  if (dtype != XG_F32 && dtype != XG_F64) return xg_fail(XG_EINVAL, "xg_wreduce_host: dtype must be XG_F32 or XG_F64");
  if (ndim < 1 || ndim > XG_MAX_NDIM) return xg_fail(XG_EINVAL, "xg_wreduce_host: bad ndim");
  if (axis < 0 || axis >= ndim) return xg_fail(XG_EINVAL, "xg_wreduce_host: axis out of range");
  if (weight && !w_strides) return xg_fail(XG_EINVAL, "xg_wreduce_host: weight strides missing");
  const size_t es = dtype == XG_F32 ? 4 : 8;
  const int sd = first_free_dim(ndim, axis);
  return spread("xg_wreduce_host", device, sd < 0 ? 1 : shape[sd], false,
                [&](int dev, int64_t r0, int64_t r1) -> int {
    Session ss;
    int rc = ss.open(dev);
    if (rc) return rc;
    const void* d_w = nullptr;
    if (weight) rc = ss.upload(kAuxPre, weight, operand_span(w_strides, shape, ndim, es), &d_w);
    if (rc) return rc;
    rc = ss.fence();
    if (rc) return rc;
    void* outs[1] = {out};
    if (sd < 0) {
      const View3 v{1, 1, shape[0]}, vo{1, 1, 1};
      auto launch = [&](int64_t, int64_t, int64_t, int64_t, const SlabBufs& b, cudaStream_t st) -> int {
        return xg_wreduce(dtype, b.in, d_w, w_strides, b.out[0], ndim, shape, axis, mode, skipna, st);
      };
      return ss.run(es, in, v, 1, outs, &vo, launch);
    }
    // result shape = shape without `axis`; the slab dim keeps its extent
    int64_t out_shape[XG_MAX_NDIM];
    int nd_o = 0, sd_o = 0;
    for (int d = 0; d < ndim; ++d) {
      if (d == axis) continue;
      if (d == sd) sd_o = nd_o;
      out_shape[nd_o++] = shape[d];
    }
    const View3 vin = view3(ndim, shape, sd), vout = view3(nd_o, out_shape, sd_o);
    auto launch = [&](int64_t j0, int64_t j1, int64_t, int64_t, const SlabBufs& b, cudaStream_t st) -> int {
      int64_t sshape[XG_MAX_NDIM];
      for (int d = 0; d < ndim; ++d) sshape[d] = shape[d];
      sshape[sd] = j1 - j0;
      const char* wm = static_cast<const char*>(d_w);
      if (wm) wm += (size_t)(j0 * w_strides[sd]) * es;
      return xg_wreduce(dtype, b.in, wm, w_strides, b.out[0], ndim, sshape, axis, mode, skipna, st);
    };
    return ss.run(es, in, vin, 1, outs, &vout, launch, PipeExtra().rows(r0, r1));
  });
}

// ---------------------------------------------------------------------------------------------------
extern "C" int xg_wreduce_host_multi(int dtype, const void* in, const void* weight, const int64_t* w_strides,
                                     void* out, int ndim, const int64_t* shape, int naxes, const int* axes, int mode,
                                     int skipna, int device) {
  const std::string who = "xg_wreduce_host_multi";
  if (!in || !out || !shape || !axes) return xg_fail(XG_EINVAL, who + ": null pointer");
  if (dtype != XG_F32 && dtype != XG_F64) return xg_fail(XG_EINVAL, who + ": dtype must be XG_F32 or XG_F64");
  if (ndim < 1 || ndim > XG_MAX_NDIM) return xg_fail(XG_EINVAL, who + ": bad ndim");
  if (naxes < 2 || naxes > ndim)
    return xg_fail(XG_EINVAL, who + ": between 2 and ndim axes (use xg_wreduce_host for one)");
  if (mode != XG_REDUCE_SUM && mode != XG_REDUCE_MEAN)
    return xg_fail(XG_EINVAL, who + ": mode must be XG_REDUCE_SUM or XG_REDUCE_MEAN");
  if (weight && !w_strides) return xg_fail(XG_EINVAL, who + ": weight strides missing");
  bool red[XG_MAX_NDIM] = {false};
  for (int k = 0; k < naxes; ++k) {
    if (axes[k] < 0 || axes[k] >= ndim) return xg_fail(XG_EINVAL, who + ": axis out of range");
    if (red[axes[k]]) return xg_fail(XG_EINVAL, who + ": an axis may appear only once");
    red[axes[k]] = true;
  }
  for (int d = 0; d < ndim; ++d) {
    if (shape[d] < 0) return xg_fail(XG_EINVAL, who + ": negative extent");
    if (weight && w_strides[d] < 0) return xg_fail(XG_EINVAL, who + ": negative weight stride");
  }
  int64_t out_numel = 1;
  for (int d = 0; d < ndim; ++d)
    if (!red[d]) out_numel *= shape[d];
  if (out_numel == 0) return XG_OK;
  for (int d = 0; d < ndim; ++d)
    if (red[d] && shape[d] == 0) return xg_fail(XG_ENOTIMPL, who + ": empty reduced dim; use xg_wreduce");
  const bool mean = mode == XG_REDUCE_MEAN;
  const int mult = mean ? 2 : 1;  // a mean carries the sum and the valid weights side by side
  const size_t es = dtype == XG_F32 ? 4 : 8;

  // The launches of Grid.integrate / average on the device: one xg_wreduce per dim, innermost first, the weight in
  // the first one only; a mean reduces sum and valid weights (WVALID) side by side, then divides once (DIVNZ).
  int ord[XG_MAX_NDIM];
  int nord = 0;
  for (int d = ndim - 1; d >= 0; --d)
    if (red[d]) ord[nord++] = d;
  // Slab dim: the outermost non-reduced dim of extent > 1; every launch runs per slab.  With none (`whole`), slabs
  // of the outermost dim of extent > 1 run the launches along the dims inside it; their partials, one value per
  // index of the slab dim, stay on the device, and the launches along the slab dim and the extent-1 dims in front
  // of it run once at the end.
  int sd = -1;
  for (int d = 0; d < ndim && sd < 0; ++d)
    if (!red[d] && shape[d] > 1) sd = d;
  const bool whole = sd < 0;
  for (int d = 0; d < ndim && sd < 0; ++d)
    if (shape[d] > 1) sd = d;
  if (sd < 0) sd = 0;
  int nslab = nord;  // launches (per chain) that run per slab
  if (whole) {
    nslab = 0;
    while (nslab < nord && ord[nslab] > sd) ++nslab;
    if (nslab == 0)
      return xg_fail(XG_ENOTIMPL, who + ": no reduced dim of extent > 1 inside the slab dim; use xg_wreduce_host");
  }
  const int64_t L = shape[sd];
  // elements per slab row of each per-slab launch's result, and of the scratch that holds them
  int64_t rowel[XG_MAX_NDIM], scratch_el = 0;
  {
    int64_t c[XG_MAX_NDIM];
    for (int d = 0; d < ndim; ++d) c[d] = shape[d];
    c[sd] = 1;
    int cn = ndim;
    for (int k = 0; k < nslab; ++k) {
      for (int d = ord[k]; d + 1 < cn; ++d) c[d] = c[d + 1];
      rowel[k] = numel(--cn, c);
      if (k < nslab - 1 || (!whole && mean)) scratch_el += mult * rowel[k];
    }
  }
  // the weight: streamed beside the field when it spans the slab dim (a dense array of its own extents), else whole
  int64_t wshape[XG_MAX_NDIM];  // its own extents: 1 where it is broadcast
  if (weight) compact_shape(ndim, shape, w_strides, wshape);
  const bool stream_w = weight && wshape[sd] > 1 && is_dense(ndim, wshape, w_strides);

  const View3 vin = view3(ndim, shape, sd);
  View3 vout{1, L, 1};
  if (!whole) {
    int64_t oshape[XG_MAX_NDIM];
    int nd_o = 0, sd_o = 0;
    for (int d = 0; d < ndim; ++d) {
      if (red[d]) continue;
      if (d == sd) sd_o = nd_o;
      oshape[nd_o++] = shape[d];
    }
    vout = view3(nd_o, oshape, sd_o);
  }
  PipeExtra ex;
  if (stream_w) {
    ex.hin2 = weight;
    ex.in2 = view3(ndim, wshape, sd);
  }
  ex.scratch_row_bytes = (size_t)scratch_el * es;
  ex.row_bytes = (vin.C * vin.R + (stream_w ? ex.in2.C * ex.in2.R : 0) + scratch_el +
                  (whole ? 0 : vout.C * vout.R)) * (int64_t)es;

  // `whole` keeps its partials along the slab dim on one device: it runs on a group's first member alone
  return spread(who.c_str(), device, L, false, [&](int dev, int64_t r0, int64_t r1) -> int {
    Session ss;
    int rc = ss.open(dev);
    if (rc) return rc;
    const void* d_w = nullptr;
    if (weight && !stream_w) rc = ss.upload(kAuxPre, weight, operand_span(w_strides, shape, ndim, es), &d_w);
    if (rc) return rc;
    rc = ss.fence();
    if (rc) return rc;
    // `whole`: [sum partials (L)][valid-weight partials (L)], the results of the last launches, the mean
    char* partial = nullptr;
    int64_t partial_el = mult * L + 1;
    if (whole) {
      int64_t c[XG_MAX_NDIM];
      for (int d = 0; d < ndim; ++d) c[d] = shape[d];
      int cn = ndim;
      for (int k = 0; k < nord; ++k) {
        for (int d = ord[k]; d + 1 < cn; ++d) c[d] = c[d + 1];
        if (k >= nslab) partial_el += mult * numel(cn - 1, c);
        --cn;
      }
      void* p = nullptr;
      rc = ss.aux(kAuxPartial, (size_t)partial_el * es, &p);
      if (rc) return rc;
      partial = static_cast<char*>(p);
    }
    // launches k0 .. k1 - 1 of the chain on `cur` (cnd dims), from num_in (den_in: the valid weights of a mean), the
    // weight with launch 0; the results of each go to the next free `scratch` elements, or to num_last / den_last
    // for the last one when they are given
    auto chain = [&](int k0, int k1, int64_t* cur, int cnd, const void* num_in, const void* den_in, const void* wp,
                     const int64_t* ws, char* scratch, void* num_last, void* den_last, const void** num_out,
                     const void** den_out, cudaStream_t st) -> int {
      for (int k = k0; k < k1; ++k) {
        const int64_t count = numel(cnd, cur) / cur[ord[k]];
        void* nd = num_last;
        void* dd = den_last;
        if (k < k1 - 1 || !num_last) {
          nd = scratch;
          dd = mean ? scratch + (size_t)count * es : nullptr;
          scratch += (size_t)(mult * count) * es;
        }
        int rc2;
        if (k == 0) {
          rc2 = mean ? xg_wreduce(dtype, num_in, wp, ws, dd, cnd, cur, ord[k], XG_REDUCE_WVALID, skipna, st) : XG_OK;
          if (rc2 == XG_OK) rc2 = xg_wreduce(dtype, num_in, wp, ws, nd, cnd, cur, ord[k], XG_REDUCE_SUM, skipna, st);
        } else {
          rc2 = xg_wreduce(dtype, num_in, nullptr, nullptr, nd, cnd, cur, ord[k], XG_REDUCE_SUM, skipna, st);
          if (rc2 == XG_OK && mean)
            rc2 = xg_wreduce(dtype, den_in, nullptr, nullptr, dd, cnd, cur, ord[k], XG_REDUCE_SUM, 0, st);
        }
        if (rc2) return rc2;
        num_in = nd;
        den_in = dd;
        for (int d = ord[k]; d + 1 < cnd; ++d) cur[d] = cur[d + 1];
        --cnd;
      }
      *num_out = num_in;
      *den_out = den_in;
      return XG_OK;
    };
    // the mean: sum / valid weights, NaN where no weight is valid
    auto divide = [&](const void* num, const void* den, void* res, int64_t count, cudaStream_t st) -> int {
      const int64_t one = 1;
      return xg_binary(XG_BIN_DIVNZ, dtype, num, den, &one, res, 1, &count, st);
    };
    auto launch = [&](int64_t j0, int64_t j1, int64_t, int64_t, const SlabBufs& b, cudaStream_t st) -> int {
      const int64_t rows = j1 - j0;
      int64_t cur[XG_MAX_NDIM], ws[XG_MAX_NDIM];
      for (int d = 0; d < ndim; ++d) cur[d] = shape[d];
      cur[sd] = rows;
      const void* wp = nullptr;
      if (stream_w) {  // the slab's own dense layout
        int64_t c[XG_MAX_NDIM];
        for (int d = 0; d < ndim; ++d) c[d] = wshape[d];
        c[sd] = rows;
        dense_strides(ndim, c, ws);
        for (int d = 0; d < ndim; ++d)
          if (c[d] == 1) ws[d] = 0;
        wp = b.in2;
      } else if (d_w) {
        for (int d = 0; d < ndim; ++d) ws[d] = w_strides[d];
        wp = static_cast<const char*>(d_w) + (size_t)(j0 * w_strides[sd]) * es;
      }
      void* num_last = whole ? partial + (size_t)j0 * es : (mean ? nullptr : b.out[0]);
      void* den_last = whole && mean ? partial + (size_t)(L + j0) * es : nullptr;
      const void *num, *den;
      int rc2 = chain(0, nslab, cur, ndim, b.in, nullptr, wp, wp ? ws : nullptr, static_cast<char*>(b.scratch),
                      num_last, den_last, &num, &den, st);
      if (rc2 || whole || !mean) return rc2;
      return divide(num, den, b.out[0], rows * rowel[nslab - 1], st);
    };
    if (!whole) return ss.run(es, in, vin, 1, &out, &vout, launch, ex.rows(r0, r1));
    rc = ss.run(es, in, vin, 0, nullptr, &vout, launch, ex);
    if (rc) return rc;
    // the launches along the slab dim and the dims in front of it, once, on the partials
    int64_t cur[XG_MAX_NDIM];
    int cnd = 0;
    for (int d = 0; d < ndim; ++d)
      if (!(red[d] && d > sd)) cur[cnd++] = shape[d];
    const void *num, *den;
    char* next = partial + (size_t)(mult * L) * es;
    rc = chain(nslab, nord, cur, cnd, partial, mean ? partial + (size_t)L * es : nullptr, nullptr, nullptr, next,
               nullptr, nullptr, &num, &den, ss.kernel_stream());
    if (rc) return rc;
    if (mean) {
      void* res = partial + (size_t)(partial_el - 1) * es;  // the last element
      rc = divide(num, den, res, 1, ss.kernel_stream());
      if (rc) return rc;
      num = res;
    }
    return ss.download(out, num, es);
  }, !whole);
}

// ---------------------------------------------------------------------------------------------------
extern "C" int xg_vinterp_linear_host(int dtype, const void* phi, const void* theta, const int64_t* theta_strides,
                                      const void* target, const int64_t* target_strides, int64_t m, void* out,
                                      int ndim, const int64_t* shape, int axis, int mask_edges, int bypass_checks,
                                      int logarithmic, int device) {
  if (!phi || !theta || !theta_strides || !target || !out || !shape)
    return xg_fail(XG_EINVAL, "xg_vinterp_linear_host: null pointer");
  if (dtype != XG_F32 && dtype != XG_F64)
    return xg_fail(XG_EINVAL, "xg_vinterp_linear_host: dtype must be XG_F32 or XG_F64");
  if (ndim < 1 || ndim > XG_MAX_NDIM) return xg_fail(XG_EINVAL, "xg_vinterp_linear_host: bad ndim");
  if (axis < 0 || axis >= ndim) return xg_fail(XG_EINVAL, "xg_vinterp_linear_host: axis out of range");
  if (m < 0) return xg_fail(XG_EINVAL, "xg_vinterp_linear_host: negative number of target levels");
  const size_t es = dtype == XG_F32 ? 4 : 8;
  // theta: a dense field streams beside phi, a broadcast one is uploaded whole; target whole
  ThetaPlan plan;
  plan_theta(&plan, dtype, theta_strides, 0, shape[axis], ndim, shape, axis);
  const TransformViews tv = transform_views(ndim, shape, axis, m, plan, theta);
  plan.sd = tv.sd;
  return spread("xg_vinterp_linear_host", device, tv.sd >= 0 ? shape[tv.sd] : 1, false,
                [&](int dev, int64_t r0, int64_t r1) -> int {
    Session ss;
    int rc = ss.open(dev);
    if (rc) return rc;
    ThetaPlan tp = plan;
    rc = upload_theta(ss, &tp, theta, theta_strides);
    if (rc) return rc;
    const void* d_target = nullptr;
    int64_t tshape[XG_MAX_NDIM];
    for (int d = 0; d < ndim; ++d) tshape[d] = shape[d];
    tshape[axis] = m;
    const size_t tbytes = target_strides ? operand_span(target_strides, tshape, ndim, es) : (size_t)m * es;
    rc = ss.upload(kAuxTarget, target, tbytes ? tbytes : es, &d_target);
    if (rc) return rc;
    rc = ss.fence();
    if (rc) return rc;
    void* outs[1] = {out};
    auto launch = [&](int64_t j0, int64_t j1, int64_t, int64_t, const SlabBufs& b, cudaStream_t st) -> int {
      int64_t sshape[XG_MAX_NDIM], th_strides[XG_MAX_NDIM];
      for (int d = 0; d < ndim; ++d) sshape[d] = shape[d];
      const char* tg = static_cast<const char*>(d_target);
      if (tv.sd >= 0) {
        sshape[tv.sd] = j1 - j0;
        if (target_strides) tg += (size_t)(j0 * target_strides[tv.sd]) * es;
      }
      const void* th = nullptr;
      const int rc2 = tp.slab(j0, j1, b, st, &th, th_strides);
      if (rc2) return rc2;
      return xg_vinterp_linear(dtype, b.in, th, th_strides, tg, target_strides, m, b.out[0], ndim, sshape, axis,
                               mask_edges, bypass_checks, logarithmic, st);
    };
    return ss.run(es, phi, tv.vin, 1, outs, &tv.vout, launch, tv.ex.rows(r0, r1));
  });
}

// ---------------------------------------------------------------------------------------------------
extern "C" int xg_vinterp_conservative_host(int dtype, const void* phi, const void* theta,
                                            const int64_t* theta_strides, int theta_at_centers,
                                            const void* target_bins, int64_t m, int flip_out, void* out, int ndim,
                                            const int64_t* shape, int axis, int device) {
  if (!phi || !theta || !target_bins || !out || !shape)
    return xg_fail(XG_EINVAL, "xg_vinterp_conservative_host: null pointer");
  if (!theta_strides) return xg_fail(XG_EINVAL, "xg_vinterp_conservative_host: theta strides missing");
  if (dtype != XG_F32 && dtype != XG_F64)
    return xg_fail(XG_EINVAL, "xg_vinterp_conservative_host: dtype must be XG_F32 or XG_F64");
  if (ndim < 1 || ndim > XG_MAX_NDIM) return xg_fail(XG_EINVAL, "xg_vinterp_conservative_host: bad ndim");
  if (axis < 0 || axis >= ndim) return xg_fail(XG_EINVAL, "xg_vinterp_conservative_host: axis out of range");
  for (int d = 0; d < ndim; ++d)
    if (shape[d] < 0) return xg_fail(XG_EINVAL, "xg_vinterp_conservative_host: negative extent");
  if (m < 2) return xg_fail(XG_EINVAL, "xg_vinterp_conservative_host: need at least two bin edges");
  const int64_t n = shape[axis];
  int64_t tshape[XG_MAX_NDIM];
  for (int d = 0; d < ndim; ++d) tshape[d] = shape[d];
  tshape[axis] = theta_at_centers ? n : n + 1;
  int rc = check_theta("xg_vinterp_conservative_host", ndim, tshape, theta_strides, axis, theta_at_centers);
  if (rc) return rc;
  const size_t es = dtype == XG_F32 ? 4 : 8;
  int64_t ncols = 1;
  for (int d = 0; d < ndim; ++d)
    if (d != axis) ncols *= shape[d];
  if (ncols == 0) return XG_OK;
  if (n == 0) {  // no source cells: every bin receives nothing and stays NaN, as in k_vconserv
    const int64_t count = ncols * (m - 1);
    if (dtype == XG_F32)
      for (int64_t i = 0; i < count; ++i) static_cast<float*>(out)[i] = NAN;
    else
      for (int64_t i = 0; i < count; ++i) static_cast<double*>(out)[i] = NAN;
    return XG_OK;
  }
  // theta: streamed (dense) or whole (its bounds made on the device at centres); bins whole
  ThetaPlan plan;
  plan_theta(&plan, dtype, theta_strides, theta_at_centers, tshape[axis], ndim, shape, axis);
  const TransformViews tv = transform_views(ndim, shape, axis, m - 1, plan, theta);
  plan.sd = tv.sd;
  return spread("xg_vinterp_conservative_host", device, tv.sd >= 0 ? shape[tv.sd] : 1, false,
                [&](int dev, int64_t r0, int64_t r1) -> int {
    Session ss;
    int rc = ss.open(dev);
    if (rc) return rc;
    ThetaPlan tp = plan;
    rc = upload_theta(ss, &tp, theta, theta_strides);
    if (rc) return rc;
    const void* d_bins = nullptr;
    rc = ss.upload(kAuxTarget, target_bins, (size_t)m * es, &d_bins);
    if (rc) return rc;
    rc = ss.fence();
    if (rc) return rc;
    rc = plan_theta_bounds(ss, &tp, theta_strides);
    if (rc) return rc;
    void* outs[1] = {out};
    auto launch = [&](int64_t j0, int64_t j1, int64_t, int64_t, const SlabBufs& b, cudaStream_t st) -> int {
      int64_t sshape[XG_MAX_NDIM], th_strides[XG_MAX_NDIM];
      for (int d = 0; d < ndim; ++d) sshape[d] = shape[d];
      if (tv.sd >= 0) sshape[tv.sd] = j1 - j0;
      const void* th = nullptr;
      const int rc2 = tp.slab(j0, j1, b, st, &th, th_strides);
      if (rc2) return rc2;
      return xg_vinterp_conservative(dtype, b.in, th, th_strides, d_bins, m, flip_out, b.out[0], ndim, sshape, axis,
                                     st);
    };
    return ss.run(es, phi, tv.vin, 1, outs, &tv.vout, launch, tv.ex.rows(r0, r1));
  });
}
