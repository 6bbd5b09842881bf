// xg_stencil2_host — the fused stencil on HOST buffers, streamed through the GPU.
//
// This is the call the reference-facing API makes for numpy-backed fields: the
// whole of xgcm/padding.py:575-616 + gridops.py + the metric passes for one axis,
// with host<->device copies inside.  The field is cut into slabs along dim 0
// (contiguous in host memory).  Three streams form a pipeline
//     H2D(slab s+1)  ||  kernel(slab s)  ||  D2H(slab s-1)
// so PCIe runs full duplex and the kernel time hides entirely behind the copies.
// When dim 0 is the operated axis the slabs overlap by the one-cell halo and the
// exterior halo plane (periodic wrap) is uploaded once.
//
// xg_stencil2_host_fold / xg_stencil2_host_connected run the same slab loop with a per-slab halo stage
// on the kernel stream: the slab's halo_lo / halo_hi planes are built from the slab buffers (one
// xg_fold_rows launch, or the face-connection copy list clipped to the slab and replayed with
// xg_strided_copy_batch) just before its xg_stencil2 launch.  Dim 0 is then a batch dim, so the planes
// of one slab depend on that slab (and the partner component's slab) alone.
//
// xg_stencil_pair_host / xg_stencil_pair_host_fold run the two-field composite on the same loop: field a
// is the slab input, field b streams through the partner slots, and each slab is one xg_stencil_pair_halo
// launch (after the xg_fold_rows launch of b's folded row, for the fold).
//
// Workspace (device slabs + events + streams) is cached per device and reused;
// xg_host_workspace_release() frees it.
#include <stdlib.h>

#include <mutex>
#include <vector>

#include "xg_common.cuh"

namespace {

constexpr int kSlots = 3;

struct Workspace {
  int device = -1;
  std::mutex mu;  // one host call at a time per device; different devices run concurrently
  size_t slab_in_bytes = 0, slab_out_bytes = 0, metric_bytes[3] = {0, 0, 0}, halo_bytes = 0;
  size_t partner_bytes = 0, const_bytes = 0;
  void* d_in[kSlots] = {nullptr, nullptr, nullptr};
  void* d_out[kSlots] = {nullptr, nullptr, nullptr};
  void* d_partner[kSlots] = {nullptr, nullptr, nullptr};  // second vector component, or field b of a pair
  void* d_metric[3] = {nullptr, nullptr, nullptr};       // pre, post, and pre_a of a pair
  void* d_halo[2] = {nullptr, nullptr};  // wrap planes along dim 0, or the per-slab lo / hi halo planes
  void* d_const = nullptr;               // the fill constant the unconnected face edges copy from
  cudaStream_t s_h2d = nullptr, s_k = nullptr, s_d2h = nullptr;
  cudaEvent_t e_up[kSlots], e_done[kSlots], e_down[kSlots];
  bool events = false;
};

std::mutex g_ws_mutex;
std::vector<Workspace*> g_ws;

#define XG_CUDA(call)                                                                   \
  do {                                                                                  \
    cudaError_t e_ = (call);                                                            \
    if (e_ != cudaSuccess)                                                              \
      return xg_fail(XG_ECUDA, std::string(#call) + ": " + cudaGetErrorString(e_));     \
  } while (0)

int ensure(void** p, size_t* have, size_t want) {
  if (*have >= want && *p) return XG_OK;
  if (*p) XG_CUDA(cudaFree(*p));
  *p = nullptr;
  *have = 0;
  if (want == 0) return XG_OK;
  XG_CUDA(cudaMalloc(p, want));
  *have = want;
  return XG_OK;
}

int get_workspace(int device, Workspace** out) {
  for (Workspace* w : g_ws)
    if (w->device == device) {
      *out = w;
      return XG_OK;
    }
  Workspace* w = new Workspace();
  w->device = device;
  XG_CUDA(cudaStreamCreateWithFlags(&w->s_h2d, cudaStreamNonBlocking));
  XG_CUDA(cudaStreamCreateWithFlags(&w->s_k, cudaStreamNonBlocking));
  XG_CUDA(cudaStreamCreateWithFlags(&w->s_d2h, cudaStreamNonBlocking));
  for (int i = 0; i < kSlots; ++i) {
    XG_CUDA(cudaEventCreateWithFlags(&w->e_up[i], cudaEventDisableTiming));
    XG_CUDA(cudaEventCreateWithFlags(&w->e_done[i], cudaEventDisableTiming));
    XG_CUDA(cudaEventCreateWithFlags(&w->e_down[i], cudaEventDisableTiming));
  }
  w->events = true;
  g_ws.push_back(w);
  *out = w;
  return XG_OK;
}

// bytes spanned by a broadcast operand laid out with `strides` over `shape`
size_t operand_span(const int64_t* strides, const int64_t* shape, int ndim, size_t es) {
  int64_t last = 0;
  for (int d = 0; d < ndim; ++d)
    if (shape[d] > 1) last += (shape[d] - 1) * strides[d];
  return (size_t)(last + 1) * es;
}

}  // namespace

void xg_host_pipe_release();  // xg_host_pipe.cu

extern "C" int xg_host_workspace_release(void) {
  xg_host_pipe_release();
  std::lock_guard<std::mutex> lock(g_ws_mutex);
  for (Workspace* w : g_ws) {
    cudaSetDevice(w->device);
    for (int i = 0; i < kSlots; ++i) {
      if (w->d_in[i]) cudaFree(w->d_in[i]);
      if (w->d_out[i]) cudaFree(w->d_out[i]);
      if (w->d_partner[i]) cudaFree(w->d_partner[i]);
      if (w->events) {
        cudaEventDestroy(w->e_up[i]);
        cudaEventDestroy(w->e_done[i]);
        cudaEventDestroy(w->e_down[i]);
      }
    }
    for (int i = 0; i < 3; ++i)
      if (w->d_metric[i]) cudaFree(w->d_metric[i]);
    for (int i = 0; i < 2; ++i)
      if (w->d_halo[i]) cudaFree(w->d_halo[i]);
    if (w->d_const) cudaFree(w->d_const);
    if (w->s_h2d) cudaStreamDestroy(w->s_h2d);
    if (w->s_k) cudaStreamDestroy(w->s_k);
    if (w->s_d2h) cudaStreamDestroy(w->s_d2h);
    delete w;
  }
  g_ws.clear();
  return XG_OK;
}

namespace {

// The x term and the second field of xg_stencil_pair_host.  Its Call describes the term along `axis`
// (op_b, lo_b, hi_b, bc_b, fill_b, pre_b) and `post`, and its `in` is field a, the slab input.
struct PairTerm {
  const void* b;
  int op_a, lo_a, hi_a, bc_a;
  double fill_a;
  const void* pre_a;
  const int64_t* pre_a_strides;
  int subtract;
};

// The stencil call the slab loop runs, slab by slab.
struct Call {
  int op, dtype;
  const void* in;
  void* out;
  int ndim;
  const int64_t* shape;
  int axis, lo, hi, bc;
  double fill_value;
  const void* pre;
  const int64_t* pre_strides;
  const void* post;
  const int64_t* post_strides;
  int device;
  const PairTerm* pair = nullptr;  // xg_stencil_pair_halo instead of xg_stencil2
};

enum { kHaloNone = 0, kHaloFold = 1, kHaloCopies = 2 };
enum { kSrcField = 0, kSrcPartner = 1, kSrcFill = 2 };

// What builds a slab's halo planes on s_k before its xg_stencil2 launch (none for xg_stencil2_host).
struct HaloStage {
  int kind = kHaloNone;
  // kHaloFold: the folded north row of the slab is halo_hi, and halo_lo when the south edge is periodic
  int seam_axis = 0, skip = 0, negate = 0;
  int64_t mirror = 0, period = 1;
  // kHaloCopies: strided copies into the lo / hi planes, described once for the whole field (dim-0 extent n0)
  const void* partner = nullptr;
  int64_t partner_row = 0;  // partner elements per dim-0 index
  int ncopies = 0, cndim = 0;
  const int *side = nullptr, *source = nullptr, *negate_c = nullptr;
  const int64_t *dst_offset = nullptr, *src_offset = nullptr, *shapes = nullptr;
  const int64_t *dst_strides = nullptr, *src_strides = nullptr;
};

// Argument checks shared by the host stencil entry points; no CUDA call.
int validate_call(const char* who, const Call& c) {
  const std::string w(who);
  if (!c.in || !c.out || !c.shape) return xg_fail(XG_EINVAL, w + ": null pointer");
  if (c.dtype != XG_F32 && c.dtype != XG_F64)
    return xg_fail(XG_EINVAL, w + ": dtype must be XG_F32 or XG_F64");
  if (c.ndim < 1 || c.ndim > XG_MAX_NDIM) return xg_fail(XG_EINVAL, w + ": bad ndim");
  if (c.axis < 0 || c.axis >= c.ndim) return xg_fail(XG_EINVAL, w + ": axis out of range");
  if (c.lo < 0 || c.lo > 1 || c.hi < 0 || c.hi > 1)
    return xg_fail(XG_EINVAL, w + ": halo widths must be 0 or 1");
  if ((c.lo || c.hi) && (c.bc <= XG_BC_NONE || c.bc > XG_BC_EXTRAPOLATE))
    return xg_fail(XG_EINVAL, w + ": no boundary condition was specified but the operation needs to pad the axis");
  if (c.shape[c.axis] == 0) return xg_fail(XG_EINVAL, w + ": empty operated axis");
  if ((c.pre && !c.pre_strides) || (c.post && !c.post_strides))
    return xg_fail(XG_EINVAL, w + ": metric strides missing");
  if (c.axis == 0 && c.bc == XG_BC_PERIODIC && c.pre)
    return xg_fail(XG_ENOTIMPL, w + ": periodic halo with a pre-metric along the outermost axis; "
                                    "use the device entry point");
  return XG_OK;
}

// The halo entry points build their planes per slab: dim 0 must be a batch dim the halo does not touch.
int validate_halo_call(const char* who, const Call& c) {
  int rc = validate_call(who, c);
  if (rc) return rc;
  if (c.ndim < 2 || c.axis == 0)
    return xg_fail(XG_EINVAL, std::string(who) + ": dim 0 is cut into slabs and must not be the operated dim");
  for (int d = 0; d < c.ndim; ++d)
    if (c.shape[d] < 0) return xg_fail(XG_EINVAL, std::string(who) + ": negative extent");
  return XG_OK;
}

// The fold parameters of the _fold entry points (the checks xg_fold_rows makes, before any CUDA call).
int validate_fold(const char* who, const Call& c, int seam_axis, int skip, int64_t mirror, int64_t period) {
  const std::string w(who);
  if (seam_axis < 0 || seam_axis >= c.ndim) return xg_fail(XG_EINVAL, w + ": seam axis out of range");
  if (seam_axis == 0) return xg_fail(XG_EINVAL, w + ": dim 0 is cut into slabs and must not be the seam dim");
  if (seam_axis == c.axis) return xg_fail(XG_EINVAL, w + ": the fold and seam axes must differ");
  if (c.hi != 1) return xg_fail(XG_EINVAL, w + ": the fold is the upper halo: hi must be 1");
  if (skip < 0 || skip > 1) return xg_fail(XG_EINVAL, w + ": skip must be 0 or 1");
  if (c.shape[c.axis] - skip < 1)
    return xg_fail(XG_EINVAL, w + ": halo width exceeds the interior rows of the fold axis");
  if (period < 1) return xg_fail(XG_EINVAL, w + ": period must be positive");
  for (int64_t k = 0; k < c.shape[seam_axis]; ++k) {
    int64_t src = (mirror - k) % period;
    if (src < 0) src += period;
    if (src >= c.shape[seam_axis])
      return xg_fail(XG_ENOTIMPL, w + ": seam position incompatible with the pivot: the mirror "
                                      "partner of a seam index lies outside the seam dim");
  }
  return XG_OK;
}

// The checks xg_stencil_pair makes, plus those of the slab loop (dim 0 a batch dim), before any CUDA call.
int validate_pair_call(const char* who, const Call& c) {
  const std::string w(who);
  const PairTerm& t = *c.pair;
  if (!t.b) return xg_fail(XG_EINVAL, w + ": null pointer");
  int rc = validate_halo_call(who, c);
  if (rc) return rc;
  if (c.axis >= c.ndim - 1) return xg_fail(XG_EINVAL, w + ": axis_b must be a dimension other than the innermost one");
  if (t.lo_a < 0 || t.hi_a < 0 || t.lo_a + t.hi_a != 1 || c.lo + c.hi != 1)
    return xg_fail(XG_ENOTIMPL, w + ": both stencils must be length preserving (lo + hi == 1)");
  for (int bc : {t.bc_a, c.bc})
    if (bc < XG_BC_PERIODIC || bc > XG_BC_EXTEND)
      return xg_fail(XG_EINVAL, w + ": boundary must be periodic, fill or extend");
  for (int op : {t.op_a, c.op})
    if (op < XG_OP_DIFF || op > XG_OP_MAX) return xg_fail(XG_EINVAL, w + ": unknown op");
  if (t.pre_a && !t.pre_a_strides) return xg_fail(XG_EINVAL, w + ": metric strides missing");
  if (t.subtract < 0 || t.subtract > 2) return xg_fail(XG_EINVAL, w + ": subtract must be 0, 1 or 2");
  if (c.in == c.out || t.b == c.out) return xg_fail(XG_EINVAL, w + ": in-place operation is not supported");
  return XG_OK;
}

// Per-slab face-connection copies: rebase the whole-field copy list onto the slab buffers, `rows` high.
int halo_copies(const HaloStage& h, int dtype, size_t es, void* const planes[2], const void* field,
                const void* partner, const void* fill, int64_t rows, std::vector<void*>& dptr,
                std::vector<const void*>& sptr, std::vector<int64_t>& shp, cudaStream_t st) {
  for (int k = 0; k < h.ncopies; ++k) {
    dptr[k] = (char*)planes[h.side[k]] + (size_t)h.dst_offset[k] * es;
    const void* base = h.source[k] == kSrcField ? field : h.source[k] == kSrcPartner ? partner : fill;
    sptr[k] = (const char*)base + (size_t)h.src_offset[k] * es;
    shp[(size_t)k * h.cndim] = rows;
  }
  int rc = xg_strided_copy_batch(dtype, h.ncopies, dptr.data(), sptr.data(), h.cndim, shp.data(),
                                 h.dst_strides, h.src_strides, h.negate_c, st);
  if (rc != XG_ENOTIMPL) return rc;
  for (int k = 0; k < h.ncopies; ++k) {  // some copy does not collapse to 5 dims: one launch per copy
    rc = xg_strided_copy(dtype, dptr[k], h.dst_strides + (size_t)k * h.cndim, sptr[k],
                         h.src_strides + (size_t)k * h.cndim, h.cndim, shp.data() + (size_t)k * h.cndim,
                         h.negate_c[k], st);
    if (rc) return rc;
  }
  return XG_OK;
}

// The slab loop of every host stencil entry point (arguments already validated).
int run_slabs(const Call& c, const HaloStage& h) {
  const int ndim = c.ndim, axis = c.axis, lo = c.lo, hi = c.hi, bc = c.bc;
  const int64_t* shape = c.shape;
  const size_t es = c.dtype == XG_F32 ? 4 : 8;
  XG_CUDA(cudaSetDevice(c.device));
  Workspace* w = nullptr;
  int rc;
  {
    std::lock_guard<std::mutex> reg(g_ws_mutex);  // registry only
    rc = get_workspace(c.device, &w);
  }
  if (rc) return rc;
  std::lock_guard<std::mutex> lock(w->mu);

  int64_t out_shape[XG_MAX_NDIM];
  for (int d = 0; d < ndim; ++d) out_shape[d] = shape[d];
  out_shape[axis] = shape[axis] + lo + hi - 1;
  int64_t row_in = 1, row_out = 1;  // elements per index of dim 0
  for (int d = 1; d < ndim; ++d) {
    row_in *= shape[d];
    row_out *= out_shape[d];
  }
  const int64_t n0_out = out_shape[0];
  if (n0_out <= 0 || row_out == 0 || row_in == 0) return XG_OK;
  const void* partner = c.pair ? c.pair->b : h.partner;
  const int64_t partner_row = c.pair ? row_in : h.partner_row;
  const bool ax0 = axis == 0;

  // slab height along dim 0: ~128 MiB of input per slab, at least 4 slabs if possible
  int64_t target_bytes = 128ll << 20;
  if (const char* env = getenv("XG_HOST_SLAB_MB")) {  // tuning knob (benchmarks only)
    const long mb = atol(env);
    if (mb >= 1 && mb <= 4096) target_bytes = (int64_t)mb << 20;
  }
  int64_t rows = target_bytes / (int64_t)(row_in * es);
  if (rows < 1) rows = 1;
  if (rows > (n0_out + 3) / 4) rows = (n0_out + 3) / 4;
  if (rows < 1) rows = 1;
  if (ax0 && bc == XG_BC_EXTRAPOLATE && (lo || hi)) {
    // the extrapolated halo is 2 A[edge] - A[next]: the slab that touches an edge of the axis must hold two
    // source planes, i.e. no one-row slab at either end (a one-row tail is merged by growing the slab height)
    if (rows < 2) rows = 2;
    while (rows < n0_out && n0_out % rows == 1) ++rows;
    if (rows > n0_out) rows = n0_out;
  }
  const int64_t nslab = xg_ceil_div(n0_out, rows);
  const int64_t in_rows_max = ax0 ? rows + 1 : rows;

  for (int i = 0; i < kSlots; ++i) {
    size_t have_in = w->slab_in_bytes, have_out = w->slab_out_bytes, have_p = w->partner_bytes;
    rc = ensure(&w->d_in[i], &have_in, (size_t)(in_rows_max * row_in) * es);
    if (rc) return rc;
    rc = ensure(&w->d_out[i], &have_out, (size_t)(rows * row_out) * es);
    if (rc) return rc;
    if (partner) {
      rc = ensure(&w->d_partner[i], &have_p, (size_t)(rows * partner_row) * es);
      if (rc) return rc;
    }
    if (i == kSlots - 1) {
      w->slab_in_bytes = have_in;
      w->slab_out_bytes = have_out;
      w->partner_bytes = have_p;
    }
  }
  // (all three slots share one recorded capacity: grow them together)
  // metrics: uploaded whole, once
  const void* hm[3] = {c.pre, c.post, c.pair ? c.pair->pre_a : nullptr};
  const int64_t* ms[3] = {c.pre_strides, c.post_strides, c.pair ? c.pair->pre_a_strides : nullptr};
  const int64_t* mshape[3] = {shape, out_shape, shape};
  for (int k = 0; k < 3; ++k) {
    if (!hm[k]) continue;
    const size_t span = operand_span(ms[k], mshape[k], ndim, es);
    rc = ensure(&w->d_metric[k], &w->metric_bytes[k], span);
    if (rc) return rc;
    XG_CUDA(cudaMemcpyAsync(w->d_metric[k], hm[k], span, cudaMemcpyHostToDevice, w->s_h2d));
  }
  // exterior halo planes when dim 0 is the operated axis and the halo is data (periodic wrap)
  const char* hin = static_cast<const char*>(c.in);
  char* hout = static_cast<char*>(c.out);
  const int64_t n0 = shape[0];
  const bool wrap_planes = ax0 && bc == XG_BC_PERIODIC && c.pre == nullptr;
  if (wrap_planes) {
    size_t hb = w->halo_bytes;
    for (int k = 0; k < 2; ++k) {
      size_t have = hb;
      rc = ensure(&w->d_halo[k], &have, (size_t)row_in * es);
      if (rc) return rc;
      if (k == 1) w->halo_bytes = have;
    }
    if (lo)  // below the first plane sits the last plane
      XG_CUDA(cudaMemcpyAsync(w->d_halo[0], hin + (size_t)(n0 - 1) * row_in * es, row_in * es,
                              cudaMemcpyHostToDevice, w->s_h2d));
    if (hi)
      XG_CUDA(cudaMemcpyAsync(w->d_halo[1], hin, row_in * es, cudaMemcpyHostToDevice, w->s_h2d));
  }
  // per-slab halo planes (dim 0 is not the operated axis): one pair, built and read in order on s_k
  std::vector<void*> dptr(h.ncopies);
  std::vector<const void*> sptr(h.ncopies);
  std::vector<int64_t> shp(h.shapes ? h.shapes : (const int64_t*)nullptr,
                           h.shapes ? h.shapes + (size_t)h.ncopies * h.cndim : (const int64_t*)nullptr);
  if (h.kind != kHaloNone) {
    const int64_t plane_row = row_in / shape[axis];
    size_t hb = w->halo_bytes;
    for (int k = 0; k < 2; ++k) {
      size_t have = hb;
      rc = ensure(&w->d_halo[k], &have, (size_t)(rows * plane_row) * es);
      if (rc) return rc;
      if (k == 1) w->halo_bytes = have;
    }
    bool fill = false;
    for (int k = 0; k < h.ncopies; ++k) fill = fill || h.source[k] == kSrcFill;
    if (fill) {
      rc = ensure(&w->d_const, &w->const_bytes, es);
      if (rc) return rc;
      const float f32 = (float)c.fill_value;  // pageable: staged before cudaMemcpyAsync returns
      XG_CUDA(cudaMemcpyAsync(w->d_const, es == 4 ? (const void*)&f32 : (const void*)&c.fill_value, es,
                              cudaMemcpyHostToDevice, w->s_h2d));
    }
  }
  XG_CUDA(cudaEventRecord(w->e_up[0], w->s_h2d));
  XG_CUDA(cudaStreamWaitEvent(w->s_k, w->e_up[0], 0));  // metrics + halo planes before any kernel

  int64_t slab_shape[XG_MAX_NDIM];
  for (int d = 0; d < ndim; ++d) slab_shape[d] = shape[d];

  int64_t prev_last_row = -1;          // global index of the last plane of the previous slab
  const char* prev_last_ptr = nullptr;  // ... and where it sits on the device
  for (int64_t s = 0; s < nslab; ++s) {
    const int slot = (int)(s % kSlots);
    const int64_t j0 = s * rows;                                  // first output row of the slab
    const int64_t j1 = (j0 + rows < n0_out) ? j0 + rows : n0_out;  // one past the last
    // input rows needed: non-operated dim 0 -> [j0, j1); operated -> P[j0 .. j1] i.e.
    // source rows [j0 - lo, j1 - lo] clipped to [0, n0)
    int64_t i0 = j0, i1 = j1;
    int slab_lo = lo, slab_hi = hi;
    if (ax0) {
      i0 = j0 - lo;
      i1 = j1 - lo + 1;
      slab_lo = 0;
      slab_hi = 0;
      if (i0 < 0) { i0 = 0; slab_lo = 1; }
      if (i1 > n0) { i1 = n0; slab_hi = 1; }
    }
    // slot reuse: the previous D2H out of this slot must have drained, and the kernel that read
    // the slot's input must have finished before we overwrite it
    if (s >= kSlots) {
      XG_CUDA(cudaStreamWaitEvent(w->s_h2d, w->e_done[slot], 0));
      XG_CUDA(cudaStreamWaitEvent(w->s_k, w->e_down[slot], 0));
    }
    if (ax0 && s > 0 && prev_last_row == i0 && i1 - i0 > 1) {
      // consecutive slabs of the operated axis overlap by exactly one plane: carry it over on the
      // device (same in-order stream as the uploads) instead of sending it over PCIe again
      XG_CUDA(cudaMemcpyAsync(w->d_in[slot], prev_last_ptr, (size_t)row_in * es,
                              cudaMemcpyDeviceToDevice, w->s_h2d));
      XG_CUDA(cudaMemcpyAsync((char*)w->d_in[slot] + (size_t)row_in * es,
                              hin + (size_t)(i0 + 1) * row_in * es,
                              (size_t)(i1 - i0 - 1) * row_in * es, cudaMemcpyHostToDevice, w->s_h2d));
    } else {
      XG_CUDA(cudaMemcpyAsync(w->d_in[slot], hin + (size_t)i0 * row_in * es,
                              (size_t)(i1 - i0) * row_in * es, cudaMemcpyHostToDevice, w->s_h2d));
    }
    if (partner)
      XG_CUDA(cudaMemcpyAsync(w->d_partner[slot], static_cast<const char*>(partner) + (size_t)(i0 * partner_row) * es,
                              (size_t)((i1 - i0) * partner_row) * es, cudaMemcpyHostToDevice, w->s_h2d));
    prev_last_row = i1 - 1;
    prev_last_ptr = (const char*)w->d_in[slot] + (size_t)(i1 - 1 - i0) * row_in * es;
    XG_CUDA(cudaEventRecord(w->e_up[slot], w->s_h2d));
    XG_CUDA(cudaStreamWaitEvent(w->s_k, w->e_up[slot], 0));

    slab_shape[0] = i1 - i0;
    const char* pm = (const char*)w->d_metric[0];
    const char* qm = (const char*)w->d_metric[1];
    if (c.pre) pm += (size_t)(i0 * c.pre_strides[0]) * es;
    if (c.post) qm += (size_t)(j0 * c.post_strides[0]) * es;
    const char* am = (const char*)w->d_metric[2];
    if (c.pair && c.pair->pre_a) am += (size_t)(i0 * c.pair->pre_a_strides[0]) * es;
    const void* hl = nullptr;
    const void* hh = nullptr;
    if (ax0 && wrap_planes) {
      if (slab_lo) hl = w->d_halo[0];
      if (slab_hi) hh = w->d_halo[1];
    }
    if (h.kind == kHaloFold) {
      rc = xg_fold_rows(c.dtype, c.pair ? w->d_partner[slot] : w->d_in[slot], w->d_halo[1], ndim, slab_shape, axis,
                        h.seam_axis, 1, 0, 1, h.skip, h.mirror, h.period, h.negate, c.pre ? pm : nullptr,
                        c.pre_strides, w->s_k);
      hh = w->d_halo[1];
      if (lo && bc == XG_BC_PERIODIC) hl = hh;  // a periodic south edge wraps the row above the top
    } else if (h.kind == kHaloCopies) {
      rc = halo_copies(h, c.dtype, es, w->d_halo, w->d_in[slot], w->d_partner[slot], w->d_const, i1 - i0,
                       dptr, sptr, shp, w->s_k);
      if (lo) hl = w->d_halo[0];
      if (hi) hh = w->d_halo[1];
    }
    if (rc == XG_OK && c.pair) {
      const PairTerm& t = *c.pair;
      rc = xg_stencil_pair_halo(c.dtype, w->d_in[slot], w->d_partner[slot], w->d_out[slot], ndim, slab_shape, t.op_a,
                                t.lo_a, t.hi_a, t.bc_a, t.fill_a, t.pre_a ? am : nullptr, t.pre_a_strides, axis, c.op,
                                lo, hi, bc, c.fill_value, c.pre ? pm : nullptr, c.pre_strides, t.subtract,
                                c.post ? qm : nullptr, c.post_strides, hl, hh, w->s_k);
    } else if (rc == XG_OK) {
      rc = xg_stencil2(c.op, c.dtype, w->d_in[slot], w->d_out[slot], ndim, slab_shape, axis, slab_lo, slab_hi,
                       (slab_lo || slab_hi) ? bc : XG_BC_NONE, c.fill_value, c.pre ? pm : nullptr,
                       c.pre_strides, c.post ? qm : nullptr, c.post_strides, hl, hh, w->s_k);
    }
    if (rc) {
      cudaDeviceSynchronize();
      return rc;
    }
    XG_CUDA(cudaEventRecord(w->e_done[slot], w->s_k));
    XG_CUDA(cudaStreamWaitEvent(w->s_d2h, w->e_done[slot], 0));
    XG_CUDA(cudaMemcpyAsync(hout + (size_t)j0 * row_out * es, w->d_out[slot],
                            (size_t)(j1 - j0) * row_out * es, cudaMemcpyDeviceToHost, w->s_d2h));
    XG_CUDA(cudaEventRecord(w->e_down[slot], w->s_d2h));
  }
  XG_CUDA(cudaStreamSynchronize(w->s_d2h));
  XG_CUDA(cudaStreamSynchronize(w->s_k));
  XG_CUDA(cudaStreamSynchronize(w->s_h2d));
  return XG_OK;
}

// lowest and highest element a strided copy of `shape` touches from `offset`
void copy_extent(int64_t offset, const int64_t* strides, const int64_t* shape, int ndim, int64_t* lo,
                 int64_t* hi) {
  *lo = *hi = offset;
  for (int d = 0; d < ndim; ++d) {
    const int64_t span = (shape[d] - 1) * strides[d];
    if (span < 0) *lo += span;
    else *hi += span;
  }
}

}  // namespace

extern "C" int xg_stencil2_host(int op, int dtype, const void* in, void* out, int ndim,
                                const int64_t* shape, int axis, int lo, int hi, int bc,
                                double fill_value, const void* pre_metric,
                                const int64_t* pre_strides, const void* post_metric,
                                const int64_t* post_strides, int device) {
  const Call c{op, dtype, in, out, ndim, shape, axis, lo, hi, bc, fill_value,
               pre_metric, pre_strides, post_metric, post_strides, device};
  int rc = validate_call("xg_stencil2_host", c);
  if (rc) return rc;
  return run_slabs(c, HaloStage{});
}

extern "C" int xg_stencil2_host_fold(int op, int dtype, const void* in, void* out, int ndim,
                                     const int64_t* shape, int axis, int lo, int hi, int bc,
                                     double fill_value, const void* pre_metric, const int64_t* pre_strides,
                                     const void* post_metric, const int64_t* post_strides, int seam_axis,
                                     int skip, int64_t mirror, int64_t period, int negate, int device) {
  const char* who = "xg_stencil2_host_fold";
  const Call c{op, dtype, in, out, ndim, shape, axis, lo, hi, bc, fill_value,
               pre_metric, pre_strides, post_metric, post_strides, device};
  int rc = validate_halo_call(who, c);
  if (rc == XG_OK) rc = validate_fold(who, c, seam_axis, skip, mirror, period);
  if (rc) return rc;
  HaloStage h;
  h.kind = kHaloFold;
  h.seam_axis = seam_axis;
  h.skip = skip;
  h.mirror = mirror;
  h.period = period;
  h.negate = negate ? 1 : 0;
  return run_slabs(c, h);
}

extern "C" int xg_stencil2_host_connected(int op, int dtype, const void* in, const void* partner,
                                          const int64_t* partner_shape, void* out, int ndim,
                                          const int64_t* shape, int axis, int lo, int hi, double fill_value,
                                          const void* post_metric, const int64_t* post_strides, int ncopies,
                                          int copy_ndim, const int* side, const int* source,
                                          const int64_t* dst_offset, const int64_t* src_offset,
                                          const int64_t* shapes, const int64_t* dst_strides,
                                          const int64_t* src_strides, const int* negate, int device) {
  const std::string who = "xg_stencil2_host_connected";
  const Call c{op, dtype, in, out, ndim, shape, axis, lo, hi, (lo || hi) ? XG_BC_FILL : XG_BC_NONE,
               fill_value, nullptr, nullptr, post_metric, post_strides, device};
  int rc = validate_halo_call(who.c_str(), c);
  if (rc) return rc;
  if (ncopies < 0) return xg_fail(XG_EINVAL, who + ": negative copy count");
  if (ncopies > 0 && (!side || !source || !dst_offset || !src_offset || !shapes || !dst_strides ||
                      !src_strides || !negate))
    return xg_fail(XG_EINVAL, who + ": null pointer in the copy list");
  if (ncopies > 0 && (copy_ndim < 1 || copy_ndim > XG_MAX_NDIM))
    return xg_fail(XG_EINVAL, who + ": bad copy rank");
  if (partner && !partner_shape) return xg_fail(XG_EINVAL, who + ": null partner shape");
  const int64_t n0 = shape[0];
  int64_t row_in = 1;
  for (int d = 1; d < ndim; ++d) row_in *= shape[d];
  const int64_t plane_row = shape[axis] ? row_in / shape[axis] : 0;
  int64_t partner_row = 0;
  if (partner) {
    if (partner_shape[0] != n0)
      return xg_fail(XG_EINVAL, who + ": the partner component's dim-0 extent differs from the field's");
    partner_row = 1;
    for (int d = 1; d < ndim; ++d) {
      if (partner_shape[d] < 0) return xg_fail(XG_EINVAL, who + ": negative partner extent");
      partner_row *= partner_shape[d];
    }
  }
  int64_t covered[2] = {0, 0};
  for (int k = 0; k < ncopies; ++k) {
    const int64_t* sh = shapes + (size_t)k * copy_ndim;
    const int64_t* ds = dst_strides + (size_t)k * copy_ndim;
    const int64_t* ss = src_strides + (size_t)k * copy_ndim;
    const std::string at = who + ": copy " + std::to_string(k) + ": ";
    if (side[k] != 0 && side[k] != 1) return xg_fail(XG_EINVAL, at + "side must be 0 (lo) or 1 (hi)");
    if (!(side[k] ? hi : lo)) return xg_fail(XG_EINVAL, at + "writes a halo plane the call does not pad");
    if (source[k] < kSrcField || source[k] > kSrcFill)
      return xg_fail(XG_EINVAL, at + "source must be 0 (field), 1 (partner) or 2 (fill constant)");
    if (source[k] == kSrcPartner && !partner) return xg_fail(XG_EINVAL, at + "reads a partner that was not given");
    int64_t cells = 1;
    for (int d = 0; d < copy_ndim; ++d) {
      if (sh[d] < 0) return xg_fail(XG_EINVAL, at + "negative extent");
      cells *= sh[d];
    }
    covered[side[k]] += cells;
    const int64_t src_row = source[k] == kSrcField ? row_in : source[k] == kSrcPartner ? partner_row : 0;
    if (sh[0] != n0 || ds[0] != plane_row || ss[0] != src_row)
      return xg_fail(XG_EINVAL, at + "must span dim 0 in full with the contiguous dim-0 strides");
    if (cells == 0) continue;
    int64_t a, b;
    copy_extent(dst_offset[k], ds, sh, copy_ndim, &a, &b);
    if (a < 0 || b >= n0 * plane_row) return xg_fail(XG_EINVAL, at + "leaves the halo plane");
    copy_extent(src_offset[k], ss, sh, copy_ndim, &a, &b);
    if (source[k] == kSrcFill) {
      if (a != 0 || b != 0) return xg_fail(XG_EINVAL, at + "the fill constant is read with offset 0, strides 0");
    } else if (a < 0 || b >= n0 * src_row) {
      return xg_fail(XG_EINVAL, at + "leaves its source array");
    }
  }
  // the copies write disjoint cells, so together they must cover each padded plane exactly once
  if ((lo && covered[0] != n0 * plane_row) || (hi && covered[1] != n0 * plane_row))
    return xg_fail(XG_EINVAL, who + ": the copies do not cover the halo planes");
  HaloStage h;
  h.kind = kHaloCopies;
  h.partner = partner;
  h.partner_row = partner_row;
  h.ncopies = ncopies;
  h.cndim = copy_ndim;
  h.side = side;
  h.source = source;
  h.negate_c = negate;
  h.dst_offset = dst_offset;
  h.src_offset = src_offset;
  h.shapes = shapes;
  h.dst_strides = dst_strides;
  h.src_strides = src_strides;
  return run_slabs(c, h);
}

extern "C" int xg_host_workspace_bytes(int device, int64_t* bytes) {
  if (!bytes) return xg_fail(XG_EINVAL, "xg_host_workspace_bytes: null pointer");
  *bytes = 0;
  Workspace* w = nullptr;
  {
    std::lock_guard<std::mutex> reg(g_ws_mutex);
    for (Workspace* x : g_ws)
      if (x->device == device) w = x;
  }
  if (!w) return XG_OK;
  std::lock_guard<std::mutex> lock(w->mu);
  *bytes = (int64_t)(kSlots * (w->slab_in_bytes + w->slab_out_bytes + w->partner_bytes) + w->metric_bytes[0] +
                     w->metric_bytes[1] + w->metric_bytes[2] + 2 * w->halo_bytes + w->const_bytes);
  return XG_OK;
}

extern "C" int xg_stencil_pair_host(int dtype, const void* a, const void* b, void* out, int ndim, const int64_t* shape,
                                    int op_a, int lo_a, int hi_a, int bc_a, double fill_a, const void* pre_a,
                                    const int64_t* pre_a_strides, int axis_b, int op_b, int lo_b, int hi_b, int bc_b,
                                    double fill_b, const void* pre_b, const int64_t* pre_b_strides, int subtract,
                                    const void* post, const int64_t* post_strides, int device) {
  const PairTerm t{b, op_a, lo_a, hi_a, bc_a, fill_a, pre_a, pre_a_strides, subtract};
  const Call c{op_b, dtype, a, out, ndim, shape, axis_b, lo_b, hi_b, bc_b, fill_b,
               pre_b, pre_b_strides, post, post_strides, device, &t};
  int rc = validate_pair_call("xg_stencil_pair_host", c);
  if (rc) return rc;
  return run_slabs(c, HaloStage{});
}

extern "C" int xg_stencil_pair_host_fold(int dtype, const void* a, const void* b, void* out, int ndim,
                                         const int64_t* shape, int op_a, int lo_a, int hi_a, int bc_a, double fill_a,
                                         const void* pre_a, const int64_t* pre_a_strides, int axis_b, int op_b,
                                         int lo_b, int hi_b, int bc_b, double fill_b, const void* pre_b,
                                         const int64_t* pre_b_strides, int subtract, const void* post,
                                         const int64_t* post_strides, int seam_axis, int skip, int64_t mirror,
                                         int64_t period, int negate, int device) {
  const char* who = "xg_stencil_pair_host_fold";
  const PairTerm t{b, op_a, lo_a, hi_a, bc_a, fill_a, pre_a, pre_a_strides, subtract};
  const Call c{op_b, dtype, a, out, ndim, shape, axis_b, lo_b, hi_b, bc_b, fill_b,
               pre_b, pre_b_strides, post, post_strides, device, &t};
  int rc = validate_pair_call(who, c);
  if (rc == XG_OK) rc = validate_fold(who, c, seam_axis, skip, mirror, period);
  if (rc) return rc;
  HaloStage h;
  h.kind = kHaloFold;
  h.seam_axis = seam_axis;
  h.skip = skip;
  h.mirror = mirror;
  h.period = period;
  h.negate = negate ? 1 : 0;
  return run_slabs(c, h);
}
