// The host-buffer entry points' slab engine, and the stencil / pair entry points on it.
//
// Numpy-backed fields are cut into slabs along one dimension and streamed through the GPU.  Three streams form a
// pipeline
//     H2D(slab s+1)  ||  kernel(s)(slab s)  ||  D2H(slab s-1)
// over three slots, so PCIe runs full duplex and the kernel time hides behind the copies.  Session::run is that
// pipeline for every host entry point (this file and xg_host_pipe.cu): it takes a [C][L][R] view of the input
// around the slab dim (strided 2-D copies when C > 1) and a launch callback that runs a slab's kernels.  A slab of
// result rows [j0, j1) reads input rows [j0 - lo_rows, j1 + hi_rows); rows the previous slab already holds are
// copied device-to-device, so each input row crosses PCIe once.
//
// One Workspace per device holds the streams, the events and three classes of buffers: per slot, what the copy
// streams touch (the input slab, a second streamed input, up to kMaxOut result slabs); once, what only the kernel
// stream touches (the per-slab halo planes, a scratch buffer); and the aux operands uploaded whole once per call.
// Its mutex makes calls on one device take turns (they would fight for PCIe anyway); calls on different devices
// run concurrently.  Streams and events live for the process; xg_host_workspace_release() frees the buffers.
// A host device group (xg_host_group) spreads one call over several devices: spread() gives each member a block of
// the result rows on its own thread, and each member streams its block through its own workspace.
//
// The stencil entry points here slab dim 0.  xg_stencil2_host: when dim 0 is the operated axis, consecutive slabs
// overlap by the one-cell halo and the exterior halo plane (periodic wrap) is uploaded once.
// xg_stencil2_host_fold / xg_stencil2_host_connected: dim 0 is a batch dim, and a per-slab halo stage on the kernel
// stream builds the slab's halo_lo / halo_hi planes from the slab buffers (one xg_fold_rows launch, or the
// face-connection copy list clipped to the slab and replayed with xg_strided_copy_batch) just before its
// xg_stencil2 launch.  xg_stencil_pair_host / xg_stencil_pair_host_fold: field a is the slab input, field b the
// second streamed input, and each slab is one xg_stencil_pair_halo launch (after the xg_fold_rows launch of b's
// folded row, for the fold).
#include <stdlib.h>

#include <thread>
#include <vector>

#include "xg_host.cuh"

namespace xg_host {

namespace {

constexpr int kSlots = 3;

#define XG_CUDA(call)                                                                   \
  do {                                                                                  \
    cudaError_t e_ = (call);                                                            \
    if (e_ != cudaSuccess)                                                              \
      return xg_fail(XG_ECUDA, std::string(#call) + ": " + cudaGetErrorString(e_));     \
  } while (0)

}  // namespace

struct Workspace {
  struct Buf {
    void* p = nullptr;
    size_t cap = 0;
  };
  int device = -1;
  std::mutex mu;  // held by the call streaming through the workspace, and by release
  cudaStream_t s_h2d = nullptr, s_k = nullptr, s_d2h = nullptr;
  cudaEvent_t e_up[kSlots], e_done[kSlots], e_down[kSlots], e_aux;
  bool ready = false;                                  // streams and events created
  Buf in[kSlots], in2[kSlots], out[kSlots][kMaxOut];  // per slot: touched by the copy streams
  Buf scratch, plane[2];                               // once: touched by the kernel stream alone
  Buf aux[kNumAux];                                    // uploaded whole, once per call

  template <class F>
  void each_buf(F f) {
    for (int i = 0; i < kSlots; ++i) {
      f(in[i]);
      f(in2[i]);
      for (Buf& b : out[i]) f(b);
    }
    f(scratch);
    f(plane[0]);
    f(plane[1]);
    for (Buf& b : aux) f(b);
  }
};

namespace {

std::mutex g_registry;          // guards g_ws
std::vector<Workspace*> g_ws;  // one per device, kept for the process

int ensure(Workspace::Buf& b, size_t want) {
  if (b.cap >= want && b.p) return XG_OK;
  if (b.p) XG_CUDA(cudaFree(b.p));
  b = Workspace::Buf();
  if (want == 0) return XG_OK;
  XG_CUDA(cudaMalloc(&b.p, want));
  b.cap = want;
  return XG_OK;
}

Workspace* find_workspace(int device) {  // caller holds g_registry
  for (Workspace* w : g_ws)
    if (w->device == device) return w;
  return nullptr;
}

// `height` rows of `width` bytes, one cudaMemcpyAsync when there is one row
int copy_rows(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, int64_t height,
              cudaMemcpyKind kind, cudaStream_t st) {
  if (width == 0 || height == 0) return XG_OK;
  if (height == 1) XG_CUDA(cudaMemcpyAsync(dst, src, width, kind, st));
  else XG_CUDA(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, (size_t)height, kind, st));
  return XG_OK;
}

// rows [r0, r1) of the slab dim of host array `host` (view v) <-> the device block at `dev`, whose C pieces hold
// `dev_rows` rows each
int copy_slab(void* dev, int64_t dev_rows, const void* host, const View3& v, int64_t r0, int64_t r1, size_t es,
              bool to_device, cudaStream_t st) {
  char* h = const_cast<char*>(static_cast<const char*>(host)) + (size_t)r0 * v.R * es;
  const size_t width = (size_t)(r1 - r0) * v.R * es, hpitch = (size_t)v.L * v.R * es;
  const size_t dpitch = (size_t)dev_rows * v.R * es;
  if (to_device) return copy_rows(dev, dpitch, h, hpitch, width, v.C, cudaMemcpyHostToDevice, st);
  return copy_rows(h, hpitch, dev, dpitch, width, v.C, cudaMemcpyDeviceToHost, st);
}

// rows per slab of a slab dim of extent L whose one row moves `row_bytes`
int64_t slab_rows(int64_t L, int64_t row_bytes, bool edge_pairs) {
  int64_t rows = row_bytes > 0 ? slab_budget_bytes() / row_bytes : L;
  if (rows < 1) rows = 1;
  if (rows > (L + 3) / 4) rows = (L + 3) / 4;  // at least 4 slabs when the dim allows: overlap
  if (rows < 1) rows = 1;
  if (edge_pairs) {
    // e.g. an extrapolated halo is 2 A[edge] - A[next]: the slab that touches an edge must hold two input rows,
    // i.e. no one-row slab at either end (a one-row tail is merged by growing the slab height)
    if (rows < 2) rows = 2;
    while (rows < L && L % rows == 1) ++rows;
    if (rows > L) rows = L;
  }
  return rows;
}

}  // namespace

View3 view3(int ndim, const int64_t* shape, int sd) {
  View3 v{1, ndim ? shape[sd] : 1, 1};
  for (int d = 0; d < sd; ++d) v.C *= shape[d];
  for (int d = sd + 1; d < ndim; ++d) v.R *= shape[d];
  return v;
}

size_t operand_span(const int64_t* strides, const int64_t* shape, int ndim, size_t es) {
  int64_t last = 0;
  for (int d = 0; d < ndim; ++d)
    if (shape[d] > 1) last += (shape[d] - 1) * strides[d];
  return (size_t)(last + 1) * es;
}

int64_t slab_budget_bytes() {
  int64_t target_bytes = 128ll << 20;
  if (const char* env = getenv("XG_HOST_SLAB_MB")) {  // tuning knob (benchmarks only)
    const long mb = atol(env);
    if (mb >= 1 && mb <= 4096) target_bytes = (int64_t)mb << 20;
  }
  return target_bytes;
}

namespace {

std::mutex g_group_mu;                  // guards g_groups
std::vector<std::vector<int>> g_groups;  // member lists of the handles XG_HOST_GROUP_BASE + k; append-only

// the member list of group handle `handle`; XG_EINVAL for an unknown handle (no CUDA call)
int group_members(const char* who, int handle, std::vector<int>* members) {
  std::lock_guard<std::mutex> lock(g_group_mu);
  const int64_t k = (int64_t)handle - XG_HOST_GROUP_BASE;
  if (k < 0 || k >= (int64_t)g_groups.size())
    return xg_fail(XG_EINVAL, std::string(who) + ": unknown host device group " + std::to_string(handle));
  *members = g_groups[(size_t)k];
  return XG_OK;
}

}  // namespace

int spread(const char* who, int device, int64_t L, bool edge_pairs, const BlockFn& body, bool split) {
  if (device < XG_HOST_GROUP_BASE) return body(device, 0, L);
  std::vector<int> members;
  int rc = group_members(who, device, &members);
  if (rc) return rc;
  int64_t nb = split ? (int64_t)members.size() : 1;
  if (nb > L) nb = L;
  if (edge_pairs)  // the last block, the smallest, holds L / nb rows
    while (nb > 1 && L / nb < 2) --nb;
  if (nb < 1) nb = 1;
  struct Outcome {
    int rc = XG_OK;
    std::string error;
    const char* label = "";
  };
  std::vector<Outcome> res((size_t)nb);
  std::vector<std::thread> threads;
  threads.reserve((size_t)nb);
  for (int64_t k = 0; k < nb; ++k) {
    // the first L % nb blocks hold one row more
    const int64_t r0 = k * (L / nb) + (k < L % nb ? k : L % nb), r1 = r0 + L / nb + (k < L % nb ? 1 : 0);
    Outcome& o = res[(size_t)k];
    const int member = members[(size_t)k];
    try {
      threads.emplace_back([&body, &o, member, r0, r1] {
        try {
          o.rc = body(member, r0, r1);
        } catch (const std::exception& e) {
          o.rc = xg_fail(XG_ECUDA, std::string("host device group member: ") + e.what());
        }
        if (o.rc) o.error = xg_last_error();
        o.label = xg_last_launch();
      });
    } catch (const std::exception& e) {  // blocks k.. do not run
      o.rc = XG_ECUDA;
      o.error = std::string(who) + ": cannot start a thread for a host device group member: " + e.what();
      break;
    }
  }
  for (std::thread& t : threads) t.join();
  xg_set_last_launch(res[0].label);
  for (const Outcome& o : res)
    if (o.rc) return xg_fail(o.rc, o.error);
  return XG_OK;
}

Session::~Session() {
  if (w_ && w_->ready)
    for (cudaStream_t st : {w_->s_h2d, w_->s_k, w_->s_d2h}) cudaStreamSynchronize(st);
}

int Session::open(int device) {
  XG_CUDA(cudaSetDevice(device));
  {
    std::lock_guard<std::mutex> reg(g_registry);
    w_ = find_workspace(device);
    if (!w_) {
      w_ = new Workspace();
      w_->device = device;
      g_ws.push_back(w_);
    }
  }
  lock_ = std::unique_lock<std::mutex>(w_->mu);
  if (w_->ready) return XG_OK;
  for (cudaStream_t* st : {&w_->s_h2d, &w_->s_k, &w_->s_d2h})
    XG_CUDA(cudaStreamCreateWithFlags(st, cudaStreamNonBlocking));
  for (int i = 0; i < kSlots; ++i)
    for (cudaEvent_t* e : {&w_->e_up[i], &w_->e_done[i], &w_->e_down[i]})
      XG_CUDA(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
  XG_CUDA(cudaEventCreateWithFlags(&w_->e_aux, cudaEventDisableTiming));
  w_->ready = true;
  return XG_OK;
}

int Session::aux(Aux a, size_t bytes, void** dev) {
  int rc = ensure(w_->aux[a], bytes);
  if (rc) return rc;
  *dev = w_->aux[a].p;
  return XG_OK;
}

int Session::upload(Aux a, const void* host, size_t bytes, const void** dev) {
  *dev = nullptr;
  if (!host) return XG_OK;
  void* d = nullptr;
  int rc = aux(a, bytes, &d);
  if (rc) return rc;
  XG_CUDA(cudaMemcpyAsync(d, host, bytes, cudaMemcpyHostToDevice, w_->s_h2d));
  *dev = d;
  return XG_OK;
}

int Session::fence() {
  XG_CUDA(cudaEventRecord(w_->e_aux, w_->s_h2d));
  XG_CUDA(cudaStreamWaitEvent(w_->s_k, w_->e_aux, 0));
  return XG_OK;
}

cudaStream_t Session::kernel_stream() const { return w_->s_k; }

int Session::download(void* host, const void* dev, size_t bytes) {
  XG_CUDA(cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, w_->s_k));
  XG_CUDA(cudaStreamSynchronize(w_->s_k));
  return XG_OK;
}

int Session::run(size_t es, const void* hin, const View3& in, int nout, void* const* hout, const View3* out,
                 const LaunchFn& launch, const PipeExtra& ex) {
  Workspace* w = w_;
  const int64_t r0 = ex.r0, r1 = ex.r1 < 0 ? out[0].L : ex.r1;
  if (in.L == 0 || in.C == 0 || in.R == 0 || r1 <= r0) return XG_OK;
  const int64_t rows =
      slab_rows(r1 - r0, ex.row_bytes > 0 ? ex.row_bytes : in.C * in.R * (int64_t)es, ex.edge_pairs);
  const int64_t nslab = xg_ceil_div(r1 - r0, rows);
  int rc = XG_OK;
  for (int i = 0; rc == XG_OK && i < kSlots; ++i) {
    rc = ensure(w->in[i], (size_t)(in.C * (rows + ex.lo_rows + ex.hi_rows) * in.R) * es);
    if (rc == XG_OK && ex.hin2) rc = ensure(w->in2[i], (size_t)(ex.in2.C * rows * ex.in2.R) * es);
    for (int k = 0; rc == XG_OK && k < nout; ++k)
      rc = ensure(w->out[i][k], (size_t)(out[k].C * rows * out[k].R) * es);
  }
  if (rc == XG_OK) rc = ensure(w->scratch, ex.scratch_row_bytes * (size_t)rows);
  for (int k = 0; rc == XG_OK && k < 2; ++k) rc = ensure(w->plane[k], ex.plane_row_bytes * (size_t)rows);
  if (rc) return rc;

  const size_t row = (size_t)in.R * es;  // bytes of one input row in each of the C pieces
  int64_t p0 = 0, p1 = 0;                 // input rows the previous slab's buffer holds
  for (int64_t s = 0; s < nslab; ++s) {
    const int slot = (int)(s % kSlots);
    const int64_t j0 = r0 + s * rows, j1 = (j0 + rows < r1) ? j0 + rows : r1;
    const int64_t i0 = (j0 - ex.lo_rows < 0) ? 0 : j0 - ex.lo_rows;
    const int64_t i1 = (j1 + ex.hi_rows > in.L) ? in.L : j1 + ex.hi_rows;
    if (s >= kSlots) {
      XG_CUDA(cudaStreamWaitEvent(w->s_h2d, w->e_done[slot], 0));  // kernels that read this slot's input
      XG_CUDA(cudaStreamWaitEvent(w->s_k, w->e_down[slot], 0));    // downloads out of this slot's results
    }
    char* d_in = static_cast<char*>(w->in[slot].p);
    // rows [i0, i0 + keep) are on the device already (never in a block's first slab: its halo rows come up too)
    const int64_t keep = (s > 0 && p1 > i0) ? p1 - i0 : 0;
    if (keep)  // same in-order stream as the uploads
      rc = copy_rows(d_in, (size_t)(i1 - i0) * row,
                     static_cast<const char*>(w->in[(s - 1) % kSlots].p) + (size_t)(i0 - p0) * row,
                     (size_t)(p1 - p0) * row, (size_t)keep * row, in.C, cudaMemcpyDeviceToDevice, w->s_h2d);
    if (rc == XG_OK) rc = copy_slab(d_in + keep * row, i1 - i0, hin, in, i0 + keep, i1, es, true, w->s_h2d);
    if (rc == XG_OK && ex.hin2) rc = copy_slab(w->in2[slot].p, j1 - j0, ex.hin2, ex.in2, j0, j1, es, true, w->s_h2d);
    if (rc) return rc;
    p0 = i0;
    p1 = i1;
    XG_CUDA(cudaEventRecord(w->e_up[slot], w->s_h2d));
    XG_CUDA(cudaStreamWaitEvent(w->s_k, w->e_up[slot], 0));
    void* d_out[kMaxOut];
    for (int k = 0; k < nout; ++k) d_out[k] = w->out[slot][k].p;
    const SlabBufs bufs{d_in,
                        ex.hin2 ? w->in2[slot].p : nullptr,
                        ex.scratch_row_bytes ? w->scratch.p : nullptr,
                        {ex.plane_row_bytes ? w->plane[0].p : nullptr, ex.plane_row_bytes ? w->plane[1].p : nullptr},
                        d_out};
    rc = launch(j0, j1, i0, i1, bufs, w->s_k);
    if (rc) return rc;
    XG_CUDA(cudaEventRecord(w->e_done[slot], w->s_k));
    XG_CUDA(cudaStreamWaitEvent(w->s_d2h, w->e_done[slot], 0));
    for (int k = 0; rc == XG_OK && k < nout; ++k)
      rc = copy_slab(d_out[k], j1 - j0, hout[k], out[k], j0, j1, es, false, w->s_d2h);
    if (rc) return rc;
    XG_CUDA(cudaEventRecord(w->e_down[slot], w->s_d2h));
  }
  for (cudaStream_t st : {w->s_d2h, w->s_k, w->s_h2d}) XG_CUDA(cudaStreamSynchronize(st));
  return XG_OK;
}

namespace {

int workspace_bytes(const char* who, int device, int64_t* bytes) {
  if (!bytes) return xg_fail(XG_EINVAL, std::string(who) + ": null pointer");
  *bytes = 0;
  if (device >= XG_HOST_GROUP_BASE)
    return xg_fail(XG_EINVAL, std::string(who) + ": takes a device index, not a host device group");
  Workspace* w = nullptr;
  {
    std::lock_guard<std::mutex> reg(g_registry);
    w = find_workspace(device);
  }
  if (!w) return XG_OK;
  std::lock_guard<std::mutex> lock(w->mu);
  w->each_buf([&](Workspace::Buf& b) { *bytes += (int64_t)b.cap; });
  return XG_OK;
}

// ------------------------------------------------------------------------------ the stencil and pair entry points
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

// The stencil arguments of a host stencil entry point.
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
};

enum { kSrcField = 0, kSrcPartner = 1, kSrcFill = 2 };

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
int validate_pair_call(const char* who, const Call& c, const PairTerm& t) {
  const std::string w(who);
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

// A slab's halo stage, on the kernel stream before its stencil launch: builds the slab's halo planes into b.plane
// and points *hl / *hh at them.  `slab_shape` is the slab's shape, `pre` its rows of the pre-metric, `fill` the
// device copy of the fill constant (nullptr unless the entry point uploads one).  Called from every thread of a
// host device group at once: it keeps no state across calls.
typedef std::function<int(const SlabBufs& b, const int64_t* slab_shape, const void* pre, const void* fill,
                          cudaStream_t st, const void** hl, const void** hh)>
    HaloFn;

// The fold's halo stage: the folded north row of the slab (of the field across the fold: the input, or the second
// input of a pair) is halo_hi, and halo_lo too when the south edge is periodic (it wraps the row above the top).
HaloFn fold_stage(const Call& c, bool of_in2, int seam_axis, int skip, int64_t mirror, int64_t period, int negate) {
  return [=](const SlabBufs& b, const int64_t* slab_shape, const void* pre, const void*, cudaStream_t st,
             const void** hl, const void** hh) {
    *hh = b.plane[1];
    if (c.lo && c.bc == XG_BC_PERIODIC) *hl = *hh;
    return xg_fold_rows(c.dtype, of_in2 ? b.in2 : b.in, b.plane[1], c.ndim, slab_shape, c.axis, seam_axis, 1, 0, 1,
                        skip, mirror, period, negate ? 1 : 0, pre, c.pre_strides, st);
  };
}

// A stencil entry point (arguments checked) on c.device: field c.in in slabs along dim 0, `partner` (field b of pair
// `t`, or the partner vector component, `partner_row` elements per dim-0 index) beside it, the metrics (and the
// `fill_host` constant, es bytes, when given) uploaded whole.  Per slab `halo` (when dim 0 is a batch dim) builds
// the halo planes, then one xg_stencil2 or xg_stencil_pair_halo launch.
int stencil_host(const char* who, const Call& c, const PairTerm* t, const void* partner, int64_t partner_row,
                 const HaloFn& halo, const void* fill_host = nullptr) {
  const size_t es = c.dtype == XG_F32 ? 4 : 8;
  const int ndim = c.ndim, lo = c.lo;
  const bool ax0 = c.axis == 0;
  const int64_t n0 = c.shape[0];
  int64_t out_shape[XG_MAX_NDIM];
  for (int d = 0; d < ndim; ++d) out_shape[d] = c.shape[d];
  out_shape[c.axis] = c.shape[c.axis] + c.lo + c.hi - 1;
  const View3 vin = view3(ndim, c.shape, 0), vout = view3(ndim, out_shape, 0);
  const bool edge_pairs = ax0 && c.bc == XG_BC_EXTRAPOLATE && (lo || c.hi);
  return spread(who, c.device, vout.L, edge_pairs, [&](int device, int64_t r0, int64_t r1) -> int {
    Session ss;
    int rc = ss.open(device);
    if (rc) return rc;
    if (vout.L <= 0 || vout.R == 0 || vin.R == 0) return XG_OK;

    const void *d_pre, *d_post, *d_pre_a = nullptr, *d_fill = nullptr;
    const void* wrap[2] = {nullptr, nullptr};  // periodic halo planes along dim 0: plane n0 - 1 below, plane 0 above
    const size_t plane = (size_t)vin.R * es;
    rc = ss.upload(kAuxPre, c.pre, c.pre ? operand_span(c.pre_strides, c.shape, ndim, es) : 0, &d_pre);
    if (rc == XG_OK)
      rc = ss.upload(kAuxPost, c.post, c.post ? operand_span(c.post_strides, out_shape, ndim, es) : 0, &d_post);
    if (rc == XG_OK && t && t->pre_a)
      rc = ss.upload(kAuxPreA, t->pre_a, operand_span(t->pre_a_strides, c.shape, ndim, es), &d_pre_a);
    if (rc == XG_OK && ax0 && c.bc == XG_BC_PERIODIC && lo)
      rc = ss.upload(kAuxWrapLo, static_cast<const char*>(c.in) + (size_t)(n0 - 1) * plane, plane, &wrap[0]);
    if (rc == XG_OK && ax0 && c.bc == XG_BC_PERIODIC && c.hi) rc = ss.upload(kAuxWrapHi, c.in, plane, &wrap[1]);
    if (rc == XG_OK) rc = ss.upload(kAuxFill, fill_host, es, &d_fill);
    if (rc == XG_OK) rc = ss.fence();
    if (rc) return rc;

    PipeExtra ex;
    if (ax0) {  // result rows [j0, j1) read planes [j0 - lo, j1 - lo] of the padded field
      ex.lo_rows = lo;
      ex.hi_rows = 1 - lo;
      ex.edge_pairs = edge_pairs;
    }
    if (partner) {
      ex.hin2 = partner;
      ex.in2 = View3{1, n0, partner_row};
    }
    if (halo) ex.plane_row_bytes = (size_t)(vin.R / c.shape[c.axis]) * es;
    int64_t sshape[XG_MAX_NDIM];
    for (int d = 0; d < ndim; ++d) sshape[d] = c.shape[d];
    auto launch = [&](int64_t j0, int64_t j1, int64_t i0, int64_t i1, const SlabBufs& b, cudaStream_t st) -> int {
      sshape[0] = i1 - i0;
      const char* pm = d_pre ? static_cast<const char*>(d_pre) + (size_t)(i0 * c.pre_strides[0]) * es : nullptr;
      const char* qm = d_post ? static_cast<const char*>(d_post) + (size_t)(j0 * c.post_strides[0]) * es : nullptr;
      // along dim 0 a slab pads only the edges of the field its planes reach
      const int slo = ax0 ? j0 - lo < 0 : lo, shi = ax0 ? j1 - lo + 1 > n0 : c.hi;
      const void* hl = slo ? wrap[0] : nullptr;
      const void* hh = shi ? wrap[1] : nullptr;
      if (halo) {
        const int rc2 = halo(b, sshape, pm, d_fill, st, &hl, &hh);
        if (rc2) return rc2;
      }
      if (t) {
        const char* am =
            d_pre_a ? static_cast<const char*>(d_pre_a) + (size_t)(i0 * t->pre_a_strides[0]) * es : nullptr;
        return xg_stencil_pair_halo(c.dtype, b.in, b.in2, b.out[0], ndim, sshape, t->op_a, t->lo_a, t->hi_a, t->bc_a,
                                    t->fill_a, am, t->pre_a_strides, c.axis, c.op, lo, c.hi, c.bc, c.fill_value, pm,
                                    c.pre_strides, t->subtract, qm, c.post_strides, hl, hh, st);
      }
      return xg_stencil2(c.op, c.dtype, b.in, b.out[0], ndim, sshape, c.axis, slo, shi,
                         (slo || shi) ? c.bc : XG_BC_NONE, c.fill_value, pm, c.pre_strides, qm, c.post_strides, hl, hh,
                         st);
    };
    void* outs[1] = {c.out};
    return ss.run(es, c.in, vin, 1, outs, &vout, launch, ex.rows(r0, r1));
  });
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
}  // namespace xg_host

using namespace xg_host;

extern "C" int xg_host_workspace_release(void) {
  std::lock_guard<std::mutex> reg(g_registry);
  for (Workspace* w : g_ws) {
    std::lock_guard<std::mutex> lock(w->mu);  // not while a call streams through it
    cudaSetDevice(w->device);
    w->each_buf([](Workspace::Buf& b) {
      if (b.p) cudaFree(b.p);
      b = Workspace::Buf();
    });
  }
  return XG_OK;
}

extern "C" int xg_host_group(int n, const int* devices, int* group) {
  const std::string who = "xg_host_group";
  if (!devices || !group) return xg_fail(XG_EINVAL, who + ": null pointer");
  if (n < 1 || n > XG_HOST_GROUP_MAX_MEMBERS)
    return xg_fail(XG_EINVAL, who + ": between 1 and " + std::to_string(XG_HOST_GROUP_MAX_MEMBERS) + " members");
  for (int k = 0; k < n; ++k)
    if (devices[k] < 0) return xg_fail(XG_EINVAL, who + ": negative device index");
  int count = 0;
  XG_CUDA(cudaGetDeviceCount(&count));
  for (int k = 0; k < n; ++k)
    if (devices[k] >= count)
      return xg_fail(XG_EINVAL, who + ": device " + std::to_string(devices[k]) + " does not exist (" +
                                    std::to_string(count) + " visible)");
  const std::vector<int> members(devices, devices + n);
  std::lock_guard<std::mutex> lock(g_group_mu);
  for (size_t k = 0; k < g_groups.size(); ++k)
    if (g_groups[k] == members) {
      *group = XG_HOST_GROUP_BASE + (int)k;
      return XG_OK;
    }
  if (g_groups.size() >= XG_HOST_GROUP_MAX)
    return xg_fail(XG_EINVAL, who + ": " + std::to_string(XG_HOST_GROUP_MAX) + " groups are registered already");
  g_groups.push_back(members);
  *group = XG_HOST_GROUP_BASE + (int)(g_groups.size() - 1);
  return XG_OK;
}

extern "C" int xg_host_workspace_bytes(int device, int64_t* bytes) {
  return workspace_bytes("xg_host_workspace_bytes", device, bytes);
}

extern "C" int xg_host_pipe_workspace_bytes(int device, int64_t* bytes) {
  return workspace_bytes("xg_host_pipe_workspace_bytes", device, bytes);
}

extern "C" int xg_stencil2_host(int op, int dtype, const void* in, void* out, int ndim,
                                const int64_t* shape, int axis, int lo, int hi, int bc,
                                double fill_value, const void* pre_metric,
                                const int64_t* pre_strides, const void* post_metric,
                                const int64_t* post_strides, int device) {
  const Call c{op, dtype, in, out, ndim, shape, axis, lo, hi, bc, fill_value,
               pre_metric, pre_strides, post_metric, post_strides, device};
  int rc = validate_call("xg_stencil2_host", c);
  return rc ? rc : stencil_host("xg_stencil2_host", c, nullptr, nullptr, 0, nullptr);
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
  return rc ? rc
            : stencil_host(who, c, nullptr, nullptr, 0, fold_stage(c, false, seam_axis, skip, mirror, period, negate));
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
  bool fill = false;
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
    fill = fill || source[k] == kSrcFill;
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

  const size_t es = dtype == XG_F32 ? 4 : 8;
  const float f32 = (float)fill_value;  // pageable: staged before cudaMemcpyAsync returns
  const void* fill_host = fill ? (es == 4 ? (const void*)&f32 : (const void*)&fill_value) : nullptr;
  // the whole-field copy list rebased onto each slab's buffers, `rows` high.  The rebased pointers and shapes are
  // built per slab, on every path (three vectors of ncopies entries, small beside a slab's copies): the stage then
  // keeps no state between slabs, so the members of a host device group can run it at once.
  auto copies = [&](const SlabBufs& b, const int64_t* slab_shape, const void*, const void* d_fill, cudaStream_t st,
                    const void** hl, const void** hh) -> int {
    std::vector<void*> dptr(ncopies);
    std::vector<const void*> sptr(ncopies);
    std::vector<int64_t> shp(shapes ? shapes : (const int64_t*)nullptr,
                             shapes ? shapes + (size_t)ncopies * copy_ndim : (const int64_t*)nullptr);
    for (int k = 0; k < ncopies; ++k) {
      dptr[k] = static_cast<char*>(b.plane[side[k]]) + (size_t)dst_offset[k] * es;
      const void* base = source[k] == kSrcField ? b.in : source[k] == kSrcPartner ? b.in2 : d_fill;
      sptr[k] = static_cast<const char*>(base) + (size_t)src_offset[k] * es;
      shp[(size_t)k * copy_ndim] = slab_shape[0];
    }
    if (lo) *hl = b.plane[0];
    if (hi) *hh = b.plane[1];
    int rc2 = xg_strided_copy_batch(dtype, ncopies, dptr.data(), sptr.data(), copy_ndim, shp.data(), dst_strides,
                                    src_strides, negate, st);
    if (rc2 != XG_ENOTIMPL) return rc2;
    for (int k = 0; k < ncopies; ++k) {  // some copy does not collapse to 5 dims: one launch per copy
      rc2 = xg_strided_copy(dtype, dptr[k], dst_strides + (size_t)k * copy_ndim, sptr[k],
                            src_strides + (size_t)k * copy_ndim, copy_ndim, shp.data() + (size_t)k * copy_ndim,
                            negate[k], st);
      if (rc2) return rc2;
    }
    return XG_OK;
  };
  return stencil_host(who.c_str(), c, nullptr, partner, partner_row, copies, fill_host);
}

extern "C" int xg_stencil_pair_host(int dtype, const void* a, const void* b, void* out, int ndim, const int64_t* shape,
                                    int op_a, int lo_a, int hi_a, int bc_a, double fill_a, const void* pre_a,
                                    const int64_t* pre_a_strides, int axis_b, int op_b, int lo_b, int hi_b, int bc_b,
                                    double fill_b, const void* pre_b, const int64_t* pre_b_strides, int subtract,
                                    const void* post, const int64_t* post_strides, int device) {
  const PairTerm t{b, op_a, lo_a, hi_a, bc_a, fill_a, pre_a, pre_a_strides, subtract};
  const Call c{op_b, dtype, a, out, ndim, shape, axis_b, lo_b, hi_b, bc_b, fill_b,
               pre_b, pre_b_strides, post, post_strides, device};
  int rc = validate_pair_call("xg_stencil_pair_host", c, t);
  return rc ? rc : stencil_host("xg_stencil_pair_host", c, &t, b, view3(ndim, shape, 0).R, nullptr);
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
               pre_b, pre_b_strides, post, post_strides, device};
  int rc = validate_pair_call(who, c, t);
  if (rc == XG_OK) rc = validate_fold(who, c, seam_axis, skip, mirror, period);
  return rc ? rc
            : stencil_host(who, c, &t, b, view3(ndim, shape, 0).R,
                           fold_stage(c, true, seam_axis, skip, mirror, period, negate));
}
