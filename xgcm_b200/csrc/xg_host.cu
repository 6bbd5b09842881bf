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
// xg_stencil2_host_multi: the same with up to kMaxOut results of one uploaded slab, so a `Grid.diff` + `Grid.interp`
// sweep over X, Y, Z moves the field over PCIe once, not six times; its results along dim 0 keep that extent.
// xg_stencil2_host_fold / xg_stencil2_host_connected: dim 0 is a batch dim, and a per-slab halo stage on the kernel
// stream builds the slab's halo_lo / halo_hi planes from the slab buffers (one xg_fold_rows launch, or the
// face-connection copy list clipped to the slab and replayed with xg_strided_copy_batch) just before its
// xg_stencil2 launch; xg_stencil2_host_connected_weighted replays the copy list over the pre-metric too and multiplies
// the planes by those weights (xg_binary), the halo of x * pre.  xg_stencil_pair_host / xg_stencil_pair_host_fold: field a is the slab input, field b the
// second streamed input, and each slab is one xg_stencil_pair_halo launch (after the xg_fold_rows launch of b's
// folded row, for the fold).  xg_cumscan_host_fold / xg_cumscan_host_connected run the same halo stages on each
// slab's scanned rows (xg_cumscan into the scratch buffer), then place the scanned slab and its halo planes into the
// padded result slab and divide by the post-metric.  xg_stencil_chain_host_fold / _connected run a multi-axis
// diff / interp / min / max as the device route does, one axis after another: per slab, each stage builds its halo
// planes from its own input (the slab input, or the previous stage's result in the scratch buffer) and runs one
// xg_stencil2 launch into the next intermediate or the result slab.
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

int read_window(const char* who, int64_t j0, int64_t j1, int lo, int64_t n, int64_t i0, int64_t i1, Window* w) {
  *w = Window{j0 - lo, j1 - lo + 1, 0, 0};
  if (w->s0 < 0) {
    w->s0 = 0;
    w->slo = 1;
  }
  if (w->s1 > n) {
    w->s1 = n;
    w->shi = 1;
  }
  if (w->s0 < i0 || w->s1 > i1) return xg_fail(XG_EINVAL, std::string(who) + ": internal slab window error");
  return XG_OK;
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

// A stencil entry point (arguments checked) on cs[0].device: field cs[0].in in slabs along dim 0, into the `nout`
// results cs[k].out (1 .. kMaxOut), which share in, dtype, ndim, shape and device.  With one result only: `partner`
// (field b of pair `t`, or the partner vector component, `partner_row` elements per dim-0 index) beside the field,
// the metrics (and the `fill_host` constant, es bytes, when given) uploaded whole, and per slab `halo` (when dim 0 is
// a batch dim) building the halo planes.  Per slab, one xg_stencil2 or xg_stencil_pair_halo launch per result.
// `fill_host` holds `nfill` constants; `scratch_row_bytes` sizes the scratch buffer per slab row (halo stages only).
int stencil_host(const char* who, int nout, const Call* cs, const PairTerm* t, const void* partner,
                 int64_t partner_row, const HaloFn& halo, const void* fill_host = nullptr, int nfill = 1,
                 size_t scratch_row_bytes = 0) {
  const Call& c0 = cs[0];
  const size_t es = c0.dtype == XG_F32 ? 4 : 8;
  const int ndim = c0.ndim;
  const int64_t n0 = c0.shape[0];
  const View3 vin = view3(ndim, c0.shape, 0);
  int64_t out_shape[kMaxOut][XG_MAX_NDIM];
  View3 vout[kMaxOut];
  bool empty = vin.R == 0, wrap_lo = false, wrap_hi = false;
  PipeExtra ex;
  for (int k = 0; k < nout; ++k) {
    const Call& c = cs[k];
    for (int d = 0; d < ndim; ++d) out_shape[k][d] = c.shape[d];
    out_shape[k][c.axis] = c.shape[c.axis] + c.lo + c.hi - 1;
    vout[k] = view3(ndim, out_shape[k], 0);
    empty = empty || vout[k].L <= 0 || vout[k].R == 0;
    if (c.axis != 0) continue;
    // a slab reads the input rows read_window gives its results along dim 0
    if (c.lo > ex.lo_rows) ex.lo_rows = c.lo;
    if (1 - c.lo > ex.hi_rows) ex.hi_rows = 1 - c.lo;
    ex.edge_pairs = ex.edge_pairs || (c.bc == XG_BC_EXTRAPOLATE && (c.lo || c.hi));
    wrap_lo = wrap_lo || (c.bc == XG_BC_PERIODIC && c.lo);
    wrap_hi = wrap_hi || (c.bc == XG_BC_PERIODIC && c.hi);
  }
  if (partner) {
    ex.hin2 = partner;
    ex.in2 = View3{1, n0, partner_row};
  }
  if (halo) {
    ex.plane_row_bytes = (size_t)(vin.R / c0.shape[c0.axis]) * es;
    ex.scratch_row_bytes = scratch_row_bytes;
  }
  return spread(who, c0.device, vout[0].L, ex.edge_pairs, [&](int device, int64_t r0, int64_t r1) -> int {
    Session ss;
    int rc = ss.open(device);
    if (rc) return rc;
    if (empty) return XG_OK;

    const void *d_pre, *d_post, *d_pre_a = nullptr, *d_fill = nullptr;
    const void* wrap[2] = {nullptr, nullptr};  // periodic halo planes along dim 0: plane n0 - 1 below, plane 0 above
    const size_t plane = (size_t)vin.R * es;
    rc = ss.upload(kAuxPre, c0.pre, c0.pre ? operand_span(c0.pre_strides, c0.shape, ndim, es) : 0, &d_pre);
    if (rc == XG_OK)
      rc = ss.upload(kAuxPost, c0.post, c0.post ? operand_span(c0.post_strides, out_shape[0], ndim, es) : 0, &d_post);
    if (rc == XG_OK && t && t->pre_a)
      rc = ss.upload(kAuxPreA, t->pre_a, operand_span(t->pre_a_strides, c0.shape, ndim, es), &d_pre_a);
    if (rc == XG_OK && wrap_lo)
      rc = ss.upload(kAuxWrapLo, static_cast<const char*>(c0.in) + (size_t)(n0 - 1) * plane, plane, &wrap[0]);
    if (rc == XG_OK && wrap_hi) rc = ss.upload(kAuxWrapHi, c0.in, plane, &wrap[1]);
    if (rc == XG_OK) rc = ss.upload(kAuxFill, fill_host, (size_t)nfill * es, &d_fill);
    if (rc == XG_OK) rc = ss.fence();
    if (rc) return rc;

    auto launch = [&](int64_t j0, int64_t j1, int64_t i0, int64_t i1, const SlabBufs& b, cudaStream_t st) -> int {
      for (int k = 0; k < nout; ++k) {
        const Call& c = cs[k];
        // the result's input rows [s0, s1); along dim 0 a slab pads only the edges of the field its rows reach
        Window w{j0, j1, c.lo, c.hi};
        if (c.axis == 0) {
          const int rc2 = read_window(who, j0, j1, c.lo, n0, i0, i1, &w);
          if (rc2) return rc2;
        }
        int64_t sshape[XG_MAX_NDIM];
        for (int d = 0; d < ndim; ++d) sshape[d] = c.shape[d];
        sshape[0] = w.s1 - w.s0;
        const char* src = static_cast<const char*>(b.in) + (size_t)(w.s0 - i0) * plane;
        const char* pm = d_pre ? static_cast<const char*>(d_pre) + (size_t)(w.s0 * c.pre_strides[0]) * es : nullptr;
        const char* qm = d_post ? static_cast<const char*>(d_post) + (size_t)(j0 * c.post_strides[0]) * es : nullptr;
        const bool wraps = c.axis == 0 && c.bc == XG_BC_PERIODIC;
        const void* hl = wraps && w.slo ? wrap[0] : nullptr;
        const void* hh = wraps && w.shi ? wrap[1] : nullptr;
        if (halo) {
          const int rc2 = halo(b, sshape, pm, d_fill, st, &hl, &hh);
          if (rc2) return rc2;
        }
        const char* am =
            d_pre_a ? static_cast<const char*>(d_pre_a) + (size_t)(w.s0 * t->pre_a_strides[0]) * es : nullptr;
        const int rc2 =
            t ? xg_stencil_pair_halo(c.dtype, src, b.in2, b.out[k], ndim, sshape, t->op_a, t->lo_a, t->hi_a, t->bc_a,
                                     t->fill_a, am, t->pre_a_strides, c.axis, c.op, c.lo, c.hi, c.bc, c.fill_value,
                                     pm, c.pre_strides, t->subtract, qm, c.post_strides, hl, hh, st)
              : xg_stencil2(c.op, c.dtype, src, b.out[k], ndim, sshape, c.axis, w.slo, w.shi,
                            (w.slo || w.shi) ? c.bc : XG_BC_NONE, c.fill_value, pm, c.pre_strides, qm, c.post_strides,
                            hl, hh, st);
        if (rc2) return rc2;
      }
      return XG_OK;
    };
    void* outs[kMaxOut];
    for (int k = 0; k < nout; ++k) outs[k] = cs[k].out;
    return ss.run(es, c0.in, vin, nout, outs, vout, launch, ex.rows(r0, r1));
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

// The face-connection copy list of the _connected entry points, described once for the whole field (see the header).
struct CopyList {
  int n, ndim;
  const int *side, *source;
  const int64_t *dst_offset, *src_offset, *shapes, *dst_strides, *src_strides;
  const int* negate;
};

// The copy-list checks, before any CUDA call: each copy writes a padded halo plane (plane_row elements per dim-0
// index of n0) from the field (row_in per index), the partner (partner_row, when given) or the fill constant, spans
// dim 0 in full, and stays inside both arrays; together the copies cover each padded plane.  *fill: some copy reads
// the constant.
int validate_copies(const std::string& who, const CopyList& cl, int lo, int hi, int64_t n0, int64_t plane_row,
                    int64_t row_in, bool partner, int64_t partner_row, bool* fill) {
  if (cl.n < 0) return xg_fail(XG_EINVAL, who + ": negative copy count");
  if (cl.n > 0 && (!cl.side || !cl.source || !cl.dst_offset || !cl.src_offset || !cl.shapes || !cl.dst_strides ||
                   !cl.src_strides || !cl.negate))
    return xg_fail(XG_EINVAL, who + ": null pointer in the copy list");
  if (cl.n > 0 && (cl.ndim < 1 || cl.ndim > XG_MAX_NDIM)) return xg_fail(XG_EINVAL, who + ": bad copy rank");
  int64_t covered[2] = {0, 0};
  *fill = false;
  for (int k = 0; k < cl.n; ++k) {
    const int64_t* sh = cl.shapes + (size_t)k * cl.ndim;
    const int64_t* ds = cl.dst_strides + (size_t)k * cl.ndim;
    const int64_t* ss = cl.src_strides + (size_t)k * cl.ndim;
    const int side = cl.side[k], source = cl.source[k];
    const std::string at = who + ": copy " + std::to_string(k) + ": ";
    if (side != 0 && side != 1) return xg_fail(XG_EINVAL, at + "side must be 0 (lo) or 1 (hi)");
    if (!(side ? hi : lo)) return xg_fail(XG_EINVAL, at + "writes a halo plane the call does not pad");
    if (source < kSrcField || source > kSrcFill)
      return xg_fail(XG_EINVAL, at + "source must be 0 (field), 1 (partner) or 2 (fill constant)");
    if (source == kSrcPartner && !partner) return xg_fail(XG_EINVAL, at + "reads a partner that was not given");
    *fill = *fill || source == kSrcFill;
    int64_t cells = 1;
    for (int d = 0; d < cl.ndim; ++d) {
      if (sh[d] < 0) return xg_fail(XG_EINVAL, at + "negative extent");
      cells *= sh[d];
    }
    covered[side] += cells;
    const int64_t src_row = source == kSrcField ? row_in : source == kSrcPartner ? partner_row : 0;
    if (sh[0] != n0 || ds[0] != plane_row || ss[0] != src_row)
      return xg_fail(XG_EINVAL, at + "must span dim 0 in full with the contiguous dim-0 strides");
    if (cells == 0) continue;
    int64_t a, b;
    copy_extent(cl.dst_offset[k], ds, sh, cl.ndim, &a, &b);
    if (a < 0 || b >= n0 * plane_row) return xg_fail(XG_EINVAL, at + "leaves the halo plane");
    copy_extent(cl.src_offset[k], ss, sh, cl.ndim, &a, &b);
    if (source == kSrcFill) {
      if (a != 0 || b != 0) return xg_fail(XG_EINVAL, at + "the fill constant is read with offset 0, strides 0");
    } else if (a < 0 || b >= n0 * src_row) {
      return xg_fail(XG_EINVAL, at + "leaves its source array");
    }
  }
  // the copies write disjoint cells, so together they must cover each padded plane exactly once
  if ((lo && covered[0] != n0 * plane_row) || (hi && covered[1] != n0 * plane_row))
    return xg_fail(XG_EINVAL, who + ": the copies do not cover the halo planes");
  return XG_OK;
}

// The fill constants the copy lists of a call read, in the field's dtype: the fill value of each stage, or the fill
// value then the weight of a fill edge (1).  Pageable: cudaMemcpyAsync stages them before it returns, so they must
// live until stencil_host / cumscan_halo_host / chain_host returns.
struct FillConsts {
  double f64[3];
  float f32[3];
  bool used = false;
  int64_t plane_row = 0;  // of the last list checked
  void set(int k, double v) {
    f64[k] = v;
    f32[k] = (float)v;
  }
  const void* host(int dtype) const { return used ? (dtype == XG_F32 ? (const void*)f32 : (const void*)f64) : nullptr; }
};

// The checks of a copy list that builds the halo planes of a field of `shape` padded by lo / hi along `axis`
// (validate_copies, with the field's dim-0 row and the plane row worked out here), and fill constant k set to
// `fill_value`.
int check_connected(const std::string& who, const CopyList& cl, int ndim, const int64_t* shape, int axis, int lo,
                    int hi, bool partner, int64_t partner_row, int k, double fill_value, FillConsts* fc) {
  int64_t row_in = 1;
  for (int d = 1; d < ndim; ++d) row_in *= shape[d];
  fc->plane_row = shape[axis] ? row_in / shape[axis] : 0;
  bool fill = false;
  const int rc = validate_copies(who, cl, lo, hi, shape[0], fc->plane_row, row_in, partner, partner_row, &fill);
  fc->used = fc->used || fill;
  fc->set(k, fill_value);
  return rc;
}

// The face connections' halo stage: the whole-field copy list rebased onto the slab's buffers (the field is b.in, the
// partner b.in2), `slab_shape[0]` rows high, in one xg_strided_copy_batch launch.  The rebased pointers and shapes are
// built per slab, on every path (small beside a slab's copies): the stage then keeps no state between slabs, so the
// members of a host device group can run it at once.
//
// With `pre_offset` the stage builds the halo of x * pre: the batch runs the list a second time, over the slab's rows
// of the pre-metric (copy k reads it at pre_offset[k] with pre_src_strides[k]; a fill copy reads the constant 1 after
// the fill value) into two weight planes in the scratch buffer.  One xg_binary launch per padded plane then multiplies
// it by its weight plane in place, so each halo cell is the gathered x times the gathered metric, rounded once, and a
// fill edge stays the fill value.
HaloFn copy_stage(const CopyList& cl, int dtype, int lo, int hi, const int64_t* pre_offset = nullptr,
                  const int64_t* pre_src_strides = nullptr, int axis = 0, int ndim = 0) {
  return [=](const SlabBufs& b, const int64_t* slab_shape, const void* pre, const void* d_fill, cudaStream_t st,
             const void** hl, const void** hh) -> int {
    const size_t es = dtype == XG_F32 ? 4 : 8;
    const size_t n = (size_t)cl.n, nd = (size_t)cl.ndim, m = pre_offset ? 2 * n : n;
    int64_t plane_elems = 1;  // the weight planes lie side by side in the scratch buffer
    for (int d = 0; d < ndim; ++d)
      if (d != axis) plane_elems *= slab_shape[d];
    const auto weight = [&](int side) { return static_cast<char*>(b.scratch) + (size_t)side * plane_elems * es; };
    std::vector<void*> dptr(m);
    std::vector<const void*> sptr(m);
    std::vector<int64_t> shp(m * nd);
    for (size_t k = 0; k < n; ++k) {
      const void* base = cl.source[k] == kSrcField ? b.in : cl.source[k] == kSrcPartner ? b.in2 : d_fill;
      dptr[k] = static_cast<char*>(b.plane[cl.side[k]]) + (size_t)cl.dst_offset[k] * es;
      sptr[k] = static_cast<const char*>(base) + (size_t)cl.src_offset[k] * es;
      for (size_t d = 0; d < nd; ++d) shp[k * nd + d] = d ? cl.shapes[k * nd + d] : slab_shape[0];
      if (!pre_offset) continue;
      dptr[n + k] = weight(cl.side[k]) + (size_t)cl.dst_offset[k] * es;
      sptr[n + k] = cl.source[k] == kSrcFill ? static_cast<const char*>(d_fill) + es
                                             : static_cast<const char*>(pre) + (size_t)pre_offset[k] * es;
      for (size_t d = 0; d < nd; ++d) shp[(n + k) * nd + d] = shp[k * nd + d];
    }
    // the unweighted list's strides go through as given; the weighted batch appends the metric copies' strides
    const int64_t *dstr = cl.dst_strides, *sstr = cl.src_strides;
    const int* neg = cl.negate;
    std::vector<int64_t> wdstr, wsstr;
    std::vector<int> wneg;
    if (pre_offset) {
      wdstr.assign(cl.dst_strides, cl.dst_strides + n * nd);
      wdstr.insert(wdstr.end(), cl.dst_strides, cl.dst_strides + n * nd);
      wsstr.assign(cl.src_strides, cl.src_strides + n * nd);
      wsstr.insert(wsstr.end(), pre_src_strides, pre_src_strides + n * nd);
      wneg.assign(cl.negate, cl.negate + n);
      wneg.resize(2 * n, 0);
      dstr = wdstr.data(), sstr = wsstr.data(), neg = wneg.data();
    }
    int rc2 = xg_strided_copy_batch(dtype, (int)m, dptr.data(), sptr.data(), cl.ndim, shp.data(), dstr, sstr, neg, st);
    if (rc2 == XG_ENOTIMPL) {  // some copy does not collapse to 5 dims: one launch per copy
      rc2 = XG_OK;
      for (size_t k = 0; rc2 == XG_OK && k < m; ++k)
        rc2 = xg_strided_copy(dtype, dptr[k], dstr + k * nd, sptr[k], sstr + k * nd, cl.ndim, shp.data() + k * nd,
                              neg[k], st);
    }
    if (rc2) return rc2;
    const int64_t unit = 1;
    for (int side = 0; pre_offset && side < 2; ++side) {
      if (!(side ? hi : lo)) continue;
      rc2 = xg_binary(XG_BIN_MUL, dtype, b.plane[side], weight(side), &unit, b.plane[side], 1, &plane_elems, st);
      if (rc2) return rc2;
    }
    if (lo) *hl = b.plane[0];
    if (hi) *hh = b.plane[1];
    return XG_OK;
  };
}

// ---------------------------------------------------------------------------------- the cumscan entry points
// The arguments of xg_cumscan_host_fold / _connected.
struct ScanCall {
  int dtype;
  const void* in;
  void* out;
  int ndim;
  const int64_t* shape;
  int axis, reverse, trim, pad_lo, pad_hi;
  const void* pre;
  const int64_t* pre_strides;
  const void* post;
  const int64_t* post_strides;
  int skipna, device;
};

// The checks of xg_cumscan_host, plus those of the slab loop (dim 0 a batch dim), before any CUDA call.  *scan_shape:
// the shape of the scanned field (trimmed, not yet padded), which the halo is taken from.
int validate_scan_call(const char* who, const ScanCall& s, int64_t* scan_shape) {
  const std::string w(who);
  if (!s.in || !s.out || !s.shape) return xg_fail(XG_EINVAL, w + ": null pointer");
  if (s.dtype != XG_F32 && s.dtype != XG_F64) return xg_fail(XG_EINVAL, w + ": dtype must be XG_F32 or XG_F64");
  if (s.ndim < 1 || s.ndim > XG_MAX_NDIM) return xg_fail(XG_EINVAL, w + ": bad ndim");
  if (s.axis < 0 || s.axis >= s.ndim) return xg_fail(XG_EINVAL, w + ": axis out of range");
  if (s.ndim < 2 || s.axis == 0)
    return xg_fail(XG_EINVAL, w + ": dim 0 is cut into slabs and must not be the scanned dim");
  for (int d = 0; d < s.ndim; ++d) {
    if (s.shape[d] < 0) return xg_fail(XG_EINVAL, w + ": negative extent");
    scan_shape[d] = s.shape[d];
  }
  if (s.trim < XG_TRIM_NONE || s.trim > XG_TRIM_DROP_FIRST) return xg_fail(XG_EINVAL, w + ": unknown trim");
  if (s.pad_lo < 0 || s.pad_lo > 1 || s.pad_hi < 0 || s.pad_hi > 1)
    return xg_fail(XG_EINVAL, w + ": pad widths must be 0 or 1");
  if ((s.pre && !s.pre_strides) || (s.post && !s.post_strides))
    return xg_fail(XG_EINVAL, w + ": metric strides missing");
  scan_shape[s.axis] -= s.trim != XG_TRIM_NONE ? 1 : 0;
  if (scan_shape[s.axis] < 1) return xg_fail(XG_EINVAL, w + ": no scanned row to take the halo from");
  return XG_OK;
}

// A cumscan entry point with a halo (arguments checked) on s.device: the field in slabs along dim 0, the metrics
// (and the `fill_host` constant, es bytes, when given) uploaded whole.  Per slab, the device sequence of
// Grid.cumsum on such a grid: xg_cumscan (pre, reverse, trim; no pad, no post) into the scratch buffer; `halo` builds
// the halo planes from the scanned slab; one xg_strided_copy_batch launch writes the scanned slab and its planes
// into the padded result; one xg_binary launch divides it by `post` in place.
int cumscan_halo_host(const char* who, const ScanCall& s, const int64_t* scan_shape, const HaloFn& halo,
                      const void* fill_host) {
  const size_t es = s.dtype == XG_F32 ? 4 : 8;
  const int ndim = s.ndim, ax = s.axis, lo = s.pad_lo;
  const int64_t kept = scan_shape[ax];
  int64_t out_shape[XG_MAX_NDIM], plane_shape[XG_MAX_NDIM];
  for (int d = 0; d < ndim; ++d) out_shape[d] = plane_shape[d] = scan_shape[d];
  out_shape[ax] = kept + s.pad_lo + s.pad_hi;
  plane_shape[ax] = 1;
  const View3 vin = view3(ndim, s.shape, 0), vout = view3(ndim, out_shape, 0);
  const View3 vscan = view3(ndim, scan_shape, 0), vplane = view3(ndim, plane_shape, 0);
  return spread(who, s.device, vout.L, false, [&](int device, int64_t r0, int64_t r1) -> int {
    Session ss;
    int rc = ss.open(device);
    if (rc) return rc;
    if (vout.L <= 0 || vout.R == 0) return XG_OK;
    const void *d_pre, *d_post, *d_fill;
    rc = ss.upload(kAuxPre, s.pre, s.pre ? operand_span(s.pre_strides, s.shape, ndim, es) : 0, &d_pre);
    if (rc == XG_OK)
      rc = ss.upload(kAuxPost, s.post, s.post ? operand_span(s.post_strides, out_shape, ndim, es) : 0, &d_post);
    if (rc == XG_OK) rc = ss.upload(kAuxFill, fill_host, es, &d_fill);
    if (rc == XG_OK) rc = ss.fence();
    if (rc) return rc;

    PipeExtra ex;
    ex.scratch_row_bytes = (size_t)vscan.R * es;
    ex.plane_row_bytes = (size_t)vplane.R * es;
    auto launch = [&](int64_t j0, int64_t j1, int64_t, int64_t, const SlabBufs& b, cudaStream_t st) -> int {
      int64_t sshape[XG_MAX_NDIM], cshape[XG_MAX_NDIM], oshape[XG_MAX_NDIM], pshape[XG_MAX_NDIM];
      for (int d = 0; d < ndim; ++d) {
        sshape[d] = s.shape[d];
        cshape[d] = scan_shape[d];
        oshape[d] = out_shape[d];
        pshape[d] = plane_shape[d];
      }
      sshape[0] = cshape[0] = oshape[0] = pshape[0] = j1 - j0;
      const char* pm = d_pre ? static_cast<const char*>(d_pre) + (size_t)(j0 * s.pre_strides[0]) * es : nullptr;
      const char* qm = d_post ? static_cast<const char*>(d_post) + (size_t)(j0 * s.post_strides[0]) * es : nullptr;
      int rc2 = xg_cumscan(s.dtype, b.in, b.scratch, ndim, sshape, ax, s.reverse, s.trim, 0, 0, XG_BC_NONE, 0.0, pm,
                           s.pre_strides, nullptr, nullptr, s.skipna, st);
      if (rc2) return rc2;
      SlabBufs scanned = b;  // the halo is taken from the scanned slab, as pad() takes it from the scanned field
      scanned.in = b.scratch;
      const void *hl = nullptr, *hh = nullptr;
      rc2 = halo(scanned, cshape, nullptr, d_fill, st, &hl, &hh);
      if (rc2) return rc2;
      // the scanned slab at row `lo` of the padded axis, its halo planes at row 0 and row lo + kept
      int64_t ostr[XG_MAX_NDIM], cstr[XG_MAX_NDIM], pstr[XG_MAX_NDIM];
      for (int64_t d = ndim - 1, o = 1, c = 1, p = 1; d >= 0; o *= oshape[d], c *= cshape[d], p *= pshape[d], --d) {
        ostr[d] = o;
        cstr[d] = c;
        pstr[d] = p;
      }
      char* o = static_cast<char*>(b.out[0]);
      void* dst[3] = {o + (size_t)(lo * ostr[ax]) * es, nullptr, nullptr};
      const void* src[3] = {b.scratch, nullptr, nullptr};
      int64_t shapes[3 * XG_MAX_NDIM], dstr[3 * XG_MAX_NDIM], sstr[3 * XG_MAX_NDIM];  // count x ndim, row-major
      int neg[3] = {0, 0, 0}, count = 1;
      for (int d = 0; d < ndim; ++d) {
        shapes[d] = cshape[d];
        dstr[d] = ostr[d];
        sstr[d] = cstr[d];
      }
      for (int side = 0; side < 2; ++side) {
        const void* plane = side ? hh : hl;
        if (!plane) continue;
        dst[count] = o + (size_t)((side ? lo + kept : 0) * ostr[ax]) * es;
        src[count] = plane;
        for (int d = 0; d < ndim; ++d) {
          shapes[count * ndim + d] = pshape[d];
          dstr[count * ndim + d] = ostr[d];
          sstr[count * ndim + d] = pstr[d];
        }
        ++count;
      }
      // dense arrays differ in the padded axis alone: every copy collapses to at most 3 dims
      rc2 = xg_strided_copy_batch(s.dtype, count, dst, src, ndim, shapes, dstr, sstr, neg, st);
      if (rc2 || !qm) return rc2;
      return xg_binary(XG_BIN_DIV, s.dtype, o, qm, s.post_strides, o, ndim, oshape, st);
    };
    void* outs[1] = {s.out};
    return ss.run(es, s.in, vin, 1, outs, &vout, launch, ex.rows(r0, r1));
  });
}

// ---------------------------------------------------------------------------------- the chain entry points
// The checks both chain entry points share, before any CUDA call: stage count, pointers, in-place, and per stage
// (cs[s], whose shape is shapes[s]) those of a halo stencil plus its op and distinct axes.  Fills shapes[0 ..
// nstage] (the result's shape last); cs[s].shape points at shapes[s].
int validate_chain(const char* who, int dtype, const void* in, void* out, int ndim, const int64_t* shape, int nstage,
                   const int* axis, const int* op, const int* lo, const int* hi, const int* bc, const double* fill,
                   int device, Call* cs, int64_t (*shapes)[XG_MAX_NDIM]) {
  const std::string w(who);
  if (!in || !out || !shape || !axis || !op || !lo || !hi || !fill) return xg_fail(XG_EINVAL, w + ": null pointer");
  if (nstage < 2 || nstage > 3) return xg_fail(XG_EINVAL, w + ": a chain has 2 or 3 stages");
  if (ndim < 1 || ndim > XG_MAX_NDIM) return xg_fail(XG_EINVAL, w + ": bad ndim");
  if (in == out) return xg_fail(XG_EINVAL, w + ": in-place operation is not supported");
  for (int d = 0; d < ndim; ++d) shapes[0][d] = shape[d];
  for (int s = 0; s < nstage; ++s) {
    const int b = bc ? bc[s] : ((lo[s] || hi[s]) ? XG_BC_FILL : XG_BC_NONE);  // connected: the planes pad
    cs[s] = Call{op[s], dtype, in, out, ndim, shapes[s], axis[s], lo[s], hi[s], b, fill[s],
                 nullptr, nullptr, nullptr, nullptr, device};
    int rc = validate_halo_call(who, cs[s]);
    if (rc) return rc;
    if (op[s] < XG_OP_DIFF || op[s] > XG_OP_MAX) return xg_fail(XG_EINVAL, w + ": unknown op");
    for (int k = 0; k < s; ++k)
      if (axis[k] == axis[s]) return xg_fail(XG_EINVAL, w + ": each axis may appear only once");
    for (int d = 0; d < ndim; ++d) shapes[s + 1][d] = shapes[s][d];
    shapes[s + 1][axis[s]] += lo[s] + hi[s] - 1;
  }
  return XG_OK;
}

// A chain entry point (arguments checked) on cs[0].device: the field in slabs along dim 0 and, per slab, the
// per-axis launch sequence of the device route: stage s builds its halo planes from its own input (`halo[s]`, empty
// for none) and runs one xg_stencil2 into the intermediate it writes (scratch, ping-pong) or the result slab.
// `fill_host`: the stages' fill constants (nstage elements of the field's dtype) the copy lists read, or nullptr.
int chain_host(const char* who, const Call* cs, const HaloFn* halo, int nstage, const int64_t (*shapes)[XG_MAX_NDIM],
               const void* fill_host) {
  const Call& c0 = cs[0];
  const size_t es = c0.dtype == XG_F32 ? 4 : 8;
  const int ndim = c0.ndim;
  const View3 vin = view3(ndim, shapes[0], 0), vout = view3(ndim, shapes[nstage], 0);
  int64_t mid[2] = {0, 0};  // elements per dim-0 row of the intermediates (stage 0's and stage 1's results)
  PipeExtra ex;
  for (int s = 0; s < nstage; ++s) {
    if (s + 1 < nstage) mid[s] = view3(ndim, shapes[s + 1], 0).R;
    const int64_t n = shapes[s][cs[s].axis];
    const size_t plane = n ? (size_t)(view3(ndim, shapes[s], 0).R / n) * es : 0;
    if (halo[s] && plane > ex.plane_row_bytes) ex.plane_row_bytes = plane;  // planes sized for the largest stage
  }
  ex.scratch_row_bytes = (size_t)(mid[0] + mid[1]) * es;
  ex.row_bytes = (vin.R + vout.R) * (int64_t)es + (int64_t)ex.scratch_row_bytes;  // the slab counts them all
  return spread(who, c0.device, vout.L, false, [&](int device, int64_t r0, int64_t r1) -> int {
    Session ss;
    int rc = ss.open(device);
    if (rc) return rc;
    if (vout.L <= 0 || vout.R == 0 || vin.R == 0) return XG_OK;
    const void* d_fill = nullptr;
    rc = ss.upload(kAuxFill, fill_host, (size_t)nstage * es, &d_fill);
    if (rc == XG_OK) rc = ss.fence();
    if (rc) return rc;
    auto launch = [&](int64_t j0, int64_t j1, int64_t, int64_t, const SlabBufs& b, cudaStream_t st) -> int {
      char* scratch = static_cast<char*>(b.scratch);
      void* mids[2] = {scratch, scratch + (size_t)((j1 - j0) * mid[0]) * es};
      const void* src = b.in;
      for (int s = 0; s < nstage; ++s) {
        const Call& c = cs[s];
        int64_t sshape[XG_MAX_NDIM];
        for (int d = 0; d < ndim; ++d) sshape[d] = shapes[s][d];
        sshape[0] = j1 - j0;
        const void *hl = nullptr, *hh = nullptr;
        if (halo[s]) {
          SlabBufs sb = b;  // the halo stages read b.in: point it at this stage's input
          sb.in = const_cast<void*>(src);
          const void* f = d_fill ? static_cast<const char*>(d_fill) + (size_t)s * es : nullptr;
          int rc2 = halo[s](sb, sshape, nullptr, f, st, &hl, &hh);
          if (rc2) return rc2;
        }
        void* dst = s + 1 == nstage ? b.out[0] : mids[s];
        int rc2 = xg_stencil2(c.op, c.dtype, src, dst, ndim, sshape, c.axis, c.lo, c.hi,
                              (c.lo || c.hi) ? c.bc : XG_BC_NONE, c.fill_value, nullptr, nullptr, nullptr, nullptr,
                              hl, hh, st);
        if (rc2) return rc2;
        src = dst;
      }
      return XG_OK;
    };
    void* outs[1] = {c0.out};
    return ss.run(es, c0.in, vin, 1, outs, &vout, launch, ex.rows(r0, r1));
  });
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
  return rc ? rc : stencil_host("xg_stencil2_host", 1, &c, nullptr, nullptr, 0, nullptr);
}

extern "C" int xg_stencil2_host_multi(int nout, const int* op, int dtype, const void* in, void* const* out, int ndim,
                                      const int64_t* shape, const int* axis, const int* lo, const int* hi,
                                      const int* bc, const double* fill_value, int device) {
  const char* who = "xg_stencil2_host_multi";
  const std::string w(who);
  if (!in || !out || !shape || !op || !axis || !lo || !hi || !bc || !fill_value)
    return xg_fail(XG_EINVAL, w + ": null pointer");
  if (nout < 1 || nout > kMaxOut)
    return xg_fail(XG_EINVAL, w + ": between 1 and " + std::to_string(kMaxOut) + " results per call");
  Call cs[kMaxOut];
  for (int k = 0; k < nout; ++k) {
    if (!out[k]) return xg_fail(XG_EINVAL, w + ": null result pointer");
    cs[k] = Call{op[k], dtype, in, out[k], ndim, shape, axis[k], lo[k], hi[k], bc[k], fill_value[k],
                 nullptr, nullptr, nullptr, nullptr, device};
    int rc = validate_call(who, cs[k]);
    if (rc) return rc;
    // slabs are cut along dim 0: a result operated along it must keep that extent (center <-> left / right shifts)
    // and be padded at the field's ends only
    if (axis[k] == 0 && lo[k] + hi[k] != 1)
      return xg_fail(XG_ENOTIMPL, w + ": outer / inner shifts along the outermost dimension; use xg_stencil2_host "
                                      "for that result");
    if (axis[k] == 0 && bc[k] == XG_BC_EXTRAPOLATE)
      return xg_fail(XG_ENOTIMPL, w + ": extrapolate along the outermost dimension");
    // xg_stencil2 rejects an unknown code even where it pads nothing, and is given XG_BC_NONE there
    if (bc[k] < XG_BC_NONE || bc[k] > XG_BC_EXTRAPOLATE)
      return xg_fail(XG_EINVAL, "xg_stencil2: unknown boundary condition");
  }
  for (int k = 0; k < nout; ++k) {
    int64_t out_shape[XG_MAX_NDIM];
    for (int d = 0; d < ndim; ++d) out_shape[d] = shape[d];
    out_shape[axis[k]] += lo[k] + hi[k] - 1;
    const View3 v = view3(ndim, out_shape, 0);
    if (v.L == 0 || v.R == 0) return xg_fail(XG_EINVAL, w + ": empty result");
  }
  return stencil_host(who, nout, cs, nullptr, nullptr, 0, nullptr);
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
            : stencil_host(who, 1, &c, nullptr, nullptr, 0,
                           fold_stage(c, false, seam_axis, skip, mirror, period, negate));
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
  const CopyList cl{ncopies, copy_ndim, side, source, dst_offset, src_offset, shapes, dst_strides, src_strides, negate};
  int rc = validate_halo_call(who.c_str(), c);
  if (rc) return rc;
  if (partner && !partner_shape) return xg_fail(XG_EINVAL, who + ": null partner shape");
  int64_t partner_row = 0;
  if (partner) {
    if (partner_shape[0] != shape[0])
      return xg_fail(XG_EINVAL, who + ": the partner component's dim-0 extent differs from the field's");
    partner_row = 1;
    for (int d = 1; d < ndim; ++d) {
      if (partner_shape[d] < 0) return xg_fail(XG_EINVAL, who + ": negative partner extent");
      partner_row *= partner_shape[d];
    }
  }
  FillConsts fc;
  rc = check_connected(who, cl, ndim, shape, axis, lo, hi, partner != nullptr, partner_row, 0, fill_value, &fc);
  return rc ? rc
            : stencil_host(who.c_str(), 1, &c, nullptr, partner, partner_row, copy_stage(cl, dtype, lo, hi),
                           fc.host(dtype));
}

extern "C" int xg_stencil2_host_connected_weighted(
    int op, int dtype, const void* in, void* out, int ndim, const int64_t* shape, int axis, int lo, int hi,
    double fill_value, const void* pre_metric, const int64_t* pre_strides, const void* post_metric,
    const int64_t* post_strides, int ncopies, int copy_ndim, const int* side, const int* source,
    const int64_t* dst_offset, const int64_t* src_offset, const int64_t* pre_offset, const int64_t* shapes,
    const int64_t* dst_strides, const int64_t* src_strides, const int64_t* pre_src_strides, const int* negate,
    int device) {
  const std::string who = "xg_stencil2_host_connected_weighted";
  const Call c{op, dtype, in, out, ndim, shape, axis, lo, hi, (lo || hi) ? XG_BC_FILL : XG_BC_NONE,
               fill_value, pre_metric, pre_strides, post_metric, post_strides, device};
  const CopyList cl{ncopies, copy_ndim, side, source, dst_offset, src_offset, shapes, dst_strides, src_strides, negate};
  int rc = validate_halo_call(who.c_str(), c);
  if (rc) return rc;
  if (!pre_metric || !pre_strides) return xg_fail(XG_EINVAL, who + ": null pre-metric");
  FillConsts fc;
  rc = check_connected(who, cl, ndim, shape, axis, lo, hi, false, 0, 0, fill_value, &fc);
  if (rc) return rc;
  if (ncopies > 0 && (!pre_offset || !pre_src_strides)) return xg_fail(XG_EINVAL, who + ": null pointer in the copy list");
  // the metric copies: inside the pre-metric, with its dim-0 stride, or the constant 1 at offset 0, strides 0
  const size_t es = dtype == XG_F32 ? 4 : 8;
  const int64_t pre_elems = (int64_t)(operand_span(pre_strides, shape, ndim, es) / es);
  for (int k = 0; k < ncopies; ++k) {
    const int64_t* ps = pre_src_strides + (size_t)k * copy_ndim;
    const std::string at = who + ": copy " + std::to_string(k) + ": ";
    if (ps[0] != (source[k] == kSrcFill ? 0 : pre_strides[0]))
      return xg_fail(XG_EINVAL, at + "the pre-metric copy must span dim 0 with the pre-metric's dim-0 stride");
    const int64_t* sh = shapes + (size_t)k * copy_ndim;
    int64_t cells = 1;
    for (int d = 0; d < copy_ndim; ++d) cells *= sh[d];
    if (cells == 0) continue;
    int64_t a, b;
    copy_extent(pre_offset[k], ps, sh, copy_ndim, &a, &b);
    if (source[k] == kSrcFill) {
      if (a != 0 || b != 0) return xg_fail(XG_EINVAL, at + "the constant 1 is read with offset 0, strides 0");
    } else if (a < 0 || b >= pre_elems) {
      return xg_fail(XG_EINVAL, at + "leaves the pre-metric");
    }
  }
  fc.set(1, 1.0);  // the weight of a fill edge
  return stencil_host(who.c_str(), 1, &c, nullptr, nullptr, 0,
                      copy_stage(cl, dtype, lo, hi, pre_offset, pre_src_strides, axis, ndim), fc.host(dtype), 2,
                      2 * (size_t)fc.plane_row * es);
}

extern "C" int xg_cumscan_host_fold(int dtype, const void* in, void* out, int ndim, const int64_t* shape, int axis,
                                    int reverse, int trim, int pad_lo, int pad_hi, const void* pre_metric,
                                    const int64_t* pre_strides, const void* post_metric, const int64_t* post_strides,
                                    int skipna, int seam_axis, int skip, int64_t mirror, int64_t period, int device) {
  const char* who = "xg_cumscan_host_fold";
  const ScanCall s{dtype, in, out, ndim, shape, axis, reverse, trim, pad_lo, pad_hi,
                   pre_metric, pre_strides, post_metric, post_strides, skipna, device};
  int64_t scan_shape[XG_MAX_NDIM];
  int rc = validate_scan_call(who, s, scan_shape);
  if (rc) return rc;
  if (pad_lo != 0 || pad_hi != 1)
    return xg_fail(XG_EINVAL, std::string(who) + ": the fold pads the north edge alone: pad_lo must be 0, pad_hi 1");
  // the fold row of the scanned field: its own rows and skip, no weight
  const Call c{0, dtype, in, out, ndim, scan_shape, axis, 0, 1, XG_BC_NONE, 0.0, nullptr, nullptr, nullptr, nullptr,
               device};
  rc = validate_fold(who, c, seam_axis, skip, mirror, period);
  return rc ? rc
            : cumscan_halo_host(who, s, scan_shape, fold_stage(c, false, seam_axis, skip, mirror, period, 0), nullptr);
}

extern "C" int xg_cumscan_host_connected(int dtype, const void* in, void* out, int ndim, const int64_t* shape,
                                         int axis, int reverse, int trim, int pad_lo, int pad_hi, double fill_value,
                                         const void* pre_metric, const int64_t* pre_strides, const void* post_metric,
                                         const int64_t* post_strides, int skipna, int ncopies, int copy_ndim,
                                         const int* side, const int* source, const int64_t* dst_offset,
                                         const int64_t* src_offset, const int64_t* shapes, const int64_t* dst_strides,
                                         const int64_t* src_strides, const int* negate, int device) {
  const char* who = "xg_cumscan_host_connected";
  const ScanCall s{dtype, in, out, ndim, shape, axis, reverse, trim, pad_lo, pad_hi,
                   pre_metric, pre_strides, post_metric, post_strides, skipna, device};
  const CopyList cl{ncopies, copy_ndim, side, source, dst_offset, src_offset, shapes, dst_strides, src_strides, negate};
  int64_t scan_shape[XG_MAX_NDIM];
  int rc = validate_scan_call(who, s, scan_shape);
  if (rc) return rc;
  // the copies read the scanned field
  FillConsts fc;
  rc = check_connected(who, cl, ndim, scan_shape, axis, pad_lo, pad_hi, false, 0, 0, fill_value, &fc);
  return rc ? rc : cumscan_halo_host(who, s, scan_shape, copy_stage(cl, dtype, pad_lo, pad_hi), fc.host(dtype));
}

extern "C" int xg_stencil_chain_host_fold(int dtype, const void* in, void* out, int ndim, const int64_t* shape,
                                          int nstage, const int* axis, const int* op, const int* lo, const int* hi,
                                          const int* bc, const double* fill, const int* fold, const int* seam_axis,
                                          const int* skip, const int64_t* mirror, const int64_t* period, int device) {
  const char* who = "xg_stencil_chain_host_fold";
  if (!bc || !fold || !seam_axis || !skip || !mirror || !period)
    return xg_fail(XG_EINVAL, std::string(who) + ": null pointer");
  Call cs[3];
  int64_t shapes[4][XG_MAX_NDIM];
  int rc = validate_chain(who, dtype, in, out, ndim, shape, nstage, axis, op, lo, hi, bc, fill, device, cs, shapes);
  if (rc) return rc;
  HaloFn halo[3];
  for (int s = 0; s < nstage; ++s) {
    if (fold[s] != 0 && fold[s] != 1) return xg_fail(XG_EINVAL, std::string(who) + ": fold must be 0 or 1");
    if (!fold[s]) continue;
    rc = validate_fold(who, cs[s], seam_axis[s], skip[s], mirror[s], period[s]);
    if (rc) return rc;
    halo[s] = fold_stage(cs[s], false, seam_axis[s], skip[s], mirror[s], period[s], 0);
  }
  return chain_host(who, cs, halo, nstage, shapes, nullptr);
}

extern "C" int xg_stencil_chain_host_connected(int dtype, const void* in, void* out, int ndim, const int64_t* shape,
                                               int nstage, const int* axis, const int* op, const int* lo,
                                               const int* hi, const double* fill, const int* ncopies, int copy_ndim,
                                               const int* side, const int* source, const int64_t* dst_offset,
                                               const int64_t* src_offset, const int64_t* shapes,
                                               const int64_t* dst_strides, const int64_t* src_strides,
                                               const int* negate, int device) {
  const std::string who = "xg_stencil_chain_host_connected";
  if (!ncopies) return xg_fail(XG_EINVAL, who + ": null pointer");
  Call cs[3];
  int64_t sh[4][XG_MAX_NDIM];
  int rc = validate_chain(who.c_str(), dtype, in, out, ndim, shape, nstage, axis, op, lo, hi, nullptr, fill, device,
                          cs, sh);
  if (rc) return rc;
  HaloFn halo[3];
  FillConsts fc;
  int64_t k0 = 0;  // the first copy of stage s in the concatenated lists
  for (int s = 0; s < nstage; ++s) {
    const size_t k = (size_t)k0, kd = (size_t)k0 * (size_t)(copy_ndim > 0 ? copy_ndim : 0);
    const CopyList cl{ncopies[s], copy_ndim, side ? side + k : nullptr, source ? source + k : nullptr,
                      dst_offset ? dst_offset + k : nullptr, src_offset ? src_offset + k : nullptr,
                      shapes ? shapes + kd : nullptr, dst_strides ? dst_strides + kd : nullptr,
                      src_strides ? src_strides + kd : nullptr, negate ? negate + k : nullptr};
    rc = check_connected(who + ": stage " + std::to_string(s), cl, ndim, sh[s], axis[s], lo[s], hi[s], false, 0, s,
                         fill[s], &fc);
    if (rc) return rc;
    if (lo[s] || hi[s]) halo[s] = copy_stage(cl, dtype, lo[s], hi[s]);
    k0 += cl.n;
  }
  return chain_host(who.c_str(), cs, halo, nstage, sh, fc.host(dtype));
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
  return rc ? rc : stencil_host("xg_stencil_pair_host", 1, &c, &t, b, view3(ndim, shape, 0).R, nullptr);
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
            : stencil_host(who, 1, &c, &t, b, view3(ndim, shape, 0).R,
                           fold_stage(c, true, seam_axis, skip, mirror, period, negate));
}
