// Sharded operated axis: the one real exchange step of the path (SURVEY 8e) inside the C-ABI.
//
// Reference analogue: dask.array.map_overlap(depth=1) around the grid ufunc (xgcm/grid_ufunc.py:1057-1133):
// each block gets one cell of its neighbours along the core dim before the kernel runs.  Here each rank
// owns a contiguous block of the operated axis on its own GPU; one boundary plane per neighbour crosses
// NVLink through NCCL send/recv.
//
//   xg_comm_unique_id / xg_comm_init / xg_comm_destroy   a communicator of the library's own (NCCL is
//       loaded at run time with dlopen — the library links only the CUDA runtime; the unique id travels
//       through whatever the host uses for rendezvous, e.g. torch.distributed)
//   xg_halo_exchange      the bare ring step: send first / last plane, receive the neighbours', one NCCL group
//   xg_stencil2_sharded   the fused call:
//         side stream : k_pack_plane (boundary plane x pre-metric, strided -> contiguous; no torch copy)
//                       -> ncclGroupStart / Send / Recv / End
//         main stream : the ordinary fused stencil over the whole local block (edges with a neighbour get a
//                       placeholder boundary) — runs WHILE the planes are in flight
//         main stream : after the exchange event, k_edge_fix recomputes the one or two edge planes from
//                       the received halo (bit-identical to what the single-GPU kernel computes there)
//       so the exchange hides behind the interior work; only plane-sized kernels are serialised with it.
//
// NCCL errors map to XG_ENCCL (with ncclGetErrorString in xg_last_error()).
#include <dlfcn.h>
#include <string.h>

#include <mutex>

#include "xg_common.cuh"

namespace {

// ---- the slice of NCCL's ABI we use (nccl.h, stable since 2.x) ---------------------------------------
typedef struct ncclComm* ncclComm_t;
typedef struct {
  char internal[128];
} ncclUniqueId;
typedef int ncclResult_t;  // ncclSuccess == 0
constexpr int kNcclUint8 = 1;

struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  std::string error;
};

std::mutex g_nccl_mutex;
NcclApi g_nccl;

int load_nccl(const char* path) {
  std::lock_guard<std::mutex> lock(g_nccl_mutex);
  if (g_nccl.handle) return XG_OK;
  void* h = nullptr;
  if (path && *path) {
    h = dlopen(path, RTLD_NOW | RTLD_GLOBAL);
  } else {
    h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);  // the copy torch.distributed already loaded
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  }
  if (!h) {
    const char* e = dlerror();
    return xg_fail(XG_ENCCL, std::string("NCCL is not loadable: ") + (e ? e : "dlopen failed") +
                                 " (pass its path to xg_nccl_load)");
  }
  NcclApi api;
  api.handle = h;
#define XG_SYM(field, name)                                                         \
  api.field = reinterpret_cast<decltype(api.field)>(dlsym(h, name));                \
  if (!api.field) return xg_fail(XG_ENCCL, std::string("NCCL symbol missing: ") + name)
  XG_SYM(GetUniqueId, "ncclGetUniqueId");
  XG_SYM(CommInitRank, "ncclCommInitRank");
  XG_SYM(CommDestroy, "ncclCommDestroy");
  XG_SYM(Send, "ncclSend");
  XG_SYM(Recv, "ncclRecv");
  XG_SYM(GroupStart, "ncclGroupStart");
  XG_SYM(GroupEnd, "ncclGroupEnd");
  XG_SYM(GetErrorString, "ncclGetErrorString");
#undef XG_SYM
  g_nccl = api;
  return XG_OK;
}

int nccl_fail(const char* what, ncclResult_t r) {
  return xg_fail(XG_ENCCL, std::string(what) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "NCCL error"));
}
#define XG_NCCL(call, what)                 \
  do {                                      \
    ncclResult_t r_ = (call);               \
    if (r_ != 0) return nccl_fail(what, r_); \
  } while (0)
#define XG_CUDA(call)                                                               \
  do {                                                                              \
    cudaError_t e_ = (call);                                                        \
    if (e_ != cudaSuccess)                                                          \
      return xg_fail(XG_ECUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
  } while (0)

struct XgComm {
  ncclComm_t comm = nullptr;
  int nranks = 0, rank = 0, device = -1;
  cudaStream_t side = nullptr;  // the exchange runs here, next to the caller's stream
  cudaEvent_t ready = nullptr, done = nullptr;
};

// ---- plane kernels: one thread per 16-byte vector of a plane (scalar when the layout does not allow) -------
template <typename T>
struct PlaneArgs {
  const T* in;
  int64_t outer, n, inner;
  int64_t nvec_inner;  // vectors (or scalars) per row of `inner`
  bool small;          // outer * nvec_inner < 2^31
  XgFastDiv fd_nvi;    // multiply-high form of nvec_inner (valid with small)
  XgOperand pre, post;
};

// dst[o, i] = in[o, j, i] * pre[o, j, i]   (the halo carries field x metric, like the reference's padded array)
template <typename T, int VEC>
__global__ void __launch_bounds__(256) k_pack_plane(const PlaneArgs<T> a, int64_t j, T* dst) {
  const int64_t g = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (g >= a.outer * a.nvec_inner) return;
  int64_t o, iv;
  xg_divmod(g, a.nvec_inner, a.fd_nvi, a.small, o, iv);
  const int64_t i = iv * VEC;
  XgPack<T, VEC> v = xg_ld_stream<T, VEC>(a.in + (o * a.n + j) * a.inner + i);
  if (a.pre.ptr) {
    const XgOperandView<T, VEC> pv = xg_operand_view<T, VEC>(a.pre, xg_groups_offset(a.pre.outer, o), i);
    const XgPack<T, VEC> m = xg_ld_view<T, VEC>(pv, j * a.pre.axis_stride);
#pragma unroll
    for (int k = 0; k < VEC; ++k) v.v[k] = v.v[k] * m.v[k];
  }
  xg_st_stream<T, VEC>(dst + o * a.inner + i, v);
}

// out[o, j_out, i] = OP(P_lo, P_hi) / post : the plane next to a shard boundary, with the received halo as the
// missing operand.  low side: P_lo = halo, P_hi = in[., j_src, .] * pre;  high side: the other way round.
template <typename T, int VEC, int OP>
__global__ void __launch_bounds__(256) k_edge_fix(const PlaneArgs<T> a, const T* halo, int low_side, int64_t j_src,
                                                  int64_t j_out, int64_t n_out, T* out) {
  const int64_t g = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (g >= a.outer * a.nvec_inner) return;
  int64_t o, iv;
  xg_divmod(g, a.nvec_inner, a.fd_nvi, a.small, o, iv);
  const int64_t i = iv * VEC;
  XgPack<T, VEC> v = xg_ld_stream<T, VEC>(a.in + (o * a.n + j_src) * a.inner + i);
  const XgPack<T, VEC> h = xg_ld_stream<T, VEC>(halo + o * a.inner + i);
  if (a.pre.ptr) {
    const XgOperandView<T, VEC> pv = xg_operand_view<T, VEC>(a.pre, xg_groups_offset(a.pre.outer, o), i);
    const XgPack<T, VEC> m = xg_ld_view<T, VEC>(pv, j_src * a.pre.axis_stride);
#pragma unroll
    for (int k = 0; k < VEC; ++k) v.v[k] = v.v[k] * m.v[k];
  }
  XgPack<T, VEC> r;
#pragma unroll
  for (int k = 0; k < VEC; ++k) r.v[k] = low_side ? xg_apply_op<T, OP>(h.v[k], v.v[k]) : xg_apply_op<T, OP>(v.v[k], h.v[k]);
  if (a.post.ptr) {
    const XgOperandView<T, VEC> qv = xg_operand_view<T, VEC>(a.post, xg_groups_offset(a.post.outer, o), i);
    const XgPack<T, VEC> m = xg_ld_view<T, VEC>(qv, j_out * a.post.axis_stride);
#pragma unroll
    for (int k = 0; k < VEC; ++k) r.v[k] = r.v[k] / m.v[k];
  }
  xg_st_stream<T, VEC>(out + (o * n_out + j_out) * a.inner + i, r);
}

template <typename T, int VEC>
int launch_edge_fix_v(int op, const PlaneArgs<T>& a, const T* halo, int low_side, int64_t j_src, int64_t j_out,
                      int64_t n_out, T* out, unsigned blocks, cudaStream_t st) {
  switch (op) {
    case XG_OP_DIFF: k_edge_fix<T, VEC, XG_OP_DIFF><<<blocks, 256, 0, st>>>(a, halo, low_side, j_src, j_out, n_out, out); break;
    case XG_OP_INTERP: k_edge_fix<T, VEC, XG_OP_INTERP><<<blocks, 256, 0, st>>>(a, halo, low_side, j_src, j_out, n_out, out); break;
    case XG_OP_MIN: k_edge_fix<T, VEC, XG_OP_MIN><<<blocks, 256, 0, st>>>(a, halo, low_side, j_src, j_out, n_out, out); break;
    case XG_OP_MAX: k_edge_fix<T, VEC, XG_OP_MAX><<<blocks, 256, 0, st>>>(a, halo, low_side, j_src, j_out, n_out, out); break;
    default: return xg_fail(XG_EINVAL, "xg_stencil2_sharded: unknown op");
  }
  return xg_check_launch("xg_stencil2_sharded(edge)");
}

int exchange(XgComm* c, const void* send_lo, const void* send_hi, void* recv_lo, void* recv_hi, size_t bytes,
             int periodic, cudaStream_t st) {
  const int prev = (c->rank - 1 + c->nranks) % c->nranks, next = (c->rank + 1) % c->nranks;
  const bool has_prev = periodic || c->rank > 0, has_next = periodic || c->rank < c->nranks - 1;
  if (c->nranks == 1 || bytes == 0) return XG_OK;
  XG_NCCL(g_nccl.GroupStart(), "ncclGroupStart");
  // towards the upper neighbour: my last plane (its halo_lo); from it: its first plane (my halo_hi)
  if (send_hi && has_next) XG_NCCL(g_nccl.Send(send_hi, bytes, kNcclUint8, next, c->comm, st), "ncclSend");
  if (recv_lo && has_prev) XG_NCCL(g_nccl.Recv(recv_lo, bytes, kNcclUint8, prev, c->comm, st), "ncclRecv");
  if (send_lo && has_prev) XG_NCCL(g_nccl.Send(send_lo, bytes, kNcclUint8, prev, c->comm, st), "ncclSend");
  if (recv_hi && has_next) XG_NCCL(g_nccl.Recv(recv_hi, bytes, kNcclUint8, next, c->comm, st), "ncclRecv");
  XG_NCCL(g_nccl.GroupEnd(), "ncclGroupEnd");
  return XG_OK;
}

template <typename T>
int sharded_typed(XgComm* c, int op, const void* in, void* out, int ndim, const int64_t* shape, int axis, int lo, int hi,
                  int bc, double fill_value, const void* pre_metric, const int64_t* pre_strides,
                  const void* post_metric, const int64_t* post_strides, void* workspace, size_t workspace_bytes,
                  cudaStream_t st) {
  constexpr int VEC = XgVecWidth<T>::value;
  XgView v;
  int rc = xg_collapse_view(ndim, shape, axis, &v);
  if (rc) return rc;
  if (v.n == 0) return xg_fail(XG_EINVAL, "xg_stencil2_sharded: empty operated axis");
  const int64_t plane = v.outer * v.inner;
  const size_t pbytes = (size_t)plane * sizeof(T);
  const bool periodic = bc == XG_BC_PERIODIC;
  const bool has_prev = c->nranks > 1 && (periodic || c->rank > 0);
  const bool has_next = c->nranks > 1 && (periodic || c->rank < c->nranks - 1);
  const bool need_lo = lo && has_prev, need_hi = hi && has_next;    // halos I receive
  const bool give_hi = lo && has_next, give_lo = hi && has_prev;    // planes I owe (my last / my first)
  if (workspace_bytes < 4 * ((pbytes + 255) / 256 * 256) || (!workspace && plane))
    return xg_fail(XG_EINVAL, "xg_stencil2_sharded: workspace must hold 4 planes (256-byte aligned each)");
  const size_t slot = (pbytes + 255) / 256 * 256;
  char* ws = static_cast<char*>(workspace);
  T* send_lo = reinterpret_cast<T*>(ws);             // my first plane -> previous rank
  T* send_hi = reinterpret_cast<T*>(ws + slot);      // my last plane  -> next rank
  T* recv_lo = reinterpret_cast<T*>(ws + 2 * slot);  // previous rank's last plane
  T* recv_hi = reinterpret_cast<T*>(ws + 3 * slot);  // next rank's first plane

  PlaneArgs<T> pa;
  pa.in = static_cast<const T*>(in);
  pa.outer = v.outer;
  pa.n = v.n;
  pa.inner = v.inner;
  int64_t out_shape[XG_MAX_NDIM];
  for (int d = 0; d < ndim; ++d) out_shape[d] = shape[d];
  rc = xg_make_operand(pre_metric, pre_strides, ndim, shape, axis, VEC, sizeof(T), &pa.pre, "xg_stencil2_sharded(pre)");
  if (rc) return rc;
  rc = xg_make_operand(post_metric, post_strides, ndim, out_shape, axis, VEC, sizeof(T), &pa.post,
                       "xg_stencil2_sharded(post)");
  if (rc) return rc;
  constexpr int VECW = XgVecWidth<T>::value;
  // 16-byte vectors along `inner` when every row start stays aligned (workspace slots are 256-byte aligned)
  bool vec_ok = v.inner % VECW == 0 && ((uintptr_t)in % 16 == 0) && ((uintptr_t)out % 16 == 0) &&
                xg_vec_view_ok(pa.pre) && xg_vec_view_ok(pa.post);
  if (!vec_ok) {
    pa.pre.vec_ok = 0;
    pa.post.vec_ok = 0;
  }
  pa.nvec_inner = vec_ok ? v.inner / VECW : v.inner;
  pa.small = v.outer * pa.nvec_inner < (1ll << 31);
  pa.fd_nvi = xg_fastdiv_make(pa.small ? pa.nvec_inner : 1);
  const int64_t nblk = xg_ceil_div(v.outer * pa.nvec_inner, 256);
  if (nblk > 0x7fffffffLL) return xg_fail(XG_EINVAL, "xg_stencil2_sharded: plane too large");
  const unsigned blocks = (unsigned)(nblk > 0 ? nblk : 1);
  auto pack = [&](int64_t j, T* dst) -> int {
    if (vec_ok) k_pack_plane<T, VECW><<<blocks, 256, 0, c->side>>>(pa, j, dst);
    else k_pack_plane<T, 1><<<blocks, 256, 0, c->side>>>(pa, j, dst);
    return xg_check_launch("xg_stencil2_sharded(pack)");
  };
  auto fix = [&](const T* halo, int low_side, int64_t j_src, int64_t j_out, int64_t n_out_) -> int {
    if (vec_ok) return launch_edge_fix_v<T, VECW>(op, pa, halo, low_side, j_src, j_out, n_out_, static_cast<T*>(out), blocks, st);
    return launch_edge_fix_v<T, 1>(op, pa, halo, low_side, j_src, j_out, n_out_, static_cast<T*>(out), blocks, st);
  };

  // ---- side stream: pack + exchange, ordered after whatever produced `in` on the caller's stream
  XG_CUDA(cudaEventRecord(c->ready, st));
  XG_CUDA(cudaStreamWaitEvent(c->side, c->ready, 0));
  if (plane > 0) {
    if (give_lo) {
      rc = pack(0, send_lo);
      if (rc) return rc;
    }
    if (give_hi) {
      rc = pack(v.n - 1, send_hi);
      if (rc) return rc;
    }
  }
  rc = exchange(c, give_lo ? send_lo : nullptr, give_hi ? send_hi : nullptr, need_lo ? recv_lo : nullptr,
                need_hi ? recv_hi : nullptr, pbytes, periodic, c->side);
  if (rc) return rc;
  XG_CUDA(cudaEventRecord(c->done, c->side));

  // ---- main stream: the whole local block with the caller's boundary where this rank IS the edge of the
  // global axis, and a placeholder (extend) where a neighbour's plane is still in flight
  // lo + hi == 1: exactly one side is padded.  If a neighbour's plane is still in flight for it the launch takes a
  // placeholder boundary (extend) and the edge plane is recomputed below; otherwise this rank IS the edge of the
  // global axis and the caller's boundary applies.
  const bool neighbour = lo ? need_lo : need_hi;
  const int run_bc = neighbour ? XG_BC_EXTEND : bc;
  rc = xg_stencil2(op, sizeof(T) == 4 ? XG_F32 : XG_F64, in, out, ndim, shape, axis, lo, hi, run_bc, fill_value,
                   pre_metric, pre_strides, post_metric, post_strides, nullptr, nullptr, st);
  if (rc) return rc;
  // ---- after the exchange: recompute the edge planes from the received halos
  XG_CUDA(cudaStreamWaitEvent(st, c->done, 0));
  const int64_t n_out = v.n;  // lo + hi == 1
  if (plane > 0 && need_lo) {
    rc = fix(recv_lo, 1, 0, 0, n_out);
    if (rc) return rc;
  }
  if (plane > 0 && need_hi) {
    rc = fix(recv_hi, 0, v.n - 1, n_out - 1, n_out);
    if (rc) return rc;
  }
  return XG_OK;
}

}  // namespace

extern "C" int xg_nccl_load(const char* path) { return load_nccl(path); }

extern "C" int xg_comm_unique_id(void* id128) {
  if (!id128) return xg_fail(XG_EINVAL, "xg_comm_unique_id: null pointer");
  int rc = load_nccl(nullptr);
  if (rc) return rc;
  ncclUniqueId id;
  XG_NCCL(g_nccl.GetUniqueId(&id), "ncclGetUniqueId");
  memcpy(id128, id.internal, sizeof(id.internal));
  return XG_OK;
}

extern "C" int xg_comm_init(const void* id128, int nranks, int rank, void** comm) {
  if (!id128 || !comm) return xg_fail(XG_EINVAL, "xg_comm_init: null pointer");
  if (nranks < 1 || rank < 0 || rank >= nranks) return xg_fail(XG_EINVAL, "xg_comm_init: bad rank / nranks");
  int rc = load_nccl(nullptr);
  if (rc) return rc;
  XgComm* c = new XgComm();
  c->nranks = nranks;
  c->rank = rank;
  cudaError_t e = cudaGetDevice(&c->device);
  if (e != cudaSuccess) {
    delete c;
    return xg_fail(XG_ECUDA, std::string("cudaGetDevice: ") + cudaGetErrorString(e));
  }
  ncclUniqueId id;
  memcpy(id.internal, id128, sizeof(id.internal));
  ncclResult_t r = g_nccl.CommInitRank(&c->comm, nranks, id, rank);
  if (r != 0) {
    delete c;
    return nccl_fail("ncclCommInitRank", r);
  }
  // highest priority: the exchange's few CTAs must get SM resources as soon as blocks of the (much larger)
  // stencil grid retire, or they would only run once that grid is exhausted — no overlap
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
  if (cudaStreamCreateWithPriority(&c->side, cudaStreamNonBlocking, prio_hi) != cudaSuccess ||
      cudaEventCreateWithFlags(&c->ready, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&c->done, cudaEventDisableTiming) != cudaSuccess) {
    g_nccl.CommDestroy(c->comm);
    delete c;
    return xg_fail(XG_ECUDA, "xg_comm_init: could not create the exchange stream / events");
  }
  *comm = c;
  return XG_OK;
}

extern "C" int xg_comm_destroy(void* comm) {
  XgComm* c = static_cast<XgComm*>(comm);
  if (!c) return XG_OK;
  if (c->side) cudaStreamSynchronize(c->side);
  if (c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
  if (c->ready) cudaEventDestroy(c->ready);
  if (c->done) cudaEventDestroy(c->done);
  if (c->side) cudaStreamDestroy(c->side);
  delete c;
  return XG_OK;
}

extern "C" int xg_halo_exchange(void* comm, const void* send_lo, const void* send_hi, void* recv_lo, void* recv_hi,
                                size_t bytes, int periodic, void* stream) {
  XgComm* c = static_cast<XgComm*>(comm);
  if (!c) return xg_fail(XG_EINVAL, "xg_halo_exchange: null communicator");
  return exchange(c, send_lo, send_hi, recv_lo, recv_hi, bytes, periodic, static_cast<cudaStream_t>(stream));
}

extern "C" int xg_stencil2_sharded(void* comm, int op, int dtype, const void* in, void* out, int ndim,
                                   const int64_t* shape, int axis, int lo, int hi, int bc, double fill_value,
                                   const void* pre_metric, const int64_t* pre_strides, const void* post_metric,
                                   const int64_t* post_strides, void* workspace, size_t workspace_bytes, void* stream) {
  XgComm* c = static_cast<XgComm*>(comm);
  if (!c) return xg_fail(XG_EINVAL, "xg_stencil2_sharded: null communicator");
  if (!in || !out || !shape) return xg_fail(XG_EINVAL, "xg_stencil2_sharded: null pointer");
  if (lo < 0 || lo > 1 || hi < 0 || hi > 1 || lo + hi != 1)
    // grid_ufunc.py:1136-1159: map_overlap cannot change the chunk length either
    return xg_fail(XG_ENOTIMPL,
                   "xg_stencil2_sharded: a sharded operated axis supports only length-preserving shifts "
                   "(center <-> left / right)");
  if (bc <= XG_BC_NONE || bc > XG_BC_EXTEND)
    return xg_fail(XG_EINVAL, "xg_stencil2_sharded: boundary must be periodic, fill or extend");
  if (in == out) return xg_fail(XG_EINVAL, "xg_stencil2_sharded: in-place operation is not supported");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == XG_F32)
    return sharded_typed<float>(c, op, in, out, ndim, shape, axis, lo, hi, bc, fill_value, pre_metric, pre_strides,
                                post_metric, post_strides, workspace, workspace_bytes, st);
  if (dtype == XG_F64)
    return sharded_typed<double>(c, op, in, out, ndim, shape, axis, lo, hi, bc, fill_value, pre_metric, pre_strides,
                                 post_metric, post_strides, workspace, workspace_bytes, st);
  return xg_fail(XG_EINVAL, "xg_stencil2_sharded: dtype must be XG_F32 or XG_F64");
}
