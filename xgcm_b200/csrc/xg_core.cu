// Error plumbing, view collapsing and operand descriptors (host side of the C-ABI).
#include <stdio.h>
#include <string.h>

#include <string>

#include <atomic>

#include "xg_common.cuh"

static thread_local std::string g_last_error;
static std::atomic<long long> g_launches{0};
static thread_local const char* g_last_launch = "";

void xg_set_error(const std::string& msg) { g_last_error = msg; }

int xg_fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

int xg_check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    return xg_fail(XG_ECUDA, std::string(what) + ": " + cudaGetErrorString(e));
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  g_last_launch = what;  // always a string literal
  return XG_OK;
}

void xg_set_last_launch(const char* what) { g_last_launch = what; }

extern "C" const char* xg_last_launch(void) { return g_last_launch; }

extern "C" long long xg_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

extern "C" int xg_version(void) { return XG_VERSION; }

extern "C" const char* xg_last_error(void) { return g_last_error.c_str(); }

extern "C" int xg_device_info(int device, int* sm_count, int64_t* l2_bytes,
                              int64_t* hbm_bytes) {
  cudaDeviceProp p;
  cudaError_t e = cudaGetDeviceProperties(&p, device);
  if (e != cudaSuccess)
    return xg_fail(XG_ECUDA, std::string("cudaGetDeviceProperties: ") +
                                 cudaGetErrorString(e));
  if (sm_count) *sm_count = p.multiProcessorCount;
  if (l2_bytes) *l2_bytes = (int64_t)p.l2CacheSize;
  if (hbm_bytes) *hbm_bytes = (int64_t)p.totalGlobalMem;
  return XG_OK;
}

int xg_collapse_view(int ndim, const int64_t* shape, int axis, XgView* v) {
  if (ndim < 1 || ndim > XG_MAX_NDIM)
    return xg_fail(XG_EINVAL, "ndim must be in [1, " +
                                  std::to_string(XG_MAX_NDIM) + "]");
  if (axis < 0 || axis >= ndim) return xg_fail(XG_EINVAL, "axis out of range");
  v->outer = 1;
  v->inner = 1;
  for (int d = 0; d < ndim; ++d) {
    if (shape[d] < 0) return xg_fail(XG_EINVAL, "negative extent");
    if (d < axis) v->outer *= shape[d];
    if (d > axis) v->inner *= shape[d];
  }
  v->n = shape[axis];
  return XG_OK;
}

// Merge adjacent dims [d0, d1) of an operand into at most XG_MAXG groups so a
// flat C-order index over those dims maps to an element offset.
static int collapse_groups(const int64_t* shape, const int64_t* strides, int d0,
                           int d1, XgGroups* g, const char* what) {
  g->n = 0;
  g->small = 0;
  for (int k = 0; k < XG_MAXG; ++k) {
    g->size[k] = 1;
    g->stride[k] = 0;
  }
  for (int d = d0; d < d1; ++d) {
    if (shape[d] == 1) continue;  // contributes index 0 only
    int64_t st = strides[d];
    if (g->n > 0) {
      int k = g->n - 1;
      // previous group (size S, stride s) and this dim (size t, stride r) merge
      // iff s == r * t  (covers the all-broadcast case 0 == 0 * t)
      if (g->stride[k] == st * shape[d]) {
        g->size[k] *= shape[d];
        g->stride[k] = st;
        continue;
      }
    }
    if (g->n == XG_MAXG)
      return xg_fail(XG_ENOTIMPL,
                     std::string(what) +
                         ": broadcast pattern needs more than 4 index groups; "
                         "materialise the operand first");
    g->size[g->n] = shape[d];
    g->stride[g->n] = st;
    g->n++;
  }
  int64_t total = 1;
  bool small = true;
  for (int k = 0; k < g->n; ++k) {
    if (g->size[k] >= (1ll << 31)) small = false;
    if (total > (1ll << 31) / (g->size[k] > 0 ? g->size[k] : 1)) small = false;
    total *= g->size[k];
  }
  // the flat index handed to xg_groups_offset may exceed `total` only through broadcast
  // leading dims that were merged away, so bound it by the caller-visible extent as well
  int64_t extent = 1;
  for (int d = d0; d < d1; ++d) {
    if (shape[d] > 0 && extent > (1ll << 31) / shape[d]) small = false;
    extent *= shape[d] > 0 ? shape[d] : 1;
  }
  g->small = small ? 1 : 0;
  for (int k = 0; k < XG_MAXG; ++k) g->fd[k] = xg_fastdiv_make(small ? g->size[k] : 1);
  return XG_OK;
}

int xg_make_operand(const void* ptr, const int64_t* strides, int ndim,
                    const int64_t* shape, int axis, int vec, size_t elem_size,
                    XgOperand* op, const char* what) {
  memset(op, 0, sizeof(*op));
  op->ptr = ptr;
  if (!ptr) return XG_OK;
  if (!strides)
    return xg_fail(XG_EINVAL, std::string(what) + ": strides missing");
  for (int d = 0; d < ndim; ++d)
    if (strides[d] < 0)
      return xg_fail(XG_EINVAL, std::string(what) + ": negative stride");
  int rc = collapse_groups(shape, strides, 0, axis, &op->outer, what);
  if (rc) return rc;
  rc = collapse_groups(shape, strides, axis + 1, ndim, &op->inner, what);
  if (rc) return rc;
  op->axis_stride = shape[axis] == 1 ? 0 : strides[axis];
  if (op->inner.n == 0 || (op->inner.n == 1 && op->inner.stride[0] == 0)) {
    op->inner_mode = XG_IM_BCAST;
  } else if (op->inner.n == 1 && op->inner.stride[0] == 1) {
    op->inner_mode = XG_IM_CONTIG;
  } else {
    op->inner_mode = XG_IM_GENERIC;
    // offsets of the inner index lie in [0, span] (strides are non-negative), so any two differ by at most span
    int64_t span = 0;
    for (int k = 0; k < op->inner.n; ++k) {
      const int64_t ext = (op->inner.size[k] - 1) * op->inner.stride[k];
      span = (ext >= (1ll << 31) || span + ext >= (1ll << 31)) ? (1ll << 31) : span + ext;
    }
    op->wide_span = span >= (1ll << 31) ? 1 : 0;
  }
  op->vec_ok = 0;
  if (op->inner_mode == XG_IM_CONTIG && vec > 1) {
    bool ok = ((uintptr_t)ptr % (vec * elem_size)) == 0;
    ok = ok && (op->axis_stride % vec == 0);
    for (int k = 0; k < op->outer.n; ++k) ok = ok && (op->outer.stride[k] % vec == 0);
    op->vec_ok = ok ? 1 : 0;
  }
  return XG_OK;
}
