// The slab engine of the host-buffer entry points (defined in xg_host.cu): one workspace per device, one pipeline
//     H2D(slab s+1)  ||  kernel(s)(slab s)  ||  D2H(slab s-1)
// on three streams with three slots.  The entry points validate their arguments, then, through spread(), on each
// device of the call (one, or the members of a host device group, each with its block of result rows): open a
// Session, upload their whole-call operands, and pass Session::run a [C][L][R] view of the field, a launch callback
// and the block.
#pragma once

#include <functional>
#include <mutex>

#include "xg_common.cuh"

namespace xg_host {

constexpr int kMaxOut = 8;  // results per slab

// Operands uploaded whole, once per call, each into its own workspace buffer
enum Aux {
  kAuxPre,          // pre-metric, or the weight of xg_wreduce_host
  kAuxPost,         // post-metric
  kAuxPreA,         // pre-metric of a pair's x term
  kAuxWrapLo,       // periodic wrap plane below the first slab of dim 0 (plane n0 - 1)
  kAuxWrapHi,       // ... and above the last one (plane 0)
  kAuxFill,         // fill constant the unconnected face edges copy from
  kAuxTheta,        // a broadcast theta
  kAuxThetaBounds,  // its bounds, made on the device from centres
  kAuxTarget,       // target levels of xg_vinterp_linear_host, or the bins of xg_vinterp_conservative_host
  kAuxPartial,      // per-slab partials of xg_wreduce_host_multi over every dim, and what their last launches make
  kNumAux
};

// [C][L][R] view of a C-contiguous array around the slab dimension (extent L)
struct View3 {
  int64_t C, L, R;
};
View3 view3(int ndim, const int64_t* shape, int sd);

struct SlabBufs {  // device buffers a slab's kernels use
  void* in;
  void* in2;       // the second input's rows, nullptr without one
  void* scratch;   // nullptr without scratch
  void* plane[2];  // the lo / hi halo planes, nullptr without them
  void* const* out;
};

// launch(j0, j1, i0, i1, bufs, stream): kernels for result rows [j0, j1) given input rows [i0, i1)
typedef std::function<int(int64_t, int64_t, int64_t, int64_t, const SlabBufs&, cudaStream_t)> LaunchFn;

// Optional parts of a pipeline.
struct PipeExtra {
  // Input rows [j0 - lo_rows, j1 + hi_rows) of result rows [j0, j1), clipped to the input
  int64_t lo_rows = 0, hi_rows = 0;
  // The edge slabs hold at least two input rows, with no one-row tail (an extrapolated halo along the slab dim)
  bool edge_pairs = false;
  // A second host input that goes up in the same slabs, rows [j0, j1) without halo (its own view, same L)
  const void* hin2 = nullptr;
  View3 in2{0, 0, 0};
  // Buffers only the kernels touch, per slab row: a scratch buffer and two halo planes
  size_t scratch_row_bytes = 0, plane_row_bytes = 0;
  // Bytes one slab row moves, which size the slabs (0: the first input's)
  int64_t row_bytes = 0;
  // Result rows [r0, r1) of the slab dim that run streams (r1 < 0: to the end); the slabs are sized within them,
  // while row indices, halo rows and field edges stay those of the whole field
  int64_t r0 = 0, r1 = -1;

  PipeExtra rows(int64_t a, int64_t b) const {
    PipeExtra e = *this;
    e.r0 = a;
    e.r1 = b;
    return e;
  }
};

struct Workspace;

// One host call on one device: the device selected and its workspace locked until the call returns, when the
// workspace's three streams are drained (so no copy or kernel outlives the call, whatever it returns).
class Session {
 public:
  ~Session();
  int open(int device);
  // Upload `bytes` of `host` into aux buffer `a` on the upload stream; *dev = its device address (nullptr, and
  // nothing uploaded, when host is nullptr)
  int upload(Aux a, const void* host, size_t bytes, const void** dev);
  // Aux buffer `a` of at least `bytes`, for kernels to fill on kernel_stream()
  int aux(Aux a, size_t bytes, void** dev);
  int fence();  // kernels on kernel_stream() see the uploads
  cudaStream_t kernel_stream() const;
  // Copy `bytes` at `dev` to `host` after the kernels on kernel_stream(), and wait for it
  int download(void* host, const void* dev, size_t bytes);
  // Stream `hin` (view `in`) through `launch` into the `nout` results hout[k] (view out[k]); the results share
  // one L, which may differ from the input's.
  int run(size_t es, const void* hin, const View3& in, int nout, void* const* hout, const View3* out,
          const LaunchFn& launch, const PipeExtra& ex = PipeExtra());

 private:
  Workspace* w_ = nullptr;
  std::unique_lock<std::mutex> lock_;
};

// bytes spanned by a broadcast operand laid out with `strides` over `shape`
size_t operand_span(const int64_t* strides, const int64_t* shape, int ndim, size_t es);

int64_t slab_budget_bytes();  // XG_HOST_SLAB_MB, default 128 MiB

// body(device, r0, r1): one device's share of a host call, result rows [r0, r1) of the slab dim (extent L)
typedef std::function<int(int, int64_t, int64_t)> BlockFn;

// Run a host call on `device`: a device index, or a handle of xg_host_group.  A device index runs body(device, 0, L)
// on the calling thread.  A group cuts [0, L) into contiguous near-equal blocks, at most one per member (one when
// `split` is false), with no one-row block at a field edge under `edge_pairs`, and runs body(member, r0, r1) on
// one thread per block; every thread is joined, error or not.  Returns the first failing block's status, with its
// xg_last_error() text, and leaves the first block's xg_last_launch() label on the calling thread.  An unknown
// handle gives XG_EINVAL before any CUDA call.
int spread(const char* who, int device, int64_t L, bool edge_pairs, const BlockFn& body, bool split = true);

}  // namespace xg_host
