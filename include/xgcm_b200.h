/*
 * xgcm_b200.h — C-ABI of the H100-native (sm_90a) grid-ufunc stencil engine.
 *
 * This is the drop-in boundary for xgcm's data-parallel hot path.  Every entry
 * point replaces one numeric site of the reference (paths relative to the
 * xgcm source tree, snapshot 052b033a):
 *
 *   xg_stencil2        <- xgcm/padding.py:575-616 (_pad_basic -> np.pad)
 *                         + xgcm/gridops.py:23-24,76-77,123-126,172-175
 *                           (diff_forward / interp_forward / pairwise min,max)
 *                         + xgcm/grid.py:806-808,830-832,1576-1578
 *                           (metric multiply before / divide after)
 *   xg_cumscan         <- xgcm/grid.py:1306-1391 (metric, flip, cumsum, trim, pad)
 *                         + xgcm/grid.py:1411-1414 (metric divide)
 *   xg_wreduce         <- xgcm/grid.py:1598-1605 (integrate) and :1680-1685 (average)
 *   xg_vinterp_linear  <- xgcm/transform.py:15-41,44-85 (_interp_1d_linear)
 *   xg_vinterp_conservative <- xgcm/transform.py:88-191 (_interp_1d_conservative)
 *   xg_pad             <- xgcm/padding.py:765-871 (pad) for callers that want the
 *                         padded array itself (custom grid ufuncs)
 *   xg_strided_copy    <- xgcm/padding.py:260-572 (_pad_face_connections: one connected edge)
 *   xg_fold_rows       <- xgcm/padding.py:619-684 (_fold_north_halo: the north-fold halo rows)
 *   xg_binary / xg_unary
 *                      <- the xarray broadcast arithmetic around the hot path
 *                         (xgcm/grid.py:808,832,1578,1599,1657)
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / numpy / C++ types.
 *   - every array is C-contiguous; `shape` has `ndim` entries; `axis` is the
 *     operated dimension.  Internally any such array collapses to
 *     (outer, n, inner); inner == 1 selects the innermost-axis kernels.
 *   - "device" entry points take DEVICE pointers and a cudaStream_t (passed as
 *     void*); launches are asynchronous; nothing is allocated.
 *   - "*_host" entry points take HOST pointers; the library stages through the
 *     device in slabs along the outermost dimension with copy/compute overlap.
 *   - metric operands broadcast against the field: `*_strides` gives the
 *     metric's ELEMENT stride for every dim of the field (0 = broadcast).
 *     pre_* is laid out against the INPUT shape, post_* against the OUTPUT shape.
 *   - returns 0 on success, a negative xg_status otherwise; xg_last_error()
 *     returns a thread-local message.  CUDA errors never abort the process.
 *   - re-entrant: no global mutable state apart from an init-once device
 *     property cache.
 */
#ifndef XGCM_B200_H
#define XGCM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define XG_API __attribute__((visibility("default")))
#else
#define XG_API
#endif

#define XG_VERSION 100 /* 0.1.0 */
#define XG_MAX_NDIM 8

typedef enum {
  XG_OK = 0,
  XG_EINVAL = -1,   /* -> ValueError   */
  XG_ENOTIMPL = -2, /* -> NotImplementedError */
  XG_ECUDA = -3,    /* -> RuntimeError */
  XG_ENCCL = -4     /* -> RuntimeError */
} xg_status;

typedef enum { XG_F32 = 0, XG_F64 = 1 } xg_dtype;

/* gridops.py:23-24 / :76-77 / :123-126 / :172-175 */
typedef enum { XG_OP_DIFF = 0, XG_OP_INTERP = 1, XG_OP_MIN = 2, XG_OP_MAX = 3 } xg_op;

/* padding.py:15-19 ("periodic"->wrap, "fill"->constant, "extend"->edge).
 * XG_BC_NONE with a non-zero halo width is an error (padding.py:601-608).
 * XG_BC_EXTRAPOLATE (halo = 2*edge - next) has no counterpart in the
 * reference snapshot: opt-in, parity unpinned. */
typedef enum {
  XG_BC_NONE = 0,
  XG_BC_PERIODIC = 1,
  XG_BC_FILL = 2,
  XG_BC_EXTEND = 3,
  XG_BC_EXTRAPOLATE = 4
} xg_bc;

/* grid.py:1326-1383 trim table of cumsum */
typedef enum { XG_TRIM_NONE = 0, XG_TRIM_DROP_LAST = 1, XG_TRIM_DROP_FIRST = 2 } xg_trim;

/* WVALID: sum of the weights of the cells the MEAN would keep (its denominator), for multi-axis means. */
typedef enum { XG_REDUCE_SUM = 0, XG_REDUCE_MEAN = 1, XG_REDUCE_WVALID = 2 } xg_reduce_mode;

typedef enum {
  XG_BIN_MUL = 0, XG_BIN_DIV = 1, XG_BIN_ADD = 2, XG_BIN_SUB = 3,
  XG_BIN_DIVNZ = 4 /* a / b, NaN where b == 0 (a weighted mean over no valid weight) */
} xg_binop;

XG_API int xg_version(void);
XG_API const char* xg_last_error(void);

/* Number of kernels this library has launched in this process (all threads). */
XG_API long long xg_launch_count(void);

/* Label of the kernel the calling thread launched last ("" before any launch): lets tests and the
 * bench state WHICH code path served a call (e.g. the TMA-staged transform vs its fallback). */
XG_API const char* xg_last_launch(void);

/* Device properties the host side needs for planning (SM count, L2 bytes). */
XG_API int xg_device_info(int device, int* sm_count, int64_t* l2_bytes, int64_t* hbm_bytes);

/*
 * Fused halo-pad + 2-point stencil + optional metric multiply/divide along one
 * axis.  out[..., j, ...] = OP(P[j], P[j+1]) / post, where P is the array
 * (in * pre) padded by `lo` cells below and `hi` cells above (lo, hi in {0,1})
 * according to `bc`.  Output length along axis = n + lo + hi - 1.
 *
 * halo_lo / halo_hi: optional device planes of shape (outer, inner) that supply
 * the halo instead of `bc` (used when the operated axis is sharded across GPUs,
 * cf. grid_ufunc.py:1057-1133 map_overlap); values are taken as-is (already
 * metric-weighted).
 */
XG_API int xg_stencil2(int op, int dtype, const void* in, void* out, int ndim,
                const int64_t* shape, int axis, int lo, int hi, int bc,
                double fill_value, const void* pre_metric,
                const int64_t* pre_strides, const void* post_metric,
                const int64_t* post_strides, const void* halo_lo,
                const void* halo_hi, void* stream);

/*
 * 2 or 3 single-axis stencils fused into one pass: the result equals applying xg_stencil2 along
 * axes[0], then axes[1] (, then axes[2]) — each with its own op / halo / boundary acting on the
 * previous intermediate, every intermediate rounded to the field dtype — but the field is read
 * and written once (xgcm/grid.py:798-832 makes one full pass per axis).  Boundaries: periodic,
 * fill, extend.  Output extent along axes[k] = n + lo[k] + hi[k] - 1.
 */
XG_API int xg_stencil_multi(int dtype, const void* in, void* out, int ndim, const int64_t* shape,
                     int naxes, const int* axes, const int* ops, const int* lo, const int* hi,
                     const int* bc, const double* fill_value, void* stream);

/*
 * Two-FIELD composite in one pass (SURVEY 8f N1: divergence, vorticity ...):
 *   out = ( OPa(pad_a(a * pre_a)) along the INNERMOST dim  (+ | -)  OPb(pad_b(b * pre_b)) along axis_b ) / post
 * a, b, out and every metric are laid out against the one common `shape` (both stencils are length
 * preserving: lo + hi == 1).  Rounded operator by operator like the chain of Grid.diff / xarray arithmetic it
 * replaces (xgcm docs/ufunc_examples.md:105-153, grid.py:796-832): a*pre_a, OPa, b*pre_b, OPb, the sum or
 * difference (`subtract`: 0 = a + b, 1 = term a - term b, 2 = term b - term a), the division.
 * Boundaries: periodic, fill, extend.
 */
XG_API int xg_stencil_pair(int dtype, const void* a, const void* b, void* out, int ndim,
                    const int64_t* shape, int op_a, int lo_a, int hi_a, int bc_a, double fill_a,
                    const void* pre_a, const int64_t* pre_a_strides, int axis_b, int op_b, int lo_b,
                    int hi_b, int bc_b, double fill_b, const void* pre_b,
                    const int64_t* pre_b_strides, int subtract, const void* post,
                    const int64_t* post_strides, void* stream);

/*
 * xg_stencil_pair with optional halo planes for the term along axis_b (e.g. the folded north row of a
 * tripolar grid).  halo_lo_b / halo_hi_b: contiguous device planes of the common shape with extent 1
 * along axis_b, already weighted (b * pre_b at their source cell, as the halo planes of xg_stencil2);
 * each replaces bc_b on its side.  NULL planes: exactly xg_stencil_pair.
 */
XG_API int xg_stencil_pair_halo(int dtype, const void* a, const void* b, void* out, int ndim,
                                const int64_t* shape, int op_a, int lo_a, int hi_a, int bc_a, double fill_a,
                                const void* pre_a, const int64_t* pre_a_strides, int axis_b, int op_b,
                                int lo_b, int hi_b, int bc_b, double fill_b, const void* pre_b,
                                const int64_t* pre_b_strides, int subtract, const void* post,
                                const int64_t* post_strides, const void* halo_lo_b, const void* halo_hi_b,
                                void* stream);

/*
 * Cumulative sum along one axis with xgcm's position-shift bookkeeping:
 * c = cumsum(in * pre) (from the high end when reverse), then trim, then pad
 * (pad_lo, pad_hi in {0,1}) with `bc` applied to the cumsum'd data, then / post.
 * skipna != 0 treats NaN as 0 (xarray's default for float data).
 * Summation order is strictly sequential along the axis (numpy's order).
 */
XG_API int xg_cumscan(int dtype, const void* in, void* out, int ndim,
               const int64_t* shape, int axis, int reverse, int trim,
               int pad_lo, int pad_hi, int bc, double fill_value,
               const void* pre_metric, const int64_t* pre_strides,
               const void* post_metric, const int64_t* post_strides,
               int skipna, void* stream);

/*
 * Weighted reduction along one axis: out = sum_j in[j] * w[j]   (XG_REDUCE_SUM)
 * or  sum_j in*w / sum_j w over non-NaN in  (XG_REDUCE_MEAN; skipna == 0 keeps NaN cells, so the result is
 * NaN wherever the line holds one, like da.weighted(w).mean(skipna=False)).
 * weight may be NULL (plain sum / mean).  Output shape = shape without `axis`.
 */
XG_API int xg_wreduce(int dtype, const void* in, const void* weight,
               const int64_t* w_strides, void* out, int ndim,
               const int64_t* shape, int axis, int mode, int skipna,
               void* stream);

/*
 * Linear interpolation of phi (defined on theta) onto target levels, per
 * column along `axis`; output dimension is appended LAST (transform.py:233-249).
 * phi: `shape`; theta: broadcast against phi via theta_strides (a shared 1-D
 * coordinate has stride 1 on `axis` and 0 elsewhere); target: m levels, either one
 * shared contiguous vector (target_strides == NULL) or one vector per column:
 * target_strides[d] (d != axis) = stride over column dim d, target_strides[axis] =
 * stride between consecutive levels.
 * out: shape-without-axis + (m,).  fp64 arithmetic, rounded once.
 */
XG_API int xg_vinterp_linear(int dtype, const void* phi, const void* theta,
                      const int64_t* theta_strides, const void* target,
                      const int64_t* target_strides, int64_t m, void* out, int ndim, const int64_t* shape,
                      int axis, int mask_edges, int bypass_checks,
                      int logarithmic, void* stream);

/*
 * Conservative remapping (transform.py:88-191): phi holds an extensive quantity per source
 * cell (n cells along `axis`), theta the n + 1 cell bounds (broadcast via theta_strides),
 * target_bins m ASCENDING bin edges (shared 1-D).  out: shape-without-axis + (m - 1,), bins
 * reversed when flip_out (the caller was given decreasing edges).  Field-dtype arithmetic,
 * contributions per bin added in source-cell order, bins that receive nothing are NaN.
 */
XG_API int xg_vinterp_conservative(int dtype, const void* phi, const void* theta,
                            const int64_t* theta_strides, const void* target_bins,
                            int64_t m, int flip_out, void* out, int ndim,
                            const int64_t* shape, int axis, void* stream);

/* The padded array itself (padding.py:765-871), one axis per call. */
XG_API int xg_pad(int dtype, const void* in, void* out, int ndim,
           const int64_t* shape, int axis, int lo, int hi, int bc,
           double fill_value, void* stream);

/* out = a (op) b with b broadcast against a's shape via b_strides. */
XG_API int xg_binary(int binop, int dtype, const void* a, const void* b,
              const int64_t* b_strides, void* out, int ndim,
              const int64_t* shape, void* stream);

/*
 * dst[sum_d i_d * dst_strides[d]] = (negate ? -1 : 1) * src[sum_d i_d * src_strides[d]] for every
 * index tuple in `shape`.  Strides are in ELEMENTS and may be negative; dst / src point at the
 * element with index (0, ..., 0).  This is the data movement of face-connection padding
 * (xgcm/padding.py:414-541: slice the neighbour face, swap the horizontal dims, flip across /
 * along the seam, sign-flip vector components, concatenate into the halo): each connected edge
 * is one call, the host works out the strides (xgcm_b200/padding.py:_pad_face_connections).
 */
XG_API int xg_strided_copy(int dtype, void* dst, const int64_t* dst_strides, const void* src,
                    const int64_t* src_strides, int ndim, const int64_t* shape, int negate,
                    void* stream);

/*
 * North-fold halo of a tripolar grid (xgcm/padding.py:619-684): `width` rows of the field `in`
 * (`shape`, contiguous) mirrored across the fold, written into `out`, which has `in`'s shape except
 * `out_len` along fold_axis:
 *
 *   out[..., row0 + r, ..., k, ...] = (negate ? -1 : 1) * (in * pre)[..., n-1-skip-r, ..., (mirror - k) mod period, ...]
 *
 * for r < width along fold_axis and every k along seam_axis (either order; other dims are copied
 * through).  `pre` (optional) broadcasts against `in` via pre_strides and is read at the mirrored
 * cell, like the halo planes xg_stencil2 takes as already metric-weighted.  The plane of xg_stencil2
 * is out_len = 1, row0 = 0, width = 1; the north rows of a padded array are out_len = n + width,
 * row0 = n.  XG_EINVAL for null pointers, fold_axis == seam_axis, width < 1 or width > n - skip;
 * XG_ENOTIMPL if a mirror partner lies outside the seam dim (an `inner` seam under a center pivot).
 */
XG_API int xg_fold_rows(int dtype, const void* in, void* out, int ndim, const int64_t* shape,
                        int fold_axis, int seam_axis, int64_t out_len, int64_t row0, int width,
                        int skip, int64_t mirror, int64_t period, int negate, const void* pre,
                        const int64_t* pre_strides, void* stream);

/*
 * `count` strided copies of the same rank in ONE launch (all connected edges of a field:
 * padding.py:398-541 loops over faces x axes x sides).  dst[i] / src[i]: per-copy base pointers;
 * shapes, dst_strides, src_strides: count x ndim, row-major; negate: count flags.  XG_ENOTIMPL if
 * a copy does not collapse to 5 dims (callers then fall back to xg_strided_copy).
 */
XG_API int xg_strided_copy_batch(int dtype, int count, void* const* dst, const void* const* src,
                          int ndim, const int64_t* shapes, const int64_t* dst_strides,
                          const int64_t* src_strides, const int* negate, void* stream);

/*
 * Sharded operated axis (SURVEY 8e; reference analogue: map_overlap(depth=1), xgcm/grid_ufunc.py:1057-1133).
 * Every rank holds a contiguous block of the operated axis on its own GPU, rank order = axis order.
 *
 * NCCL is loaded at run time (dlopen); xg_nccl_load(path) names the library explicitly, NULL tries the copy
 * already in the process, then the default soname.  All NCCL failures return XG_ENCCL.
 *   xg_comm_unique_id   rank 0 fills 128 bytes; the host ships them to the other ranks
 *   xg_comm_init        collective over the nranks GPUs (the calling thread's current device)
 *   xg_halo_exchange    one ring step in ONE NCCL group: send_lo (my first plane) goes to rank-1, send_hi (my
 *                       last plane) to rank+1; recv_lo / recv_hi receive the neighbours' last / first plane.
 *                       NULL pointers skip that leg; the ring closes only when `periodic`.
 *   xg_stencil2_sharded xg_stencil2 (lo + hi == 1; periodic / fill / extend) on the local block: boundary
 *                       planes are packed (x pre-metric) by a kernel and exchanged on a side stream WHILE the
 *                       local block is computed; the one or two edge planes are then recomputed from the
 *                       received halos.  pre / post metrics are the LOCAL shards.  workspace: device memory for
 *                       4 planes of outer * inner elements, each rounded up to 256 bytes.
 */
XG_API int xg_nccl_load(const char* path);
XG_API int xg_comm_unique_id(void* id128);
XG_API int xg_comm_init(const void* id128, int nranks, int rank, void** comm);
XG_API int xg_comm_destroy(void* comm);
XG_API int xg_halo_exchange(void* comm, const void* send_lo, const void* send_hi, void* recv_lo,
                     void* recv_hi, size_t bytes, int periodic, void* stream);
XG_API int xg_stencil2_sharded(void* comm, int op, int dtype, const void* in, void* out, int ndim,
                        const int64_t* shape, int axis, int lo, int hi, int bc, double fill_value,
                        const void* pre_metric, const int64_t* pre_strides,
                        const void* post_metric, const int64_t* post_strides, void* workspace,
                        size_t workspace_bytes, void* stream);

/* Deterministic synthetic field: out[i] = U(0,1) keyed by (seed, offset+i);
 * identical bits on host (xg_fill_uniform_host) and device. */
XG_API int xg_fill_uniform(int dtype, void* out, int64_t count, uint64_t seed,
                    uint64_t offset, void* stream);
XG_API int xg_fill_uniform_host(int dtype, void* out, int64_t count, uint64_t seed,
                         uint64_t offset);

/*
 * Host-buffer variant of xg_stencil2: same semantics, HOST pointers.  The field
 * is streamed through the device in slabs of the outermost dimension (one-plane
 * overlap when that is the operated axis) with H2D / kernel / D2H overlapped on three streams.  Host buffers
 * should be page-locked for full PCIe rate (pageable memory is staged).
 * `device` selects the GPU.  Synchronous: returns when `out` is complete.
 */
XG_API int xg_stencil2_host(int op, int dtype, const void* in, void* out, int ndim,
                     const int64_t* shape, int axis, int lo, int hi, int bc,
                     double fill_value, const void* pre_metric,
                     const int64_t* pre_strides, const void* post_metric,
                     const int64_t* post_strides, int device);

/*
 * xg_stencil2_host on the two grid topologies whose halo is not a boundary condition.  Same slab
 * pipeline (workspace, slots, events, slab size), plus a per-slab halo stage on the kernel stream that
 * builds the slab's halo_lo / halo_hi planes before its xg_stencil2 launch.  Dim 0 is cut into slabs and
 * must be a batch dim: not the operated, fold, seam or face dim (XG_EINVAL).  Every argument is
 * checked before any CUDA call.
 *
 * _fold: north fold along `axis` (hi must be 1).  Per slab, one xg_fold_rows launch (width 1; seam_axis,
 * skip, mirror, period, negate as there, `pre_metric` read at the mirrored cell) writes halo_hi; with
 * lo = 1 and bc = XG_BC_PERIODIC it is halo_lo too, any other bc pads the south edge as usual.
 * XG_ENOTIMPL where xg_fold_rows would return it.
 *
 * _connected: face connections.  The halo planes (the field's shape with extent 1 along `axis`) are
 * written by `ncopies` strided copies of rank `copy_ndim` (copy k: side[k] 0 = lo plane, 1 = hi plane;
 * source[k] 0 = the field, 1 = `partner`, the other component of a vector, 2 = the constant fill_value;
 * element offsets into plane and source, then shape, strides and negate as in xg_strided_copy_batch),
 * described once for the WHOLE field: every copy spans dim 0 in full from index 0, with the contiguous
 * dim-0 strides of the plane and of its source (0 for the constant).  The copies must write disjoint
 * cells that cover each padded plane.  `partner` (optional, shape `partner_shape`, same ndim and dim-0
 * extent as the field) is streamed slab by slab beside it.  No pre-metric.
 */
XG_API int xg_stencil2_host_fold(int op, int dtype, const void* in, void* out, int ndim,
                                 const int64_t* shape, int axis, int lo, int hi, int bc,
                                 double fill_value, const void* pre_metric, const int64_t* pre_strides,
                                 const void* post_metric, const int64_t* post_strides, int seam_axis,
                                 int skip, int64_t mirror, int64_t period, int negate, int device);
XG_API int xg_stencil2_host_connected(int op, int dtype, const void* in, const void* partner,
                                      const int64_t* partner_shape, void* out, int ndim,
                                      const int64_t* shape, int axis, int lo, int hi, double fill_value,
                                      const void* post_metric, const int64_t* post_strides, int ncopies,
                                      int copy_ndim, const int* side, const int* source,
                                      const int64_t* dst_offset, const int64_t* src_offset,
                                      const int64_t* shapes, const int64_t* dst_strides,
                                      const int64_t* src_strides, const int* negate, int device);

/*
 * Host-buffer twins of xg_stencil_pair: same semantics, HOST pointers, `device` instead of a stream;
 * synchronous.  The slab pipeline of xg_stencil2_host: `a` is cut into slabs along dim 0, `b` streams
 * beside it slab by slab, pre_a / pre_b / post are uploaded whole.  Dim 0 must be a batch dim: not axis_b
 * (nor the innermost dim, nor the seam dim of _fold) (XG_EINVAL).  Every argument is checked before any
 * CUDA call.
 *
 * _fold: the term along axis_b crosses a north fold (hi_b must be 1).  Per slab, one xg_fold_rows launch
 * of b * pre_b (width 1; seam_axis, skip, mirror, period, negate as there) writes halo_hi_b of
 * xg_stencil_pair_halo; with lo_b = 1 and bc_b = XG_BC_PERIODIC it is halo_lo_b too.  XG_ENOTIMPL where
 * xg_fold_rows would return it.
 */
XG_API int xg_stencil_pair_host(int dtype, const void* a, const void* b, void* out, int ndim,
                                const int64_t* shape, int op_a, int lo_a, int hi_a, int bc_a, double fill_a,
                                const void* pre_a, const int64_t* pre_a_strides, int axis_b, int op_b,
                                int lo_b, int hi_b, int bc_b, double fill_b, const void* pre_b,
                                const int64_t* pre_b_strides, int subtract, const void* post,
                                const int64_t* post_strides, int device);
XG_API int xg_stencil_pair_host_fold(int dtype, const void* a, const void* b, void* out, int ndim,
                                     const int64_t* shape, int op_a, int lo_a, int hi_a, int bc_a,
                                     double fill_a, const void* pre_a, const int64_t* pre_a_strides,
                                     int axis_b, int op_b, int lo_b, int hi_b, int bc_b, double fill_b,
                                     const void* pre_b, const int64_t* pre_b_strides, int subtract,
                                     const void* post, const int64_t* post_strides, int seam_axis, int skip,
                                     int64_t mirror, int64_t period, int negate, int device);

/* Device bytes the one workspace of the *_host entry points holds on `device` (slot buffers, halo planes,
 * scratch, whole-call operands such as metrics); 0 before the first call or after xg_host_workspace_release.
 * Same number as xg_host_pipe_workspace_bytes.  `device` is a device index: a group handle gives XG_EINVAL. */
XG_API int xg_host_workspace_bytes(int device, int64_t* bytes);

/*
 * Host device groups: one *_host call spread over several GPUs.  xg_host_group registers the `n` device indices
 * `devices` and writes a handle to *group, XG_HOST_GROUP_BASE + k, which no device index reaches; the same member
 * list gives the same handle back.  A member may appear more than once: its blocks then take turns on that
 * device's workspace.  Up to XG_HOST_GROUP_MAX groups of 1 .. XG_HOST_GROUP_MAX_MEMBERS members; XG_EINVAL past
 * either cap, for a null pointer or a negative index (before any CUDA call), and for an index at or past
 * cudaGetDeviceCount.  Groups live for the process.
 *
 * Every *_host entry point that streams slabs (xg_stencil2_host and its _multi / _fold / _connected variants,
 * xg_stencil_multi_host, xg_stencil_pair_host[_fold], xg_cumscan_host, xg_wreduce_host[_multi] and both
 * xg_vinterp_*_host) takes a handle in its `device` argument.  The result rows along the call's slab dim are cut
 * into contiguous near-equal blocks, one per member (fewer when there are fewer rows), and each member streams
 * its block on its own host thread through its own workspace, with the whole-call operands uploaded once per
 * member.  Results are bit for bit those of a single device: the slabs run the same launches on the same rows.
 * The call returns when every member has finished, with the first failing member's status (in member order) and
 * message; the calling thread's xg_last_launch() is the first member's.  xg_wreduce_host_multi with every dim
 * of extent > 1 reduced keeps its partials along the slab dim on one device and runs on the first member alone.
 * An unknown handle gives XG_EINVAL before any CUDA call.
 */
#define XG_HOST_GROUP_BASE 1048576
#define XG_HOST_GROUP_MAX 64
#define XG_HOST_GROUP_MAX_MEMBERS 64
XG_API int xg_host_group(int n, const int* devices, int* group);

/*
 * One HOST field up, `nout` results down: result k = xg_stencil2(op[k], axis[k], lo[k], hi[k], bc[k],
 * fill_value[k]) of the same input (no metrics), each into its own HOST buffer out[k].  The field crosses
 * PCIe once instead of once per result (the reference re-reads it per call, xgcm/grid.py:796-832).
 * Slabs are cut along dim 0; a result operated along dim 0 must keep that extent (lo + hi == 1) and may
 * not use XG_BC_EXTRAPOLATE (XG_ENOTIMPL otherwise: use xg_stencil2_host for that result).  nout <= 8.
 */
XG_API int xg_stencil2_host_multi(int nout, const int* op, int dtype, const void* in, void* const* out,
                           int ndim, const int64_t* shape, const int* axis, const int* lo,
                           const int* hi, const int* bc, const double* fill_value, int device);

/*
 * Host-buffer twins of xg_cumscan / xg_wreduce / xg_vinterp_linear (same semantics, HOST pointers, `device`
 * instead of a stream; synchronous).  The field is streamed in slabs of a NON-operated dimension (the first
 * one for cumscan / wreduce; see xg_vinterp_conservative_host for the transform twins), with strided 2-D
 * copies when that is not dim 0, so every line along the operated axis stays whole: no halo between slabs,
 * summation order untouched.  Metric / weight / target operands are uploaded whole; a dense theta field
 * streams beside the field.  Replaces the host side of xgcm/grid.py:1316 (cumsum), :1598-1605 (integrate), :1680-1685
 * (average) and xgcm/transform.py:233-249 for numpy-backed fields.
 */
XG_API int xg_cumscan_host(int dtype, const void* in, void* out, int ndim, const int64_t* shape, int axis,
                    int reverse, int trim, int pad_lo, int pad_hi, int bc, double fill_value,
                    const void* pre_metric, const int64_t* pre_strides, const void* post_metric,
                    const int64_t* post_strides, int skipna, int device);
XG_API int xg_wreduce_host(int dtype, const void* in, const void* weight, const int64_t* w_strides,
                    void* out, int ndim, const int64_t* shape, int axis, int mode, int skipna,
                    int device);
XG_API int xg_vinterp_linear_host(int dtype, const void* phi, const void* theta,
                           const int64_t* theta_strides, const void* target,
                           const int64_t* target_strides, int64_t m, void* out, int ndim,
                           const int64_t* shape, int axis, int mask_edges, int bypass_checks,
                           int logarithmic, int device);

/*
 * Host-buffer twin of xg_vinterp_conservative (same semantics, HOST pointers, `device` instead of a stream;
 * synchronous).  Replaces the host side of xgcm/transform.py:157-198 for numpy-backed fields.  The two transform
 * twins (this and xg_vinterp_linear_host) cut slabs along the outermost non-operated dim of extent > 1 one index of
 * which (phi, theta, theta-bounds scratch and result bytes together) fits the slab budget, else the innermost such
 * dim; a dense theta field streams in the same slabs as phi, a broadcast one is uploaded whole.  theta_at_centers:
 * theta holds n cell-centre values along `axis` (not n + 1 bounds); the bounds are made on the device by the
 * center -> outer interp with extend padding, i.e. grid.interp(theta, axis, padding="extend") (transform.py:289-294).
 * A zero-length axis gives all-NaN bins.  Every argument is checked before any CUDA call (XG_EINVAL).
 */
XG_API int xg_vinterp_conservative_host(int dtype, const void* phi, const void* theta,
                                 const int64_t* theta_strides, int theta_at_centers,
                                 const void* target_bins, int64_t m, int flip_out, void* out, int ndim,
                                 const int64_t* shape, int axis, int device);

/*
 * Host-buffer twin of xg_stencil_multi (same semantics and argument checks, HOST pointers, `device` instead of a
 * stream; synchronous): one xg_stencil_multi launch per slab.  Slabs are cut along the outermost dim of extent > 1
 * that is not operated, so every operated line is whole in a slab.  When every dim of extent > 1 is operated, the
 * outermost of them is cut: each slab reads the row next to it, an inner slab edge has no boundary condition and
 * the field's own ends keep the call's; an outer / inner shift or a periodic boundary along that dim gives
 * XG_ENOTIMPL (use xg_stencil_multi).  Every argument is checked before any CUDA call.
 */
XG_API int xg_stencil_multi_host(int dtype, const void* in, void* out, int ndim, const int64_t* shape, int naxes,
                                 const int* axes, const int* ops, const int* lo, const int* hi, const int* bc,
                                 const double* fill_value, int device);

/*
 * Weighted sum (XG_REDUCE_SUM) or mean (XG_REDUCE_MEAN) of a HOST field over the `naxes` >= 2 distinct dims
 * `axes`, bit for bit the device sequence of Grid.integrate / average: one xg_wreduce per dim, innermost first,
 * `weight` (optional, broadcast via w_strides) in the first only; a mean reduces the sum and the valid weights
 * (XG_REDUCE_WVALID, then plain sums with skipna = 0) side by side and divides once (XG_BIN_DIVNZ).  out: shape
 * without `axes` (one value when every dim is reduced).  Slabs are cut along the outermost dim of extent > 1 that is
 * not reduced; with none, along the outermost dim of extent > 1, whose per-slab partials stay on the device for
 * the launches along it, run once.  A weight that spans the slab dim (a dense array of its own extents) streams
 * beside the field; otherwise it is uploaded whole.  XG_ENOTIMPL for an empty reduced dim, or when no reduced dim
 * of extent > 1 lies inside the slab dim (use xg_wreduce_host).  Every argument is checked before any CUDA call.
 */
XG_API int xg_wreduce_host_multi(int dtype, const void* in, const void* weight, const int64_t* w_strides,
                                 void* out, int ndim, const int64_t* shape, int naxes, const int* axes, int mode,
                                 int skipna, int device);

/* Device bytes the one workspace of the *_host entry points holds on `device`: the same number as
 * xg_host_workspace_bytes, kept for callers of the multi, scan, reduce and transform twins. */
XG_API int xg_host_pipe_workspace_bytes(int device, int64_t* bytes);

/* Free the cached device buffers of the *_host entry points (waiting for a call in progress on a device to
 * finish first); their streams and events are kept for later calls. */
XG_API int xg_host_workspace_release(void);

#ifdef __cplusplus
}
#endif
#endif /* XGCM_B200_H */
