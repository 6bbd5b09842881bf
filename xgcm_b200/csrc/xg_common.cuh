// Shared device/host helpers for the xgcm_b200 kernels (sm_90a).
//
// Everything here is plain LD/ST work: the path is HBM-bound (<= 0.25 flop/B),
// so there are no tensor-core instructions by design.  Arithmetic must round
// exactly like numpy does one ufunc at a time, therefore the library is built
// with --fmad=false and IEEE division (no fast-math).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>

#include "xgcm_b200.h"

#define XG_MAXG 4  // max collapsed dim groups when decomposing a flat index
// SM count of an H100 SXM: caps the grids of grid-stride kernels, and the default where the
// persistent kernels query cudaDevAttrMultiProcessorCount
#define XG_SMS 132

// ---------------------------------------------------------------------------
// error plumbing (thread-local message, never abort)
// ---------------------------------------------------------------------------
void xg_set_error(const std::string& msg);
int xg_fail(int code, const std::string& msg);
int xg_check_launch(const char* what);
// the calling thread's xg_last_launch() label (a string literal), e.g. as a worker thread left it
void xg_set_last_launch(const char* what);

// ---------------------------------------------------------------------------
// broadcast operand descriptor
// ---------------------------------------------------------------------------
// Division by a launch constant d >= 1 of a dividend below 2^31 as multiply-high + shift
// (Granlund-Montgomery: l = ceil(log2 d), mul = ceil(2^(31+l) / d), q = umulhi(x, mul) >> (l-1);
// exact for every x < 2^31).  A generic 32-bit division is ~20 SASS instructions and the fused-metric
// kernels need up to nine per thread; this form is two.
struct XgFastDiv {
  uint32_t d;
  uint32_t mul;  // 0: d == 1 (quotient = dividend)
  uint32_t sh;
};

static inline XgFastDiv xg_fastdiv_make(int64_t d) {
  XgFastDiv f;
  f.d = (uint32_t)d;
  f.mul = 0;
  f.sh = 0;
  if (d >= 2 && d < (1ll << 31)) {
    int l = 0;
    while ((1ll << l) < d) ++l;
    f.mul = (uint32_t)((((uint64_t)1 << (31 + l)) + (uint64_t)d - 1) / (uint64_t)d);
    f.sh = (uint32_t)(l - 1);
  }
  return f;
}

__host__ __device__ __forceinline__ uint32_t xg_fastdiv_q(uint32_t x, const XgFastDiv& f) {
#ifdef __CUDA_ARCH__
  return f.mul ? (__umulhi(x, f.mul) >> f.sh) : x;
#else
  return f.mul ? (uint32_t)(((uint64_t)x * f.mul) >> 32) >> f.sh : x;
#endif
}

struct XgGroups {
  int n;
  int small;  // every size and the total extent fit in 31 bits: 32-bit index math
  int64_t size[XG_MAXG];
  int64_t stride[XG_MAXG];
  XgFastDiv fd[XG_MAXG];  // of size[k]; valid when `small`
};

enum { XG_IM_BCAST = 0, XG_IM_CONTIG = 1, XG_IM_GENERIC = 2 };

// A metric (or weight / theta) operand broadcast against a field collapsed to
// (outer, n, inner).
struct XgOperand {
  const void* ptr;      // nullptr = absent
  XgGroups outer;       // flat outer index -> element offset
  int64_t axis_stride;  // element stride along the operated axis
  XgGroups inner;       // flat inner index -> element offset
  int inner_mode;       // XG_IM_*
  int vec_ok;           // CONTIG and every offset is a multiple of the vector width
  int wide_span;        // GENERIC and the inner offsets span >= 2^31 elements: two elements of one vector
                        // may lie further apart than XgOperandView's 32-bit deltas reach, so the
                        // launchers take their VEC = 1 instance (no deltas) for such an operand
};

// an operand the VEC > 1 instances of the XgOperandView kernels can take (absent operands included)
static inline bool xg_vec_view_ok(const XgOperand& m) { return !m.wide_span; }

struct XgView {
  int64_t outer, n, inner;
};

// host: collapse (shape, axis) and an operand's per-dim strides.
int xg_collapse_view(int ndim, const int64_t* shape, int axis, XgView* v);
int xg_make_operand(const void* ptr, const int64_t* strides, int ndim,
                    const int64_t* shape, int axis, int vec, size_t elem_size,
                    XgOperand* op, const char* what);
// host: every argument check of xg_stencil_multi[_weighted][_host] (error text prefixed with `who`); the metric
// arrays may be null
int xg_stencil_multi_check(const char* who, int dtype, const void* in, const void* out, int ndim,
                           const int64_t* shape, int naxes, const int* axes, const int* ops, const int* lo,
                           const int* hi, const int* bc, const double* fill_value, const void* const* pre,
                           const int64_t* pre_strides, const void* const* post, const int64_t* post_strides);

__host__ __device__ __forceinline__ int64_t xg_groups_offset(const XgGroups& g,
                                                             int64_t flat) {
  int64_t off = 0;
  if (g.n == 0) return 0;
  if (g.small) {  // 32-bit divisions are ~5x cheaper than 64-bit ones on the SM
    uint32_t f = (uint32_t)flat;
#pragma unroll
    for (int k = XG_MAXG - 1; k >= 0; --k) {
      if (k < g.n) {
        const uint32_t q = xg_fastdiv_q(f, g.fd[k]);
        off += (int64_t)(f - q * g.fd[k].d) * g.stride[k];
        f = q;
      }
    }
    return off;
  }
#pragma unroll
  for (int k = XG_MAXG - 1; k >= 0; --k) {
    if (k < g.n) {
      int64_t q = flat / g.size[k];
      off += (flat - q * g.size[k]) * g.stride[k];
      flat = q;
    }
  }
  return off;
}

// flat -> (q, r) with a 32-bit fast path (warp-unit decomposition)
__device__ __forceinline__ void xg_divmod(int64_t x, int64_t d, bool small, int64_t& q, int64_t& r) {
  if (small) {
    const uint32_t qq = (uint32_t)x / (uint32_t)d;
    q = qq;
    r = (uint32_t)x - qq * (uint32_t)d;
  } else {
    q = x / d;
    r = x - q * d;
  }
}
// the same with the divisor's multiply-high form prepared on the host (`small` implies x < 2^31)
__device__ __forceinline__ void xg_divmod(int64_t x, int64_t d, const XgFastDiv& f, bool small, int64_t& q,
                                          int64_t& r) {
  if (small) {
    const uint32_t qq = xg_fastdiv_q((uint32_t)x, f);
    q = qq;
    r = (uint32_t)x - qq * f.d;
  } else {
    q = x / d;
    r = x - q * d;
  }
}

// ---------------------------------------------------------------------------
// vector types: 16-byte accesses for both dtypes
// ---------------------------------------------------------------------------
template <typename T, int VEC>
struct XgVec;
template <>
struct XgVec<float, 4> {
  typedef float4 type;
};
template <>
struct XgVec<double, 2> {
  typedef double2 type;
};
template <>
struct XgVec<float, 1> {
  typedef float type;
};
template <>
struct XgVec<double, 1> {
  typedef double type;
};

template <typename T>
struct XgVecWidth;
template <>
struct XgVecWidth<float> {
  static const int value = 4;
};
template <>
struct XgVecWidth<double> {
  static const int value = 2;
};

template <typename T, int VEC>
struct XgPack {
  T v[VEC];
};

// streaming (evict-first) global accesses: every field element is touched once.
template <typename T, int VEC>
__device__ __forceinline__ XgPack<T, VEC> xg_ld_stream(const T* p) {
  XgPack<T, VEC> r;
  if constexpr (VEC == 1) {
    r.v[0] = __ldcs(p);
  } else {
    typedef typename XgVec<T, VEC>::type V;
    V t = __ldcs(reinterpret_cast<const V*>(p));
    const T* tp = reinterpret_cast<const T*>(&t);
#pragma unroll
    for (int k = 0; k < VEC; ++k) r.v[k] = tp[k];
  }
  return r;
}

// cached (read-only path) accesses: metrics and halo rows are re-used.
template <typename T, int VEC>
__device__ __forceinline__ XgPack<T, VEC> xg_ld_cached(const T* p) {
  XgPack<T, VEC> r;
  if constexpr (VEC == 1) {
    r.v[0] = __ldg(p);
  } else {
    typedef typename XgVec<T, VEC>::type V;
    V t = __ldg(reinterpret_cast<const V*>(p));
    const T* tp = reinterpret_cast<const T*>(&t);
#pragma unroll
    for (int k = 0; k < VEC; ++k) r.v[k] = tp[k];
  }
  return r;
}

template <typename T, int VEC>
__device__ __forceinline__ void xg_st_stream(T* p, const XgPack<T, VEC>& r) {
  if constexpr (VEC == 1) {
    __stcs(p, r.v[0]);
  } else {
    typedef typename XgVec<T, VEC>::type V;
    V t;
    T* tp = reinterpret_cast<T*>(&t);
#pragma unroll
    for (int k = 0; k < VEC; ++k) tp[k] = r.v[k];
    __stcs(reinterpret_cast<V*>(p), t);
  }
}

// Per-thread view of a broadcast operand for the VEC elements starting at flat inner index i:
// computed ONCE per thread (i is fixed while a thread marches along the axis), so the per-row
// cost of a fused metric is one (vector) load and VEC multiplies / divides.  Kept small on
// purpose (a pointer + VEC-1 32-bit deltas): register pressure decides the occupancy of the
// fused kernels.
template <typename T, int VEC>
struct XgOperandView {
  const T* p0;       // operand pointer + outer offset + inner offset of element 0
  int d[VEC];        // element k sits at p0[d[k]] (d[0] = 0); generic mode only
  int mode;          // XG_IM_* ; CONTIG with `vec` -> one 16-byte load
  bool vec;
};

template <typename T, int VEC>
__device__ __forceinline__ XgOperandView<T, VEC> xg_operand_view(const XgOperand& m, int64_t outer_off,
                                                                 int64_t i) {
  XgOperandView<T, VEC> r;
  const T* p = reinterpret_cast<const T*>(m.ptr) + outer_off;
  r.mode = m.inner_mode;
  r.vec = false;
#pragma unroll
  for (int k = 0; k < VEC; ++k) r.d[k] = 0;
  if (m.inner_mode == XG_IM_BCAST) {
    r.p0 = p;
  } else if (m.inner_mode == XG_IM_CONTIG) {
    r.p0 = p + i;
#pragma unroll
    for (int k = 0; k < VEC; ++k) r.d[k] = k;
    r.vec = VEC > 1 && m.vec_ok;
  } else {
    const int64_t o0 = xg_groups_offset(m.inner, i);
    r.p0 = p + o0;
#pragma unroll
    for (int k = 1; k < VEC; ++k) r.d[k] = (int)(xg_groups_offset(m.inner, i + k) - o0);
  }
  return r;
}

// the operand's VEC values `row_off` elements further along the operated axis
template <typename T, int VEC>
__device__ __forceinline__ XgPack<T, VEC> xg_ld_view(const XgOperandView<T, VEC>& v, int64_t row_off) {
  const T* p = v.p0 + row_off;
  XgPack<T, VEC> r;
  if (v.mode == XG_IM_BCAST) {
    const T s = __ldg(p);
#pragma unroll
    for (int k = 0; k < VEC; ++k) r.v[k] = s;
  } else if (v.vec) {
    r = xg_ld_cached<T, VEC>(p);
  } else {
#pragma unroll
    for (int k = 0; k < VEC; ++k) r.v[k] = __ldg(p + v.d[k]);
  }
  return r;
}

// ---------------------------------------------------------------------------
// the four pairwise operators, rounding exactly like numpy
// ---------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ bool xg_isnan(T x) {
  return x != x;
}

// a = P[j] (lower neighbour), b = P[j+1] (upper neighbour)
template <typename T, int OP>
__device__ __forceinline__ T xg_apply_op(T a, T b) {
  if constexpr (OP == XG_OP_DIFF) {
    return b - a;  // gridops.py:24  a[...,1:] - a[...,:-1]
  } else if constexpr (OP == XG_OP_INTERP) {
    return (a + b) * T(0.5);  // gridops.py:77 (a[:-1]+a[1:])/2.0 ; x*0.5 == x/2 in IEEE
  } else if constexpr (OP == XG_OP_MIN) {
    // gridops.py:123-126 np.min over the stacked pair: NaN propagates
    return (a < b || xg_isnan(a)) ? a : b;
  } else {
    return (a > b || xg_isnan(a)) ? a : b;
  }
}

// ---------------------------------------------------------------------------
// division by a divisor shared between several cells (same metric value for every level)
// ---------------------------------------------------------------------------
// Correctly rounded a / b from r = RN(1/b) with five fp64 operations instead of the ~30 of the
// generic division (Markstein's FMA-based sequence: q0 = RN(a r) is within 2 ulp, the first
// correction makes it faithful, and for a faithful q with r within half an ulp of 1/b the second
// correction q + RN(a - b q) r rounds to exactly RN(a / b)).  Only valid when no intermediate
// can leave the normal range; the caller guards the exponents of a and b and falls back to `/`.
__device__ __forceinline__ double xg_div_with_recip(double a, double b, double r) {
  const double q0 = a * r;
  const double e0 = fma(-b, q0, a);
  const double q1 = fma(e0, r, q0);
  const double e1 = fma(-b, q1, a);
  return fma(e1, r, q1);
}
__device__ __forceinline__ bool xg_exponent_safe(double v) {
  // |v| in [2^-400, 2^400]: biased exponent in [623, 1423]; false for 0, subnormals, NaN, inf
  const unsigned e = ((unsigned)__double2hiint(v) >> 20) & 0x7ffu;
  return (e - 623u) <= 800u;
}

// x / b for many x and one b, bit-identical to the IEEE division.
//   float : RN32(RN64(x * RN64(1 / b))).  The fp64 product is within 2^-52 (relative) of x / b,
//           while a quotient of two 24-bit significands is never closer than 2^-49 to a rounding
//           boundary of binary32 (midpoints have 25-bit significands; subnormal and overflow
//           boundaries included), so the second rounding lands where the direct one would.
//           Zeros, infinities and NaNs follow from IEEE arithmetic on the reciprocal; no guard.
//   double: Markstein's sequence above behind the exponent guards, else the plain division.
template <typename T>
struct XgSharedDivisor;
template <>
struct XgSharedDivisor<float> {
  double r;
  __device__ __forceinline__ void set(float b) { r = __drcp_rn((double)b); }
  __device__ __forceinline__ float div(float x) const { return (float)((double)x * r); }
};
template <>
struct XgSharedDivisor<double> {
  double b, r;  // r == 0: no fast path for this divisor
  __device__ __forceinline__ void set(double b_) {
    b = b_;
    r = xg_exponent_safe(b_) ? 1.0 / b_ : 0.0;
  }
  __device__ __forceinline__ double div(double x) const {
    return (r != 0.0 && xg_exponent_safe(x)) ? xg_div_with_recip(x, b, r) : x / b;
  }
};

__host__ __device__ static inline int64_t xg_ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
