// xg_stencil_multi — 2 or 3 single-axis stencils fused into ONE pass over HBM.
//
// `Grid.interp(da, ['X', 'Y'])` (and diff / min / max over several axes) is, in the reference,
// one full pad + ufunc pass per axis (xgcm/grid.py:798-832; its own TODO notes the waste).  Here
// the chain  op_K(pad_K( ... op_1(pad_1(a)) ... ))  is evaluated per output cell straight from the
// input: 2^K neighbour loads (absorbed by L1 / L2: DRAM sees one read and one write per cell),
// every intermediate rounded to the field dtype exactly where the sequential passes would round,
// each axis with its own halo rule applied to ITS intermediate (fill is a constant of that level,
// periodic / extend re-index the source).  Bit-identical to K consecutive xg_stencil2 calls at
// 1/K of their traffic.
//
// Work split: a block owns one output row along the innermost dim; threads take 16-byte vectors
// of it.  The recursion is resolved at compile time (K ops, position LAST of the op acting on the
// innermost dim, or -1): row ops combine two windows of W values; the innermost op consumes a
// window of W + 1 consecutive source positions (one aligned vector + one neighbour element).
//
// Roofline: HBM, 2 * sizeof(T) bytes per output cell.
//
// Weighted chains (xg_stencil_multi_weighted, Grid.<op>(da, axes, metric_weighted=...)): stage m may carry a
// pre-metric on its input and a post-metric on its output, u_{m+1} = op_m(pad_m(u_m * pre_m)) / post_m, each
// product and quotient rounded to the field dtype where the per-axis launches round it (post_m and pre_{m+1} are
// applied, not cancelled).  A metric is read at the coordinates of the intermediate it weights: output coordinates
// of the axes applied before the stage, source positions (wrapped / clamped like the field) of the others, so a
// periodic / extend halo cell is the weighted value of its source and a fill halo cell is the bare fill.  The
// weighted body is selected at run time inside the same instances (MultiArgs::met), so the metric-free body is
// unchanged; its blocks walk every row group of one march segment before the next segment, so a metric that
// broadcasts over the non-operated dims (2-D areas against 75 levels) is read from DRAM about once and from L2
// for the other levels.
#include <stdlib.h>

#include "xg_common.cuh"
#include "xg_stencil_tile.cuh"

namespace {

constexpr int kMaxAx = 3;
constexpr int kMaxGroups = 2 * kMaxAx;  // row groups (everything but the innermost group)
constexpr int kMetU = 2;  // march steps in flight in the weighted body (2 measured faster than 4)

template <typename T>
struct AxisOp {
  int op, lo, hi, bc;
  T fill;
  int64_t n;          // input (and intermediate) length along this axis
  int64_t in_stride;  // element stride of this axis in the INPUT (1 for the innermost dim)
};

// pre- or post-metric of one stage: element strides along the dim of each applied axis and the innermost dim;
// the row-group strides live in MultiArgs::row_met.  p == nullptr: the stage has none.
template <typename T>
struct StageMet {
  const T* p;
  int64_t ax[kMaxAx];
  int64_t x;
  int vec;  // x stride 1, 16-byte aligned, every other stride a multiple of the vector width
};

template <typename T>
struct MultiArgs {
  const T* in;
  T* out;
  AxisOp<T> ax[kMaxAx];  // in application order
  int met;                                  // weighted chain: the metric body of k_stencil_multi
  StageMet<T> pre[kMaxAx], post[kMaxAx];
  int64_t row_met[kMaxGroups][2 * kMaxAx];  // stride of each row group in pre[0..K), post[0..K)
  int64_t nrows;                            // product of row_size
  int nrow_groups;
  int64_t row_size[kMaxGroups];        // extent in the OUTPUT, outermost first
  int64_t row_in_stride[kMaxGroups];   // input element stride (non-operated groups)
  int64_t row_out_stride[kMaxGroups];  // output element stride
  int row_axis[kMaxGroups];            // application index of the operated axis, or -1
  int64_t last_n_out;                  // output extent of the innermost group
  // the march axis (last applied row-axis op): not part of the row groups
  int64_t march_n_out, march_out_stride;
  int J;
  int64_t nseg;
};

template <typename T>
__device__ __forceinline__ T apply_rt(int op, T a, T b) {
  switch (op) {
    case XG_OP_DIFF: return xg_apply_op<T, XG_OP_DIFF>(a, b);
    case XG_OP_INTERP: return xg_apply_op<T, XG_OP_INTERP>(a, b);
    case XG_OP_MIN: return xg_apply_op<T, XG_OP_MIN>(a, b);
    default: return xg_apply_op<T, XG_OP_MAX>(a, b);
  }
}

// source index of padded position idx along an axis; false when the halo is the fill constant
template <typename T>
__device__ __forceinline__ bool resolve(const AxisOp<T>& a, int64_t idx, int64_t& s) {
  s = idx - a.lo;
  if (s < 0) {
    if (a.bc == XG_BC_FILL) { s = 0; return false; }
    s = (a.bc == XG_BC_PERIODIC) ? s + a.n : 0;
  } else if (s >= a.n) {
    if (a.bc == XG_BC_FILL) { s = a.n - 1; return false; }
    s = (a.bc == XG_BC_PERIODIC) ? s - a.n : a.n - 1;
  }
  return true;
}

template <typename T, int W>
struct Win {
  T v[W];
};

// metric offsets of every stage's operands at the current position of the recursion: the row groups, the
// applied axes other than the stage's own and the innermost dim
struct MetOff {
  int64_t pre[kMaxAx], post[kMaxAx];
};

// the source coordinate s of applied axis m, added to the operands of the stages below m (their input and output
// both hold axis m at its source position)
template <typename T, int m>
__device__ __forceinline__ MetOff met_below(const MultiArgs<T>& a, MetOff mo, int64_t s) {
#pragma unroll
  for (int i = 0; i < m; ++i) {
    mo.pre[i] += s * a.pre[i].ax[m];
    mo.post[i] += s * a.post[i].ax[m];
  }
  return mo;
}

// w.v[q] *= (MUL) or /= the metric at innermost coordinate x + q of the intermediate after k ops: while the
// innermost op is still to come (LAST >= k) that coordinate may be -1 or n, read where the halo reads the field.
// A window of VEC values starts at a multiple of VEC; one of VEC + 1 is such a vector and one neighbour (as in
// load_window), so a metric laid out for vectors (StageMet::vec) is read with one 16-byte load (+ one element); a
// metric constant along x with one load.
template <typename T, int VEC, int LAST, int k, int W, bool MUL>
__device__ __forceinline__ void met_apply(const MultiArgs<T>& a, const StageMet<T>& m, int64_t off, int64_t x,
                                          Win<T, W>& w) {
  if (!m.p) return;
  auto wrap = [&](int64_t pos) -> int64_t {
    if constexpr (LAST >= 0 && LAST >= k) {
      const AxisOp<T>& ax = a.ax[LAST];
      if (pos < 0) pos = (ax.bc == XG_BC_PERIODIC) ? pos + ax.n : 0;
      else if (pos >= ax.n) pos = (ax.bc == XG_BC_PERIODIC) ? pos - ax.n : ax.n - 1;
    }
    return pos;
  };
  auto use = [&](int q, T v) { w.v[q] = MUL ? w.v[q] * v : w.v[q] / v; };
  const T* p = m.p + off;
  if (m.x == 0) {
    const T v = __ldg(p);
#pragma unroll
    for (int q = 0; q < W; ++q) use(q, v);
    return;
  }
  if constexpr (VEC > 1 && (W == VEC || W == VEC + 1)) {
    if (m.vec) {
      if constexpr (W == VEC) {
        const XgPack<T, VEC> pk = xg_ld_cached<T, VEC>(p + x);
#pragma unroll
        for (int q = 0; q < VEC; ++q) use(q, pk.v[q]);
      } else {
        const bool lead = (x & (VEC - 1)) != 0;  // the neighbour comes first
        const XgPack<T, VEC> pk = xg_ld_cached<T, VEC>(p + (lead ? x + 1 : x));
        const T extra = __ldg(p + wrap(lead ? x : x + VEC));
#pragma unroll
        for (int q = 0; q <= VEC; ++q) {
          const T from_lead = (q == 0) ? extra : pk.v[q > 0 ? q - 1 : 0];
          const T from_tail = (q < VEC) ? pk.v[q < VEC ? q : 0] : extra;
          use(q, lead ? from_lead : from_tail);
        }
      }
      return;
    }
  }
#pragma unroll
  for (int q = 0; q < W; ++q) use(q, __ldg(p + wrap(x + q) * m.x));
}

// W consecutive input elements along the innermost dim starting at source position xs (which may
// be -1, and xs + W - 1 may be n, only when the innermost dim is operated: those ends follow the
// halo rule of that op; a fill halo is patched by the caller, here it just reads a valid cell).
template <typename T, int VEC, int W, int LAST>
__device__ __forceinline__ Win<T, W> load_window(const MultiArgs<T>& a, int64_t off, int64_t xs) {
  Win<T, W> r;
  const T* p = a.in + off;
  if constexpr (LAST < 0) {
    static_assert(W == VEC, "window == vector when the innermost dim is not operated");
    XgPack<T, VEC> pk = xg_ld_cached<T, VEC>(p + xs);
#pragma unroll
    for (int q = 0; q < VEC; ++q) r.v[q] = pk.v[q];
  } else {
    const AxisOp<T>& ax = a.ax[LAST];
    auto scalar_at = [&](int64_t pos) -> T {
      if (pos < 0) pos = (ax.bc == XG_BC_PERIODIC) ? pos + ax.n : 0;
      else if (pos >= ax.n) pos = (ax.bc == XG_BC_PERIODIC) ? pos - ax.n : ax.n - 1;
      return __ldg(p + pos);
    };
    if constexpr (VEC > 1 && W == VEC + 1) {
      // exactly one aligned vector plus one neighbour: xs = x0 - lo with x0 a multiple of VEC
      const bool lead = (xs & (VEC - 1)) != 0;  // lo == 1: the neighbour comes first
      const int64_t xv = lead ? xs + 1 : xs;
      XgPack<T, VEC> pk = xg_ld_cached<T, VEC>(p + xv);
      const T extra = scalar_at(lead ? xs : xs + VEC);
      // static indices only (a runtime-indexed window would live in local memory)
#pragma unroll
      for (int q = 0; q <= VEC; ++q) {
        const T from_lead = (q == 0) ? extra : pk.v[q > 0 ? q - 1 : 0];
        const T from_tail = (q < VEC) ? pk.v[q < VEC ? q : 0] : extra;
        r.v[q] = lead ? from_lead : from_tail;
      }
    } else {
#pragma unroll
      for (int q = 0; q < W; ++q) r.v[q] = scalar_at(xs + q);
    }
  }
  return r;
}

// Window of W values of the intermediate after the first k ops, at row coordinates j (axes < k
// in their output space; axes >= k already folded into `off`), innermost coordinate x.  MET: the stages' metrics
// apply, at offsets `mo` (MetOff).
template <typename T, int VEC, int K, int LAST, int OP, bool MET>
struct Eval {
  template <int k, int W>
  static __device__ __forceinline__ Win<T, W> run(const MultiArgs<T>& a, const int64_t* j, int64_t off,
                                                   int64_t x, const MetOff& mo) {
    if constexpr (k == 0) {
      return load_window<T, VEC, W, LAST>(a, off, x);
    } else {
      constexpr int m = k - 1;  // the op applied at this level
      const AxisOp<T>& ax = a.ax[m];
      Win<T, W> r;
      if constexpr (m == LAST) {
        // innermost op: padded positions x .. x+W  <-  sources x-lo .. x-lo+W
        const int64_t xs = x - ax.lo;
        Win<T, W + 1> w = run<k - 1, W + 1>(a, j, off, xs, mo);
        if constexpr (MET) met_apply<T, VEC, LAST, m, W + 1, true>(a, a.pre[m], mo.pre[m], xs, w);
        if (ax.bc == XG_BC_FILL) {  // the ends of the window may be halo cells of THIS level
          if (xs < 0) w.v[0] = ax.fill;
          if (xs + W >= ax.n) w.v[W] = ax.fill;
        }
#pragma unroll
        for (int q = 0; q < W; ++q) r.v[q] = xg_apply_op<T, OP>(w.v[q], w.v[q + 1]);
        if constexpr (MET) met_apply<T, VEC, LAST, k, W, false>(a, a.post[m], mo.post[m], x, r);
      } else {
        int64_t s0, s1;
        const bool ok0 = resolve(ax, j[m], s0);  // block-uniform: j is this block's row
        const bool ok1 = resolve(ax, j[m] + 1, s1);
        // branch-free: a fill halo still reads a (clamped, valid) row and is replaced afterwards,
        // so every load of the recursion can be issued before the first value is consumed
        Win<T, W> lo_v, hi_v;
        if constexpr (MET) {
          lo_v = run<k - 1, W>(a, j, off + s0 * ax.in_stride, x, met_below<T, m>(a, mo, s0));
          hi_v = run<k - 1, W>(a, j, off + s1 * ax.in_stride, x, met_below<T, m>(a, mo, s1));
          met_apply<T, VEC, LAST, m, W, true>(a, a.pre[m], mo.pre[m] + s0 * a.pre[m].ax[m], x, lo_v);
          met_apply<T, VEC, LAST, m, W, true>(a, a.pre[m], mo.pre[m] + s1 * a.pre[m].ax[m], x, hi_v);
        } else {
          lo_v = run<k - 1, W>(a, j, off + s0 * ax.in_stride, x, mo);
          hi_v = run<k - 1, W>(a, j, off + s1 * ax.in_stride, x, mo);
        }
#pragma unroll
        for (int q = 0; q < W; ++q)
          r.v[q] = xg_apply_op<T, OP>(ok0 ? lo_v.v[q] : ax.fill, ok1 ? hi_v.v[q] : ax.fill);
        if constexpr (MET) met_apply<T, VEC, LAST, k, W, false>(a, a.post[m], mo.post[m] + j[m] * a.post[m].ax[m], x, r);
      }
      return r;
    }
  }
};

// MARCH = application index of the LAST applied row-axis op.  A thread owns one vector position of
// the innermost dim and walks J consecutive output coordinates of that axis: the lower operand of
// step j+1 is the upper operand of step j (consecutive padded positions), so it stays in
// registers and only ONE evaluation of the levels below is needed per output — for
// interp(['X','Y']) that is one 16-byte load plus one neighbour element per 16-byte store.  The
// only level that can sit above MARCH is the op on the innermost dim (elementwise on the window).
template <typename T, int VEC, int K, int LAST, int MARCH, int OP, bool MET>
__device__ __forceinline__ void multi_body(const MultiArgs<T>& a) {
  constexpr bool kInnerAbove = (LAST > MARCH);
  constexpr int WM = kInnerAbove ? VEC + 1 : VEC;  // window width at the march level
  constexpr int U = MET ? kMetU : 4;
  // With row ops below the march level the select form wins; the plain X,Y case has a single
  // load per step and was faster with the branch.
  constexpr bool kBranchFreeMarch = !(K == 2 && LAST >= 0);
  typedef Eval<T, VEC, K, LAST, OP, MET> E;
  // this block: a segment of the march axis at fixed coordinates of every other row group (MET: the row groups
  // vary fastest, so the blocks of one segment run together and share its metric rows in L2)
  int64_t unit = blockIdx.x;
  int64_t seg;
  if constexpr (MET) {
    seg = unit / a.nrows;
    unit -= seg * a.nrows;
  } else {
    seg = unit % a.nseg;
    unit /= a.nseg;
  }
  int64_t j0 = 0, j1 = 0, j2 = 0;  // separate scalars: a runtime-indexed array would live in local memory
  int64_t off_in = 0, off_out = 0;
  MetOff mo0;
  if constexpr (MET) {
#pragma unroll
    for (int m = 0; m < kMaxAx; ++m) mo0.pre[m] = mo0.post[m] = 0;
  }
#pragma unroll
  for (int g = kMaxGroups - 1; g >= 0; --g) {
    if (g < a.nrow_groups) {
      const int64_t q = unit / a.row_size[g];
      const int64_t c = unit - q * a.row_size[g];
      unit = q;
      off_out += c * a.row_out_stride[g];
      const int ra = a.row_axis[g];
      if (ra == 0) j0 = c;
      else if (ra == 1) j1 = c;
      else if (ra == 2) j2 = c;
      else off_in += c * a.row_in_stride[g];
      if constexpr (MET) {  // row_met holds the stride of an applied axis only for the stages after it
#pragma unroll
        for (int m = 0; m < K; ++m) {
          mo0.pre[m] += c * a.row_met[g][m];
          mo0.post[m] += c * a.row_met[g][K + m];
        }
      }
    }
  }
  const int64_t j[kMaxAx] = {j0, j1, j2};
  const AxisOp<T>& mx = a.ax[MARCH];
  const int64_t jm0 = seg * a.J;
  const int64_t jm1 = (jm0 + a.J < a.march_n_out) ? jm0 + a.J : a.march_n_out;
  const int64_t nvec = (a.last_n_out + VEC - 1) / VEC;  // exact when VEC > 1 (host guarantees it)

  for (int64_t v = threadIdx.x; v < nvec; v += blockDim.x) {
    const int64_t x0 = v * VEC;
    int64_t xw = x0;  // innermost coordinate of the window at the march level
    if constexpr (kInnerAbove) xw = x0 - a.ax[LAST].lo;
    // padded intermediate below the march op at padded position p of the march axis
    auto below = [&](int64_t p) -> Win<T, WM> {
      int64_t sidx;
      const bool ok = resolve(mx, p, sidx);
      auto eval = [&]() -> Win<T, WM> {
        if constexpr (MET) {
          Win<T, WM> r = E::template run<MARCH, WM>(a, j, off_in + sidx * mx.in_stride, xw,
                                                    met_below<T, MARCH>(a, mo0, sidx));
          met_apply<T, VEC, LAST, MARCH, WM, true>(a, a.pre[MARCH], mo0.pre[MARCH] + sidx * a.pre[MARCH].ax[MARCH], xw, r);
          return r;
        } else {
          return E::template run<MARCH, WM>(a, j, off_in + sidx * mx.in_stride, xw, mo0);
        }
      };
      if constexpr (kBranchFreeMarch) {
        // a fill halo reads the clamped row and is replaced, so the U loads batch ahead of use
        Win<T, WM> r = eval();
#pragma unroll
        for (int q = 0; q < WM; ++q) r.v[q] = ok ? r.v[q] : mx.fill;
        return r;
      } else {
        if (ok) return eval();
        Win<T, WM> r;
#pragma unroll
        for (int q = 0; q < WM; ++q) r.v[q] = mx.fill;
        return r;
      }
    };
    auto finish = [&](int64_t jm, const Win<T, WM>& lo_w, const Win<T, WM>& hi_w) {
      Win<T, WM> r;
#pragma unroll
      for (int q = 0; q < WM; ++q) r.v[q] = xg_apply_op<T, OP>(lo_w.v[q], hi_w.v[q]);
      if constexpr (MET)
        met_apply<T, VEC, LAST, MARCH + 1, WM, false>(a, a.post[MARCH], mo0.post[MARCH] + jm * a.post[MARCH].ax[MARCH],
                                                 xw, r);
      XgPack<T, VEC> res;
      if constexpr (kInnerAbove) {
        const AxisOp<T>& ix = a.ax[LAST];
        if constexpr (MET)
          met_apply<T, VEC, LAST, LAST, WM, true>(a, a.pre[LAST], mo0.pre[LAST] + jm * a.pre[LAST].ax[MARCH], xw, r);
        if (ix.bc == XG_BC_FILL) {  // halo cells of the innermost op's own level
          if (xw < 0) r.v[0] = ix.fill;
          if (xw + VEC >= ix.n) r.v[VEC] = ix.fill;
        }
        Win<T, VEC> o;
#pragma unroll
        for (int q = 0; q < VEC; ++q) o.v[q] = xg_apply_op<T, OP>(r.v[q], r.v[q + 1]);
        if constexpr (MET)
          met_apply<T, VEC, LAST, LAST + 1, VEC, false>(a, a.post[LAST], mo0.post[LAST] + jm * a.post[LAST].ax[MARCH],
                                                   x0, o);
#pragma unroll
        for (int q = 0; q < VEC; ++q) res.v[q] = o.v[q];
      } else {
#pragma unroll
        for (int q = 0; q < VEC; ++q) res.v[q] = r.v[q];
      }
      xg_st_stream<T, VEC>(a.out + off_out + jm * a.march_out_stride + x0, res);
    };
    Win<T, WM> prev = below(jm0);
    int64_t jm = jm0;
    for (; jm + U <= jm1; jm += U) {
      Win<T, WM> cur[U];
#pragma unroll
      for (int u = 0; u < U; ++u) cur[u] = below(jm + u + 1);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        finish(jm + u, prev, cur[u]);
        prev = cur[u];
      }
    }
    for (; jm < jm1; ++jm) {
      Win<T, WM> cur = below(jm + 1);
      finish(jm, prev, cur);
      prev = cur;
    }
  }
}

// the weighted body is a call of its own, not inlined beside the metric-free body (which timed as before, DESIGN §3.4)
template <typename T, int VEC, int K, int LAST, int MARCH, int OP>
__device__ __noinline__ void multi_body_met(const MultiArgs<T>& a) {
  multi_body<T, VEC, K, LAST, MARCH, OP, true>(a);
}

template <typename T, int VEC, int K, int LAST, int MARCH, int OP>
__global__ void __launch_bounds__(256, 4) k_stencil_multi(const __grid_constant__ MultiArgs<T> a) {
  if (a.met) multi_body_met<T, VEC, K, LAST, MARCH, OP>(a);  // grid-uniform
  else multi_body<T, VEC, K, LAST, MARCH, OP, false>(a);
}

template <typename T, int VEC, int K, int LAST, int MARCH>
int launch_op(int op, const MultiArgs<T>& a, int64_t nblocks, int threads, cudaStream_t st) {
  const unsigned grid = (unsigned)nblocks;
  switch (op) {
    case XG_OP_DIFF: k_stencil_multi<T, VEC, K, LAST, MARCH, XG_OP_DIFF><<<grid, threads, 0, st>>>(a); break;
    case XG_OP_INTERP: k_stencil_multi<T, VEC, K, LAST, MARCH, XG_OP_INTERP><<<grid, threads, 0, st>>>(a); break;
    case XG_OP_MIN: k_stencil_multi<T, VEC, K, LAST, MARCH, XG_OP_MIN><<<grid, threads, 0, st>>>(a); break;
    default: k_stencil_multi<T, VEC, K, LAST, MARCH, XG_OP_MAX><<<grid, threads, 0, st>>>(a); break;
  }
  return xg_check_launch(a.met ? "xg_stencil_multi(weighted)" : "xg_stencil_multi");
}

template <typename T, int VEC, int K, int LAST>
int launch_march(int march, const MultiArgs<T>& a, int64_t nblocks, int threads, cudaStream_t st) {
  const int op = a.ax[0].op;  // the fused kernel applies one operator along all axes
  // multi_typed marches along the highest application index other than LAST; only that MARCH is
  // instantiated for each (K, LAST)
  constexpr int MARCH = LAST == K - 1 ? K - 2 : K - 1;
  if (march != MARCH) return xg_fail(XG_EINVAL, "xg_stencil_multi: bad march axis");
  return launch_op<T, VEC, K, LAST, MARCH>(op, a, nblocks, threads, st);
}

template <typename T, int VEC, int K>
int launch_last(int last, int march, const MultiArgs<T>& a, int64_t nblocks, int threads, cudaStream_t st) {
  switch (last) {
    case -1: return launch_march<T, VEC, K, -1>(march, a, nblocks, threads, st);
    case 0: return launch_march<T, VEC, K, 0>(march, a, nblocks, threads, st);
    case 1: return launch_march<T, VEC, K, 1>(march, a, nblocks, threads, st);
    case 2:
      if constexpr (K == 3) return launch_march<T, VEC, K, 2>(march, a, nblocks, threads, st);
    default: return xg_fail(XG_EINVAL, "xg_stencil_multi: bad innermost op index");
  }
}

template <typename T>
int multi_typed(const void* in, void* out, int ndim, const int64_t* shape, int naxes, const int* axes,
                const int* ops, const int* lo, const int* hi, const int* bc, const double* fill,
                const void* const* pre, const int64_t* pre_strides, const void* const* post,
                const int64_t* post_strides, cudaStream_t st) {
  constexpr int VEC = XgVecWidth<T>::value;
  MultiArgs<T> a;
  a.in = static_cast<const T*>(in);
  a.out = static_cast<T*>(out);
  a.met = 0;
  for (int k = 0; k < naxes; ++k)
    if ((pre && pre[k]) || (post && post[k])) a.met = 1;
  int64_t out_shape[XG_MAX_NDIM], in_stride[XG_MAX_NDIM], out_stride[XG_MAX_NDIM];
  int app_index[XG_MAX_NDIM];
  for (int d = 0; d < ndim; ++d) {
    out_shape[d] = shape[d];
    app_index[d] = -1;
  }
  for (int k = 0; k < naxes; ++k) {
    const int d = axes[k];
    if (d < 0 || d >= ndim) return xg_fail(XG_EINVAL, "xg_stencil_multi: axis out of range");
    if (app_index[d] >= 0) return xg_fail(XG_EINVAL, "xg_stencil_multi: an axis may appear only once");
    if (lo[k] < 0 || lo[k] > 1 || hi[k] < 0 || hi[k] > 1)
      return xg_fail(XG_EINVAL, "xg_stencil_multi: halo widths must be 0 or 1");
    if ((lo[k] || hi[k]) && (bc[k] < XG_BC_PERIODIC || bc[k] > XG_BC_EXTEND))
      return xg_fail(XG_EINVAL,
                     "xg_stencil_multi: each padded axis needs a periodic / fill / extend boundary");
    if (shape[d] == 0) return xg_fail(XG_EINVAL, "xg_stencil_multi: empty operated axis");
    app_index[d] = k;
    out_shape[d] = shape[d] + lo[k] + hi[k] - 1;
  }
  int64_t total_out = 1;
  {
    int64_t si = 1, so = 1;
    for (int d = ndim - 1; d >= 0; --d) {
      in_stride[d] = si;
      out_stride[d] = so;
      si *= shape[d];
      so *= out_shape[d];
      total_out *= out_shape[d];
    }
  }
  if (total_out == 0) return XG_OK;
  for (int k = 0; k < naxes; ++k) {
    const int d = axes[k];
    a.ax[k].op = ops[k];
    a.ax[k].lo = lo[k];
    a.ax[k].hi = hi[k];
    a.ax[k].bc = bc[k];
    a.ax[k].fill = static_cast<T>(fill[k]);
    a.ax[k].n = shape[d];
    a.ax[k].in_stride = in_stride[d];
  }
  // the common chain — innermost axis first over the last two / three dims, every op length preserving —
  // has a TMA-staged form (xg_stencil_multi_tma.cu); everything else runs the kernel below
  if (!a.met) {
    bool ok = ndim >= 2;
    for (int k = 0; k < naxes && ok; ++k) {
      ok = lo[k] + hi[k] == 1 && axes[k] >= ndim - 3 && (k == 0 || axes[k] < axes[k - 1]);
    }
    if (ok) {
      XgMultiTileSpec<T> ms;
      ms.in = a.in;
      ms.out = a.out;
      ms.op = ops[0];
      for (int q = 0; q < 3; ++q) {
        ms.has[q] = 0;
        ms.lo[q] = 0;
        ms.bc[q] = XG_BC_FILL;
        ms.fill[q] = T(0);
      }
      for (int k = 0; k < naxes; ++k) {
        const int q = ndim - 1 - axes[k];  // 0 = x, 1 = rows, 2 = levels
        ms.has[q] = 1;
        ms.lo[q] = lo[k];
        ms.bc[q] = bc[k];
        ms.fill[q] = static_cast<T>(fill[k]);
      }
      ms.n = shape[ndim - 1];
      ms.P = shape[ndim - 2];
      ms.L = 1;
      for (int d = 0; d < ndim - 2; ++d) ms.L *= shape[d];
      // an operated level axis must be the only level dim (the dims before it have extent 1)
      if (ms.has[2]) ok = ndim >= 3 && ms.L == shape[ndim - 3];
      if (ok) {
        bool launched = false;
        const int rc = xg_multi_tile<T>(ms, st, &launched);
        if (rc || launched) return rc;
      }
    }
  }
  // innermost group: the last dim if it is operated, else the run of trailing non-operated dims
  int last = app_index[ndim - 1];
  int d_end = ndim - 1;  // dims [0, d_end) form the row space
  int64_t last_n_out = out_shape[ndim - 1];
  if (last < 0) {
    while (d_end > 0 && app_index[d_end - 1] < 0) {
      --d_end;
      last_n_out *= out_shape[d_end];
    }
  }
  a.last_n_out = last_n_out;
  // the march axis: the last applied op that is not on the innermost dim
  int march = -1;
  for (int k = naxes - 1; k >= 0; --k)
    if (k != last) { march = k; break; }
  const int march_dim = axes[march];
  a.march_n_out = out_shape[march_dim];
  a.march_out_stride = out_stride[march_dim];
  a.J = a.march_n_out <= 16 ? (int)a.march_n_out : 16;  // flat optimum of a sweep (not repeated on H100)
  if (const char* e = getenv("XG_MULTI_J")) {  // tuning knob (benchmarks only)
    const int tj = atoi(e);
    if (tj > 0) a.J = tj < a.march_n_out ? tj : (int)a.march_n_out;
  }
  a.nseg = xg_ceil_div(a.march_n_out, a.J);
  // row groups: operated dims alone, runs of non-operated dims merged
  a.nrow_groups = 0;
  int64_t nrows = 1;
  for (int d = 0; d < d_end; ++d) {
    if (d == march_dim) continue;
    if (out_shape[d] == 1 && app_index[d] < 0) continue;
    const bool merge = !a.met && a.nrow_groups > 0 && app_index[d] < 0 && a.row_axis[a.nrow_groups - 1] < 0 &&
                       a.row_in_stride[a.nrow_groups - 1] == in_stride[d] * shape[d] &&
                       a.row_out_stride[a.nrow_groups - 1] == out_stride[d] * out_shape[d];
    if (merge) {
      const int g = a.nrow_groups - 1;
      a.row_size[g] *= out_shape[d];
      a.row_in_stride[g] = in_stride[d];
      a.row_out_stride[g] = out_stride[d];
    } else {
      if (a.nrow_groups == kMaxGroups)
        return xg_fail(XG_ENOTIMPL, "xg_stencil_multi: too many interleaved dimensions");
      const int g = a.nrow_groups++;
      a.row_size[g] = out_shape[d];
      a.row_in_stride[g] = in_stride[d];
      a.row_out_stride[g] = out_stride[d];
      a.row_axis[g] = app_index[d];
      // metric strides of the group (a weighted chain keeps one dim per group): a non-operated dim in every
      // operand, an applied axis in the operands of the stages after it
      for (int m = 0; m < naxes; ++m) {
        const bool on = app_index[d] < m;
        a.row_met[g][m] = (a.met && on && pre && pre[m]) ? pre_strides[m * ndim + d] : 0;
        a.row_met[g][naxes + m] = (a.met && on && post && post[m]) ? post_strides[m * ndim + d] : 0;
      }
    }
    nrows *= out_shape[d];
  }
  a.nrows = nrows;
  for (int m = 0; m < kMaxAx; ++m) {
    StageMet<T>* sm[2] = {&a.pre[m], &a.post[m]};
    for (int w = 0; w < 2; ++w) {
      const void* const* ptrs = w ? post : pre;
      const int64_t* st_ = w ? post_strides : pre_strides;
      const bool has = m < naxes && ptrs && ptrs[m];
      sm[w]->p = has ? static_cast<const T*>(ptrs[m]) : nullptr;
      for (int k = 0; k < kMaxAx; ++k) sm[w]->ax[k] = (has && k < naxes) ? st_[m * ndim + axes[k]] : 0;
      sm[w]->x = has ? st_[m * ndim + ndim - 1] : 0;
      bool vec = has && sm[w]->x == 1 && (uintptr_t)ptrs[m] % 16 == 0;
      for (int d = 0; d < ndim - 1 && vec; ++d) vec = st_[m * ndim + d] % VEC == 0;
      sm[w]->vec = vec ? 1 : 0;
    }
  }
  const int64_t nblocks = nrows * a.nseg;
  if (nblocks > 0x7fffffffLL) return xg_fail(XG_ENOTIMPL, "xg_stencil_multi: more than 2^31 blocks");
  // vector path: aligned rows whose length the vector width divides; an operated innermost dim must
  // keep its length (lo + hi == 1) so input and output rows stay aligned with each other
  bool vec_ok = ((uintptr_t)in % 16 == 0) && ((uintptr_t)out % 16 == 0) && (last_n_out % VEC == 0);
  if (last >= 0) vec_ok = vec_ok && (lo[last] + hi[last] == 1) && (shape[ndim - 1] % VEC == 0) && shape[ndim - 1] >= 2 * VEC;
  for (int d = 0; d < ndim - 1 && vec_ok; ++d)
    if (shape[d] > 1 && in_stride[d] % VEC != 0) vec_ok = false;
  for (int d = 0; d < ndim - 1 && vec_ok; ++d)
    if (out_shape[d] > 1 && out_stride[d] % VEC != 0) vec_ok = false;
  const int64_t nvec = vec_ok ? last_n_out / VEC : last_n_out;
  int threads = 256;
  while (threads > 32 && threads / 2 >= nvec) threads /= 2;
  if (naxes == 2) {
    if (vec_ok) return launch_last<T, VEC, 2>(last, march, a, nblocks, threads, st);
    return launch_last<T, 1, 2>(last, march, a, nblocks, threads, st);
  }
  if (vec_ok) return launch_last<T, VEC, 3>(last, march, a, nblocks, threads, st);
  return launch_last<T, 1, 3>(last, march, a, nblocks, threads, st);
}

// Strides of the metric operands: naxes x ndim, stage m against the stage's input (pre) or output (post) shape.
// A stride along a dim of extent 1 is never used.
int check_met(const char* who, int ndim, const int64_t* shape, int naxes, const int* axes, const int* lo,
                     const int* hi, const void* const* met, const int64_t* strides, bool post) {
  if (!met) return XG_OK;
  int64_t sh[XG_MAX_NDIM];
  for (int d = 0; d < ndim; ++d) sh[d] = shape[d];
  for (int m = 0; m < naxes; ++m) {
    if (post) sh[axes[m]] = shape[axes[m]] + lo[m] + hi[m] - 1;
    if (met[m]) {
      if (!strides) return xg_fail(XG_EINVAL, std::string(who) + ": metric strides missing");
      for (int d = 0; d < ndim; ++d)
        if (sh[d] > 1 && strides[m * ndim + d] < 0)
          return xg_fail(XG_EINVAL, std::string(who) + ": negative metric stride");
    }
    if (!post) sh[axes[m]] = shape[axes[m]] + lo[m] + hi[m] - 1;
  }
  return XG_OK;
}

int multi_impl(const char* who, int dtype, const void* in, void* out, int ndim, const int64_t* shape,
                      int naxes, const int* axes, const int* ops, const int* lo, const int* hi, const int* bc,
                      const double* fill_value, const void* const* pre, const int64_t* pre_strides,
                      const void* const* post, const int64_t* post_strides, void* stream) {
  const int rc = xg_stencil_multi_check(who, dtype, in, out, ndim, shape, naxes, axes, ops, lo, hi, bc, fill_value,
                                        pre, pre_strides, post, post_strides);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == XG_F32)
    return multi_typed<float>(in, out, ndim, shape, naxes, axes, ops, lo, hi, bc, fill_value, pre, pre_strides, post,
                              post_strides, st);
  return multi_typed<double>(in, out, ndim, shape, naxes, axes, ops, lo, hi, bc, fill_value, pre, pre_strides, post,
                             post_strides, st);
}

}  // namespace

int xg_stencil_multi_check(const char* who, int dtype, const void* in, const void* out, int ndim,
                           const int64_t* shape, int naxes, const int* axes, const int* ops, const int* lo,
                           const int* hi, const int* bc, const double* fill_value, const void* const* pre,
                           const int64_t* pre_strides, const void* const* post, const int64_t* post_strides) {
  const std::string w = who;
  if (!in || !out || !shape || !axes || !ops || !lo || !hi || !bc || !fill_value)
    return xg_fail(XG_EINVAL, w + ": null pointer");
  if (ndim < 1 || ndim > XG_MAX_NDIM) return xg_fail(XG_EINVAL, w + ": bad ndim");
  if (naxes < 2 || naxes > kMaxAx) return xg_fail(XG_EINVAL, w + ": 2 or 3 axes (use xg_stencil2 for one)");
  for (int k = 0; k < naxes; ++k) {
    if (ops[k] < XG_OP_DIFF || ops[k] > XG_OP_MAX) return xg_fail(XG_EINVAL, w + ": unknown op");
    if (ops[k] != ops[0])
      return xg_fail(XG_ENOTIMPL, w + ": the fused kernel applies ONE operator along all axes "
                                      "(what Grid.diff / interp / min / max do); chain xg_stencil2 for mixed ones");
  }
  if (in == out) return xg_fail(XG_EINVAL, w + ": in-place operation is not supported");
  if (dtype != XG_F32 && dtype != XG_F64) return xg_fail(XG_EINVAL, w + ": dtype must be XG_F32 or XG_F64");
  for (int d = 0; d < ndim; ++d)
    if (shape[d] < 0) return xg_fail(XG_EINVAL, w + ": negative extent");
  bool seen[XG_MAX_NDIM] = {};
  for (int k = 0; k < naxes; ++k) {
    if (axes[k] < 0 || axes[k] >= ndim) return xg_fail(XG_EINVAL, w + ": axis out of range");
    if (seen[axes[k]]) return xg_fail(XG_EINVAL, w + ": an axis may appear only once");
    seen[axes[k]] = true;
    if (lo[k] < 0 || lo[k] > 1 || hi[k] < 0 || hi[k] > 1) return xg_fail(XG_EINVAL, w + ": halo widths must be 0 or 1");
    if ((lo[k] || hi[k]) && (bc[k] < XG_BC_PERIODIC || bc[k] > XG_BC_EXTEND))
      return xg_fail(XG_EINVAL, w + ": each padded axis needs a periodic / fill / extend boundary");
    if (shape[axes[k]] == 0) return xg_fail(XG_EINVAL, w + ": empty operated axis");
  }
  int rc = check_met(who, ndim, shape, naxes, axes, lo, hi, pre, pre_strides, false);
  if (!rc) rc = check_met(who, ndim, shape, naxes, axes, lo, hi, post, post_strides, true);
  if (rc) return rc;
  // a weighted chain addresses its metrics by the coordinates of one innermost dim: the last dim operated, or the
  // one before it
  bool met = false;
  for (int k = 0; k < naxes; ++k) met = met || (pre && pre[k]) || (post && post[k]);
  if (met && ndim >= 2 && !seen[ndim - 1] && !seen[ndim - 2])
    return xg_fail(XG_ENOTIMPL, w + ": metrics with more than one non-operated dim after the last operated one");
  return XG_OK;
}

extern "C" int xg_stencil_multi(int dtype, const void* in, void* out, int ndim, const int64_t* shape,
                                int naxes, const int* axes, const int* ops, const int* lo, const int* hi,
                                const int* bc, const double* fill_value, void* stream) {
  return multi_impl("xg_stencil_multi", dtype, in, out, ndim, shape, naxes, axes, ops, lo, hi, bc, fill_value,
                    nullptr, nullptr, nullptr, nullptr, stream);
}

extern "C" int xg_stencil_multi_weighted(int dtype, const void* in, void* out, int ndim, const int64_t* shape,
                                         int naxes, const int* axes, const int* ops, const int* lo, const int* hi,
                                         const int* bc, const double* fill_value, const void* const* pre,
                                         const int64_t* pre_strides, const void* const* post,
                                         const int64_t* post_strides, void* stream) {
  return multi_impl("xg_stencil_multi_weighted", dtype, in, out, ndim, shape, naxes, axes, ops, lo, hi, bc,
                    fill_value, pre, pre_strides, post, post_strides, stream);
}
