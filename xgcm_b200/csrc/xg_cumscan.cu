// xg_cumscan — cumulative sum with xgcm's position-shift bookkeeping, one HBM pass.
//
// Replaces xgcm/grid.py:1306-1414:  (x metric) -> [flip] -> DataArray.cumsum -> [flip]
// -> trim (table :1326-1383) -> pad() of the cumsum'd data (:1385-1391) -> (/ metric).
//
// Summation order is STRICTLY SEQUENTIAL along the axis, because np.cumsum is
// (on every layout) and a tree scan already differs by 2e-6 rel in fp32 at
// n = 3600 (SURVEY H4) — outside the 1e-6 parity budget.  Parallelism comes from
// the independent lines instead:
//   k_scan_strided  inner > 1: one thread per 16-byte column vector marches the
//       axis; U independent loads in flight, only the adds are serial.
//   k_scan_rows     inner == 1: a warp owns 32 rows; 32x32 tiles go through
//       shared memory (coalesced 128 B row segments in, lane-per-row serial scan,
//       coalesced segments out) with the running sums carried in registers.
//
// Roofline: HBM, 2 * sizeof(T) bytes per cell.
#include "xg_common.cuh"

namespace {

constexpr int kThreads = 128;

template <typename T>
struct ScanArgs {
  const T* in;
  T* out;
  int64_t outer, n, inner, n_out;
  int64_t k_first, k_last;  // kept range of the cumsum (after trim), inclusive
  int reverse, pad_lo, pad_hi, bc, skipna;
  T fill;
  XgOperand pre, post;
  int64_t nvec_inner;
  bool small_index;  // outer * nvec_inner < 2^31
  XgFastDiv fd_nvi;  // multiply-high form of nvec_inner (valid with small_index)
};

template <typename T>
__device__ __forceinline__ T nan_to_zero(T v, int skipna) {
  return (skipna && xg_isnan(v)) ? T(0) : v;
}

// value of a halo cell from the recorded ends of the trimmed cumsum
template <typename T>
__device__ __forceinline__ T halo_value(bool low, int bc, T fill, T cf, T cf1, T cl1, T cl) {
  if (bc == XG_BC_FILL) return fill;
  if (bc == XG_BC_PERIODIC) return low ? cl : cf;
  if (bc == XG_BC_EXTEND) return low ? cf : cl;
  return low ? (T(2) * cf - cf1) : (T(2) * cl - cl1);  // extrapolate
}

// ------------------------------------------------------------------ strided axis
template <typename T, int VEC, bool MET, int U>
__global__ void __launch_bounds__(kThreads) k_scan_strided(const ScanArgs<T> a) {
  typedef XgPack<T, VEC> Pack;
  const int64_t g = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (g >= a.outer * a.nvec_inner) return;
  int64_t o, iv;
  xg_divmod(g, a.nvec_inner, a.fd_nvi, a.small_index, o, iv);
  const int64_t i = iv * VEC;
  const T* ibase = a.in + o * a.n * a.inner + i;
  T* obase = a.out + o * a.n_out * a.inner + i;
  const bool has_pre = MET && a.pre.ptr != nullptr;
  const bool has_post = MET && a.post.ptr != nullptr;
  XgOperandView<T, VEC> pre_v, post_v;
  if (MET) {
    if (has_pre) pre_v = xg_operand_view<T, VEC>(a.pre, xg_groups_offset(a.pre.outer, o), i);
    if (has_post) post_v = xg_operand_view<T, VEC>(a.post, xg_groups_offset(a.post.outer, o), i);
  }
  auto loadA = [&](int64_t k) -> Pack {
    Pack v = xg_ld_stream<T, VEC>(ibase + k * a.inner);
    if (has_pre) {
      Pack m = xg_ld_view<T, VEC>(pre_v, k * a.pre.axis_stride);
#pragma unroll
      for (int q = 0; q < VEC; ++q) v.v[q] = v.v[q] * m.v[q];
    }
    return v;
  };
  auto store = [&](int64_t j_out, Pack v) {
    if (has_post) {
      Pack m = xg_ld_view<T, VEC>(post_v, j_out * a.post.axis_stride);
#pragma unroll
      for (int q = 0; q < VEC; ++q) v.v[q] = v.v[q] / m.v[q];
    }
    xg_st_stream<T, VEC>(obase + j_out * a.inner, v);
  };

  Pack acc, cf, cf1, cl1, cl;
#pragma unroll
  for (int q = 0; q < VEC; ++q) acc.v[q] = cf.v[q] = cf1.v[q] = cl1.v[q] = cl.v[q] = T(0);

  const int n = (int)a.n;  // < 2^31, checked on the host
  const int k_first = (int)a.k_first, k_last = (int)a.k_last;
  auto kof = [&](int kk) -> int { return a.reverse ? (n - 1 - kk) : kk; };
  // the ends of the trimmed cumsum (needed by the halo rules) live in the first / last three
  // rows; only those rows pay for the bookkeeping
  auto step_slow = [&](int kk, const Pack& v) {
    const int k = kof(kk);
#pragma unroll
    for (int q = 0; q < VEC; ++q) acc.v[q] = acc.v[q] + nan_to_zero(v.v[q], a.skipna);
    if (k == k_first) cf = acc;
    if (k == k_first + 1) cf1 = acc;
    if (k == k_last - 1) cl1 = acc;
    if (k == k_last) cl = acc;
    if (k >= k_first && k <= k_last) store(a.pad_lo + (k - k_first), acc);
  };
  auto step_fast = [&](int kk, const Pack& v) {  // interior rows are always kept
#pragma unroll
    for (int q = 0; q < VEC; ++q) acc.v[q] = acc.v[q] + nan_to_zero(v.v[q], a.skipna);
    store(a.pad_lo + (kof(kk) - k_first), acc);
  };

  int kk = 0;
  const int head = n < 3 ? n : 3;
  for (; kk < head; ++kk) step_slow(kk, loadA(kof(kk)));
  const int mid_end = n - 3;  // rows [3, n-3) are interior
  // software pipeline: the loads of chunk c+1 are in flight while chunk c is summed (the adds
  // are serial by construction, so memory-level parallelism has to come from prefetch depth)
  if (mid_end - kk >= U) {
    Pack cur[U], nxt[U];
#pragma unroll
    for (int u = 0; u < U; ++u) cur[u] = loadA(kof(kk + u));
    for (; kk + 2 * U <= mid_end; kk += U) {
#pragma unroll
      for (int u = 0; u < U; ++u) nxt[u] = loadA(kof(kk + U + u));
#pragma unroll
      for (int u = 0; u < U; ++u) step_fast(kk + u, cur[u]);
#pragma unroll
      for (int u = 0; u < U; ++u) cur[u] = nxt[u];
    }
#pragma unroll
    for (int u = 0; u < U; ++u) step_fast(kk + u, cur[u]);
    kk += U;
  }
  for (; kk < mid_end; ++kk) step_fast(kk, loadA(kof(kk)));
  for (; kk < n; ++kk) step_slow(kk, loadA(kof(kk)));

  if (a.k_last - a.k_first < 1) {  // a single kept cell: "next" is the edge itself
    cf1 = cf;
    cl1 = cl;
  }
  if (a.pad_lo) {
    Pack h;
#pragma unroll
    for (int q = 0; q < VEC; ++q)
      h.v[q] = halo_value<T>(true, a.bc, a.fill, cf.v[q], cf1.v[q], cl1.v[q], cl.v[q]);
    store(0, h);
  }
  if (a.pad_hi) {
    Pack h;
#pragma unroll
    for (int q = 0; q < VEC; ++q)
      h.v[q] = halo_value<T>(false, a.bc, a.fill, cf.v[q], cf1.v[q], cl1.v[q], cl.v[q]);
    store(a.n_out - 1, h);
  }
}

// ------------------------------------------------------------------ innermost axis
constexpr int kRowWarps = 4;
constexpr int kTile = 32;
constexpr int kStages = 2;

// 4- / 8-byte asynchronous global->shared copy (LDGSTS): the tile of the NEXT step is in flight
// while the current one is scanned, at no register cost
template <typename T>
__device__ __forceinline__ void cp_async_elem(T* smem_dst, const T* gsrc) {
  const unsigned dst = (unsigned)__cvta_generic_to_shared(smem_dst);
  if constexpr (sizeof(T) == 4)
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(gsrc) : "memory");
  else
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

template <typename T>
struct RowTileSmem {
  T tile[kRowWarps][kStages][kTile][kTile + 1];
  int64_t pre_off[kRowWarps][kTile];
  int64_t post_off[kRowWarps][kTile];
};

template <typename T, bool MET>
__global__ void __launch_bounds__(kRowWarps * 32) k_scan_rows(const ScanArgs<T> a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  RowTileSmem<T>& sm = *reinterpret_cast<RowTileSmem<T>*>(smem_raw);
  const int w = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int64_t unit = (int64_t)blockIdx.x * kRowWarps + w;
  const int64_t r0 = unit * kTile;
  if (r0 >= a.outer) return;  // warp-uniform
  const int64_t my_row = r0 + lane;
  const bool row_ok = my_row < a.outer;
  const int nrows = (int)((a.outer - r0 < kTile) ? (a.outer - r0) : kTile);
  if (MET) {
    sm.pre_off[w][lane] = (a.pre.ptr && row_ok) ? xg_groups_offset(a.pre.outer, my_row) : 0;
    sm.post_off[w][lane] = (a.post.ptr && row_ok) ? xg_groups_offset(a.post.outer, my_row) : 0;
  }
  __syncwarp();
  const T* prep = reinterpret_cast<const T*>(a.pre.ptr);
  const T* postp = reinterpret_cast<const T*>(a.post.ptr);
  const T* in0 = a.in + r0 * a.n;

  const int64_t ntile = xg_ceil_div(a.n, kTile);
  auto tile_c0 = [&](int64_t tt) -> int64_t { return (a.reverse ? (ntile - 1 - tt) : tt) * kTile; };
  // coalesced: one 32-element row segment per instruction, all 32 rows in flight at once
  auto issue = [&](int64_t tt, int stage) {
    const int64_t kcol = tile_c0(tt) + lane;
    T(*tile)[kTile + 1] = sm.tile[w][stage];
    if (kcol < a.n) {
      const T* src = in0 + kcol;
      if (nrows == kTile) {
#pragma unroll
        for (int rr = 0; rr < kTile; ++rr) cp_async_elem<T>(&tile[rr][lane], src + (int64_t)rr * a.n);
      } else {
#pragma unroll 8
        for (int rr = 0; rr < kTile; ++rr) {
          if (rr < nrows) cp_async_elem<T>(&tile[rr][lane], src + (int64_t)rr * a.n);
          else tile[rr][lane] = T(0);
        }
      }
    } else {
#pragma unroll 8
      for (int rr = 0; rr < kTile; ++rr) tile[rr][lane] = T(0);
    }
    cp_async_commit();
  };

  T acc = T(0), cf = T(0), cf1 = T(0), cl1 = T(0), cl = T(0);
  const int n = (int)a.n;  // < 2^31, checked on the host
  const int k_first = (int)a.k_first, k_last = (int)a.k_last;
  const int shift = a.pad_lo - k_first;  // j_out = k + shift
  issue(0, 0);
  for (int64_t tt = 0; tt < ntile; ++tt) {
    const int stage = (int)(tt % kStages);
    if (tt + 1 < ntile) {
      issue(tt + 1, (int)((tt + 1) % kStages));
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncwarp();
    T(*tile)[kTile + 1] = sm.tile[w][stage];
    const int c0 = (int)tile_c0(tt);
    const int kcol = c0 + lane;
    const bool col_ok = kcol < n;
    // tiles holding one of the recorded ends of the trimmed cumsum (first / last two cells) or
    // the ragged end of the row take the careful path; every other tile is branch-free
    const bool interior = (c0 > k_first + 1) && (c0 + kTile - 1 < k_last - 1) && (c0 + kTile <= n);
    if (MET && prep) {  // metric multiply with coalesced metric loads (lane = column)
      if (col_ok) {
#pragma unroll 8
        for (int rr = 0; rr < kTile; ++rr)
          if (rr < nrows)
            tile[rr][lane] = tile[rr][lane] * __ldg(prep + sm.pre_off[w][rr] + (int64_t)kcol * a.pre.axis_stride);
      }
      __syncwarp();
    }
    // serial scan: lane = row (row pitch 33 words: conflict-free)
    if (row_ok) {
      if (interior) {
        if (a.reverse) {
#pragma unroll
          for (int c = kTile - 1; c >= 0; --c) {
            acc = acc + nan_to_zero(tile[lane][c], a.skipna);
            tile[lane][c] = acc;
          }
        } else {
#pragma unroll
          for (int c = 0; c < kTile; ++c) {
            acc = acc + nan_to_zero(tile[lane][c], a.skipna);
            tile[lane][c] = acc;
          }
        }
      } else {
#pragma unroll 4
        for (int cc = 0; cc < kTile; ++cc) {
          const int c = a.reverse ? (kTile - 1 - cc) : cc;
          const int k = c0 + c;
          if (k < n) {
            acc = acc + nan_to_zero(tile[lane][c], a.skipna);
            tile[lane][c] = acc;
            if (k == k_first) cf = acc;
            if (k == k_first + 1) cf1 = acc;
            if (k == k_last - 1) cl1 = acc;
            if (k == k_last) cl = acc;
          }
        }
      }
    }
    __syncwarp();
    // coalesced store of the kept cells (shifted by pad_lo - k_first)
    if (col_ok && kcol >= k_first && kcol <= k_last) {
      const int j_out = kcol + shift;
      T* optr = a.out + r0 * a.n_out + j_out;
      if (MET && postp) {
#pragma unroll 8
        for (int rr = 0; rr < kTile; ++rr) {
          if (rr < nrows) {
            const T v = tile[rr][lane] / __ldg(postp + sm.post_off[w][rr] + (int64_t)j_out * a.post.axis_stride);
            __stcs(optr + (int64_t)rr * a.n_out, v);
          }
        }
      } else if (nrows == kTile) {
#pragma unroll
        for (int rr = 0; rr < kTile; ++rr) __stcs(optr + (int64_t)rr * a.n_out, tile[rr][lane]);
      } else {
        for (int rr = 0; rr < nrows; ++rr) __stcs(optr + (int64_t)rr * a.n_out, tile[rr][lane]);
      }
    }
    __syncwarp();  // the stage is overwritten by the copy issued two iterations later
  }
  if (!row_ok) return;
  if (a.k_last - a.k_first < 1) {
    cf1 = cf;
    cl1 = cl;
  }
  if (a.pad_lo) {
    T h = halo_value<T>(true, a.bc, a.fill, cf, cf1, cl1, cl);
    if (MET && postp) h = h / __ldg(postp + sm.post_off[w][lane]);
    a.out[my_row * a.n_out] = h;
  }
  if (a.pad_hi) {
    T h = halo_value<T>(false, a.bc, a.fill, cf, cf1, cl1, cl);
    if (MET && postp)
      h = h / __ldg(postp + sm.post_off[w][lane] + (a.n_out - 1) * a.post.axis_stride);
    a.out[my_row * a.n_out + a.n_out - 1] = h;
  }
}

// ------------------------------------------------------------------ innermost axis, wide tiles
// Same algorithm with 16-byte shared / global accesses: a tile is 32 rows x 32 chunks of 16 B
// (128 fp32 or 64 fp64 columns).  Per byte moved this issues 4x fewer LDGSTS / LDS / STS / STG
// than the 32x32 scalar tile, which is what bounds that kernel (MIO
// throughput).  Chunks are XOR-swizzled with the row index so that both the row-wise copies
// (lane = chunk) and the lane-per-row scan (lane = row, LDS.128) are bank-conflict free.
constexpr int kWideWarps = 2;
constexpr int kChunks = 32;  // 16-byte chunks per tile row

struct __align__(16) Chunk16 {
  unsigned int w[4];
};

template <typename T>
struct WideSmem {
  Chunk16 tile[kWideWarps][kStages][kTile][kChunks];
  int64_t pre_off[kWideWarps][kTile];
  int64_t post_off[kWideWarps][kTile];
};

__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gsrc) {
  const unsigned dst = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(gsrc) : "memory");
}

template <typename T, bool MET>
__global__ void __launch_bounds__(kWideWarps * 32) k_scan_rows_wide(const ScanArgs<T> a) {
  constexpr int E = 16 / sizeof(T);       // elements per chunk
  constexpr int TW = kChunks * E;         // tile width in elements
  extern __shared__ __align__(16) unsigned char smem_raw[];
  WideSmem<T>& sm = *reinterpret_cast<WideSmem<T>*>(smem_raw);
  const int w = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int64_t unit = (int64_t)blockIdx.x * kWideWarps + w;
  const int64_t r0 = unit * kTile;
  if (r0 >= a.outer) return;  // warp-uniform
  const int64_t my_row = r0 + lane;
  const bool row_ok = my_row < a.outer;
  const int nrows = (int)((a.outer - r0 < kTile) ? (a.outer - r0) : kTile);
  if (MET) {
    sm.pre_off[w][lane] = (a.pre.ptr && row_ok) ? xg_groups_offset(a.pre.outer, my_row) : 0;
    sm.post_off[w][lane] = (a.post.ptr && row_ok) ? xg_groups_offset(a.post.outer, my_row) : 0;
  }
  __syncwarp();
  const T* prep = reinterpret_cast<const T*>(a.pre.ptr);
  const T* postp = reinterpret_cast<const T*>(a.post.ptr);
  const T* in0 = a.in + r0 * a.n;
  const int n = (int)a.n;
  const int k_first = (int)a.k_first, k_last = (int)a.k_last;
  const int shift = a.pad_lo - k_first;  // j_out = k + shift
  const bool wide_store = (shift == 0) && (a.n_out % E == 0) && (((uintptr_t)a.out & 15) == 0) && !(MET && postp);
  const int ntile = (n + TW - 1) / TW;
  auto tile_c0 = [&](int tt) -> int { return (a.reverse ? (ntile - 1 - tt) : tt) * TW; };

  // row-wise copy: lane = chunk; chunk q of row rr lands in physical slot q ^ (rr & 31)
  auto issue = [&](int tt, int stage) {
    const int kc = tile_c0(tt) + lane * E;  // first element of this lane's chunk
    Chunk16(*tile)[kChunks] = sm.tile[w][stage];
    if (kc < n) {  // rows are multiples of E long: a chunk is entirely in or out
      const T* src = in0 + kc;
#pragma unroll 8
      for (int rr = 0; rr < kTile; ++rr)
        if (rr < nrows) cp_async_16(&tile[rr][lane ^ rr], src + (int64_t)rr * a.n);
    }
    cp_async_commit();
  };

  T acc = T(0), cf = T(0), cf1 = T(0), cl1 = T(0), cl = T(0);
  issue(0, 0);
  for (int tt = 0; tt < ntile; ++tt) {
    const int stage = tt % kStages;
    if (tt + 1 < ntile) {
      issue(tt + 1, (tt + 1) % kStages);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncwarp();
    Chunk16(*tile)[kChunks] = sm.tile[w][stage];
    const int c0 = tile_c0(tt);
    const int kc = c0 + lane * E;
    const bool chunk_ok = kc < n;
    const int nchunk = (n - c0 >= TW) ? kChunks : (n - c0) / E;  // valid chunks in this tile
    const bool interior = (c0 > k_first + 1) && (c0 + TW - 1 < k_last - 1) && (nchunk == kChunks);
    if (MET && prep) {  // metric multiply, lane = chunk (coalesced metric reads)
      if (chunk_ok) {
        for (int rr = 0; rr < nrows; ++rr) {
          Chunk16 c = tile[rr][lane ^ rr];
          T* v = reinterpret_cast<T*>(&c);
          const T* mp = prep + sm.pre_off[w][rr] + (int64_t)kc * a.pre.axis_stride;
#pragma unroll
          for (int e = 0; e < E; ++e) v[e] = v[e] * __ldg(mp + (int64_t)e * a.pre.axis_stride);
          tile[rr][lane ^ rr] = c;
        }
      }
      __syncwarp();
    }
    // serial scan: lane = row, one 16-byte chunk per shared-memory access
    if (row_ok) {
      if (interior) {
#pragma unroll 8
        for (int qq = 0; qq < kChunks; ++qq) {
          const int q = a.reverse ? (kChunks - 1 - qq) : qq;
          Chunk16 c = tile[lane][q ^ lane];
          T* v = reinterpret_cast<T*>(&c);
          if (a.reverse) {
#pragma unroll
            for (int e = E - 1; e >= 0; --e) { acc = acc + nan_to_zero(v[e], a.skipna); v[e] = acc; }
          } else {
#pragma unroll
            for (int e = 0; e < E; ++e) { acc = acc + nan_to_zero(v[e], a.skipna); v[e] = acc; }
          }
          tile[lane][q ^ lane] = c;
        }
      } else {
        for (int qq = 0; qq < nchunk; ++qq) {
          const int q = a.reverse ? (nchunk - 1 - qq) : qq;
          Chunk16 c = tile[lane][q ^ lane];
          T* v = reinterpret_cast<T*>(&c);
#pragma unroll
          for (int ee = 0; ee < E; ++ee) {
            const int e = a.reverse ? (E - 1 - ee) : ee;
            const int k = c0 + q * E + e;
            acc = acc + nan_to_zero(v[e], a.skipna);
            v[e] = acc;
            if (k == k_first) cf = acc;
            if (k == k_first + 1) cf1 = acc;
            if (k == k_last - 1) cl1 = acc;
            if (k == k_last) cl = acc;
          }
          tile[lane][q ^ lane] = c;
        }
      }
    }
    __syncwarp();
    // store: lane = chunk
    if (chunk_ok) {
      if (wide_store && interior) {
        T* optr = a.out + r0 * a.n_out + kc;
        if (nrows == kTile) {
#pragma unroll 8
          for (int rr = 0; rr < kTile; ++rr)
            __stcs(reinterpret_cast<uint4*>(optr + (int64_t)rr * a.n_out),
                   *reinterpret_cast<const uint4*>(&tile[rr][lane ^ rr]));
        } else {
          for (int rr = 0; rr < nrows; ++rr)
            __stcs(reinterpret_cast<uint4*>(optr + (int64_t)rr * a.n_out),
                   *reinterpret_cast<const uint4*>(&tile[rr][lane ^ rr]));
        }
      } else {
        for (int rr = 0; rr < nrows; ++rr) {
          Chunk16 c = tile[rr][lane ^ rr];
          const T* v = reinterpret_cast<const T*>(&c);
#pragma unroll
          for (int e = 0; e < E; ++e) {
            const int k = kc + e;
            if (k >= k_first && k <= k_last) {
              const int j_out = k + shift;
              T val = v[e];
              if (MET && postp) val = val / __ldg(postp + sm.post_off[w][rr] + (int64_t)j_out * a.post.axis_stride);
              __stcs(a.out + (r0 + rr) * a.n_out + j_out, val);
            }
          }
        }
      }
    }
    __syncwarp();
  }
  if (!row_ok) return;
  if (a.k_last - a.k_first < 1) {
    cf1 = cf;
    cl1 = cl;
  }
  if (a.pad_lo) {
    T h = halo_value<T>(true, a.bc, a.fill, cf, cf1, cl1, cl);
    if (MET && postp) h = h / __ldg(postp + sm.post_off[w][lane]);
    a.out[my_row * a.n_out] = h;
  }
  if (a.pad_hi) {
    T h = halo_value<T>(false, a.bc, a.fill, cf, cf1, cl1, cl);
    if (MET && postp)
      h = h / __ldg(postp + sm.post_off[w][lane] + (a.n_out - 1) * a.post.axis_stride);
    a.out[my_row * a.n_out + a.n_out - 1] = h;
  }
}

template <typename T, bool MET>
int scan_launch(ScanArgs<T>& a, cudaStream_t st) {
  constexpr int VEC = XgVecWidth<T>::value;
  constexpr int U = 8;
  if (a.inner > 1) {
    bool vec_ok = (a.inner % VEC == 0) && ((uintptr_t)a.in % 16 == 0) && ((uintptr_t)a.out % 16 == 0) &&
                  xg_vec_view_ok(a.pre) && xg_vec_view_ok(a.post);
    // few columns: prefer 4x more (scalar) threads over 16-byte accesses
    if (vec_ok && a.outer * (a.inner / VEC) < XG_SMS * 64) vec_ok = false;
    if (vec_ok) {
      a.nvec_inner = a.inner / VEC;
      a.small_index = a.outer * a.nvec_inner < (1ll << 31);
      a.fd_nvi = xg_fastdiv_make(a.small_index ? a.nvec_inner : 1);
      const int64_t blocks = xg_ceil_div(a.outer * a.nvec_inner, kThreads);
      if (blocks > 0x7fffffffLL) return xg_fail(XG_EINVAL, "xg_cumscan: grid too large");
      k_scan_strided<T, VEC, MET, U><<<(unsigned)blocks, kThreads, 0, st>>>(a);
    } else {
      a.pre.vec_ok = 0;
      a.post.vec_ok = 0;
      a.nvec_inner = a.inner;
      a.small_index = a.outer * a.nvec_inner < (1ll << 31);
      a.fd_nvi = xg_fastdiv_make(a.small_index ? a.nvec_inner : 1);
      const int64_t blocks = xg_ceil_div(a.outer * a.nvec_inner, kThreads);
      if (blocks > 0x7fffffffLL) return xg_fail(XG_EINVAL, "xg_cumscan: grid too large");
      k_scan_strided<T, 1, MET, U><<<(unsigned)blocks, kThreads, 0, st>>>(a);
    }
    return xg_check_launch(vec_ok ? "xg_cumscan(strided, vec)" : "xg_cumscan(strided, scalar)");
  }
  const int64_t units = xg_ceil_div(a.outer, kTile);
  constexpr int E = 16 / sizeof(T);
  if (a.n % E == 0 && a.n >= 4 * E * kChunks && ((uintptr_t)a.in & 15) == 0) {
    const int64_t wblocks = xg_ceil_div(units, kWideWarps);
    if (wblocks > 0x7fffffffLL) return xg_fail(XG_EINVAL, "xg_cumscan: grid too large");
    const size_t wsmem = sizeof(WideSmem<T>);
    cudaError_t e = cudaFuncSetAttribute(k_scan_rows_wide<T, MET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsmem);
    if (e != cudaSuccess) return xg_fail(XG_ECUDA, std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e));
    k_scan_rows_wide<T, MET><<<(unsigned)wblocks, kWideWarps * 32, wsmem, st>>>(a);
    return xg_check_launch("xg_cumscan(rows, wide)");
  }
  const int64_t blocks = xg_ceil_div(units, kRowWarps);
  if (blocks > 0x7fffffffLL) return xg_fail(XG_EINVAL, "xg_cumscan: grid too large");
  const size_t smem = sizeof(RowTileSmem<T>);
  {  // > 48 KiB for fp64: opt in (per device, cheap)
    cudaError_t e = cudaFuncSetAttribute(k_scan_rows<T, MET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return xg_fail(XG_ECUDA, std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e));
  }
  k_scan_rows<T, MET><<<(unsigned)blocks, kRowWarps * 32, smem, st>>>(a);
  return xg_check_launch("xg_cumscan(rows)");
}

template <typename T>
int cumscan_typed(const void* in, void* out, int ndim, const int64_t* shape, int axis, int reverse,
                  int trim, int pad_lo, int pad_hi, int bc, double fill, const void* pre_metric,
                  const int64_t* pre_strides, const void* post_metric,
                  const int64_t* post_strides, int skipna, cudaStream_t st) {
  constexpr int VEC = XgVecWidth<T>::value;
  XgView v;
  int rc = xg_collapse_view(ndim, shape, axis, &v);
  if (rc) return rc;
  ScanArgs<T> a;
  a.in = static_cast<const T*>(in);
  a.out = static_cast<T*>(out);
  a.outer = v.outer;
  a.n = v.n;
  a.inner = v.inner;
  a.k_first = (trim == XG_TRIM_DROP_FIRST) ? 1 : 0;
  a.k_last = v.n - 1 - ((trim == XG_TRIM_DROP_LAST) ? 1 : 0);
  const int64_t kept = a.k_last - a.k_first + 1;
  if (kept < 0) return xg_fail(XG_EINVAL, "xg_cumscan: operated axis too short to trim");
  if (v.n >= (1ll << 31)) return xg_fail(XG_EINVAL, "xg_cumscan: operated axis longer than 2^31");
  a.n_out = kept + pad_lo + pad_hi;
  a.reverse = reverse ? 1 : 0;
  a.pad_lo = pad_lo;
  a.pad_hi = pad_hi;
  a.bc = bc;
  a.skipna = skipna ? 1 : 0;
  a.fill = static_cast<T>(fill);
  a.nvec_inner = 0;
  a.small_index = false;
  a.fd_nvi = xg_fastdiv_make(1);
  if (kept == 0 && (pad_lo || pad_hi) && bc != XG_BC_FILL)
    return xg_fail(XG_EINVAL, "xg_cumscan: cannot wrap/extend an empty axis");
  if (v.outer == 0 || v.inner == 0 || a.n_out == 0) return XG_OK;
  int64_t out_shape[XG_MAX_NDIM];
  for (int d = 0; d < ndim; ++d) out_shape[d] = shape[d];
  out_shape[axis] = a.n_out;
  rc = xg_make_operand(pre_metric, pre_strides, ndim, shape, axis, VEC, sizeof(T), &a.pre,
                       "xg_cumscan(pre_metric)");
  if (rc) return rc;
  rc = xg_make_operand(post_metric, post_strides, ndim, out_shape, axis, VEC, sizeof(T), &a.post,
                       "xg_cumscan(post_metric)");
  if (rc) return rc;
  if (a.pre.ptr || a.post.ptr) return scan_launch<T, true>(a, st);
  return scan_launch<T, false>(a, st);
}

}  // namespace

extern "C" int xg_cumscan(int dtype, const void* in, void* out, int ndim, const int64_t* shape,
                          int axis, int reverse, int trim, int pad_lo, int pad_hi, int bc,
                          double fill_value, const void* pre_metric, const int64_t* pre_strides,
                          const void* post_metric, const int64_t* post_strides, int skipna,
                          void* stream) {
  if (!in || !out || !shape) return xg_fail(XG_EINVAL, "xg_cumscan: null pointer");
  if (pad_lo < 0 || pad_lo > 1 || pad_hi < 0 || pad_hi > 1)
    return xg_fail(XG_EINVAL, "xg_cumscan: halo widths must be 0 or 1");
  if (trim < XG_TRIM_NONE || trim > XG_TRIM_DROP_FIRST)
    return xg_fail(XG_EINVAL, "xg_cumscan: unknown trim mode");
  if ((pad_lo || pad_hi) && (bc <= XG_BC_NONE || bc > XG_BC_EXTRAPOLATE))
    // padding.py:601-608
    return xg_fail(XG_EINVAL,
                   "xg_cumscan: no boundary condition was specified but the operation needs to "
                   "pad the axis");
  if (in == out) return xg_fail(XG_EINVAL, "xg_cumscan: in-place operation is not supported");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == XG_F32)
    return cumscan_typed<float>(in, out, ndim, shape, axis, reverse, trim, pad_lo, pad_hi, bc,
                                fill_value, pre_metric, pre_strides, post_metric, post_strides,
                                skipna, st);
  if (dtype == XG_F64)
    return cumscan_typed<double>(in, out, ndim, shape, axis, reverse, trim, pad_lo, pad_hi, bc,
                                 fill_value, pre_metric, pre_strides, post_metric, post_strides,
                                 skipna, st);
  return xg_fail(XG_EINVAL, "xg_cumscan: dtype must be XG_F32 or XG_F64");
}
