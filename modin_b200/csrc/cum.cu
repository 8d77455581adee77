// cum.cu — the Fold template's kernels: running sum / max / min and forward fill down the rows of every column.
//
// Reference path: Fold.register (alg/fold.py:32-95) -> PandasDataframe.fold (df.py:2357-2400) ->
// map_axis_partitions(keep_partitioning=True): every column partition is gathered into ONE pandas frame, the
// function (pandas.DataFrame.cumsum / cummax / cummin, qc.py:2429-2431; fillna(method="ffill"), qc.py:2809-2810)
// runs over it sequentially, the result is split again.  pandas' cumulative functions skip NaN: the running value
// ignores them and the output keeps NaN where the input had it (nanops / masked_accumulations: fill with the identity,
// accumulate, restore).  That is a scan over a monoid, so it parallelises:
//
//   value v[i]  = identity where x[i] is NaN (+0.0 for the sum, whose identity is -0.0), else x[i]
//   S[i]        = v[0] (+) ... (+) v[i]            (+) in {+, max, min, "latest valid"}
//   out[i]      = NaN where x[i] is NaN, else S[i]  (forward fill: S[i] everywhere)
//
// Three launches over tiles of 4096 rows, one grid row per column (columns are separate buffers):
//   1. cum_tile_reduce_kernel   tile -> its aggregate                                   (reads 8 B / element)
//   2. cum_scan_tiles_kernel    one CTA per column: exclusive scan of the tile aggregates, in place; column total out
//   3. cum_tile_scan_kernel     tile + its prefix (+ the carry of the rows that precede this block: lower ranks,
//                               earlier row partitions) -> output                      (reads 8, writes 8 B / element)
// Algorithmic traffic 16 B / element; this first version moves 24 (the input is read twice), so its ceiling is 2/3 of
// the HBM roofline.  A single-pass decoupled look-back scan would reach 16 B; it makes CTAs wait on each other,
// which is not something to write without a GPU to debug on (DESIGN.md §6).  Tiles are staged through shared memory:
// coalesced 8-byte accesses on the global side (any 8-byte-aligned view works, ragged tails included), 16 consecutive
// elements per thread on the scan side (index padded by 1 per 16 so both sides are bank-conflict free).
//
// Every reduction here keeps operand ORDER (shfl_down / shfl_up trees, left operand = earlier rows), because
// "latest valid" is not commutative.  Float sums are associated differently from pandas' sequential loop: the tests
// state the bound (|err| <= 4 log2(n) eps * running sum of |x|); max / min / forward fill and all int64 results are
// bit-exact.
#include <limits.h>

#include "common.cuh"

namespace mb200 {

constexpr int kCumBlock = 256, kCumPer = 16, kCumTile = kCumBlock * kCumPer;  // 4096 rows per tile
constexpr int kCumCols = 32;

struct CumCols {
  const void* in[kCumCols];
  void* out[kCumCols];
};

template <typename T>
struct CumT;
template <>
struct CumT<double> {
  static __device__ __forceinline__ bool skip(double x) { return x != x; }
  template <int OP>
  static __device__ __forceinline__ double ident() {
    if (OP == MB200_CUM_SUM) return __longlong_as_double(0x8000000000000000LL);  // -0.0: x + -0.0 = x for every x
    if (OP == MB200_CUM_MAX) return __longlong_as_double(0xfff0000000000000LL);  // -inf
    if (OP == MB200_CUM_MIN) return __longlong_as_double(0x7ff0000000000000LL);  // +inf
    return __longlong_as_double(0x7ff8000000000000LL);                           // FFILL: NaN = "nothing valid yet"
  }
};
template <>
struct CumT<long long> {
  static __device__ __forceinline__ bool skip(long long) { return false; }
  template <int OP>
  static __device__ __forceinline__ long long ident() {
    if (OP == MB200_CUM_MAX) return LLONG_MIN;
    if (OP == MB200_CUM_MIN) return LLONG_MAX;
    return 0;
  }
};

// a (+) b with a covering EARLIER rows than b
template <int OP, typename T>
__device__ __forceinline__ T cum_comb(T a, T b) {
  if (OP == MB200_CUM_SUM) return a + b;
  // ties go to the later operand: pandas' cummax / cummin (numpy's maximum / minimum.accumulate) return the latest
  // of equal values, which tells -0.0 from 0.0
  if (OP == MB200_CUM_MAX) return b >= a ? b : a;
  if (OP == MB200_CUM_MIN) return b <= a ? b : a;
  return CumT<T>::skip(b) ? a : b;  // FFILL: the latest valid value
}

// the running value after a row: NaN rows leave max / min / forward fill as they were and add +0.0 to a sum.  pandas
// fills NaN with 0.0 and accumulates from the first row, so cumsum([-0.0]) = [-0.0] (hence the identity -0.0) but
// cumsum([NaN, -0.0]) = [NaN, +0.0]
template <int OP, typename T>
__device__ __forceinline__ T cum_step(T run, T v) {
  if (!CumT<T>::skip(v)) return cum_comb<OP, T>(run, v);
  return OP == MB200_CUM_SUM ? cum_comb<OP, T>(run, (T)0) : run;
}

__device__ __forceinline__ int cum_slot(int j) { return j + (j >> 4); }

// coalesced global -> padded shared tile; rows past the end read as the identity
template <typename T>
__device__ __forceinline__ void cum_load_tile(const T* __restrict__ x, long long base, long long n, T fill, T* tile) {
#pragma unroll
  for (int k = 0; k < kCumPer; ++k) {
    const int j = k * kCumBlock + threadIdx.x;
    const long long i = base + j;
    tile[cum_slot(j)] = i < n ? x[i] : fill;
  }
}

// ---- 1. tile -> aggregate ------------------------------------------------------------------------------------
template <typename T, int OP>
__global__ void __launch_bounds__(kCumBlock) cum_tile_reduce_kernel(const __grid_constant__ CumCols cols, long long n,
                                                                    long long ntiles, T* __restrict__ agg) {
  __shared__ T tile[kCumTile + kCumTile / kCumPer];
  __shared__ T warp_tot[kCumBlock / 32];
  const T id = CumT<T>::template ident<OP>();
  const T* x = static_cast<const T*>(cols.in[blockIdx.y]);
  cum_load_tile<T>(x, (long long)blockIdx.x * kCumTile, n, id, tile);
  __syncthreads();
  T acc = id;
  const int s0 = (int)threadIdx.x * (kCumPer + 1);  // cum_slot(16 t + k) = 17 t + k
#pragma unroll
  for (int k = 0; k < kCumPer; ++k) {
    acc = cum_step<OP, T>(acc, tile[s0 + k]);
  }
  // ordered tree: after the step with distance m, lane i holds rows of lanes [i, i + 2m)
#pragma unroll
  for (int m = 1; m < 32; m <<= 1) {
    const T y = __shfl_down_sync(0xffffffffu, acc, m);
    acc = cum_comb<OP, T>(acc, y);  // lanes whose partner is out of range hold garbage; only lane 0 is used
  }
  if ((threadIdx.x & 31) == 0) warp_tot[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    T t = warp_tot[0];
    for (int w = 1; w < kCumBlock / 32; ++w) t = cum_comb<OP, T>(t, warp_tot[w]);
    agg[(long long)blockIdx.y * ntiles + blockIdx.x] = t;
  }
}

// ---- 2. per column: exclusive scan of the tile aggregates (in place), column total ---------------------------------
template <typename T, int OP>
__global__ void __launch_bounds__(1024) cum_scan_tiles_kernel(T* __restrict__ agg, long long ntiles,
                                                              T* __restrict__ totals) {
  __shared__ T part[1024];
  const T id = CumT<T>::template ident<OP>();
  T* a = agg + (long long)blockIdx.x * ntiles;
  const int t = threadIdx.x;
  const long long per = (ntiles + 1023) / 1024;
  const long long lo = (long long)t * per;
  long long hi = lo + per;
  if (hi > ntiles) hi = ntiles;
  T s = id;
  for (long long i = lo; i < hi; ++i) s = cum_comb<OP, T>(s, a[i]);
  part[t] = s;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    const T v = t >= off ? part[t - off] : id;
    __syncthreads();
    part[t] = cum_comb<OP, T>(v, part[t]);
    __syncthreads();
  }
  T run = t ? part[t - 1] : id;
  for (long long i = lo; i < hi; ++i) {
    const T c = a[i];
    a[i] = run;
    run = cum_comb<OP, T>(run, c);
  }
  if (t == 1023 && totals) totals[blockIdx.x] = part[1023];
}

// ---- 3. tile + prefix -> output ------------------------------------------------------------------------------------
template <typename T, int OP>
__global__ void __launch_bounds__(kCumBlock) cum_tile_scan_kernel(const __grid_constant__ CumCols cols, long long n,
                                                                  long long ntiles, const T* __restrict__ prefix,
                                                                  const T* __restrict__ carry) {
  __shared__ T tile[kCumTile + kCumTile / kCumPer];
  __shared__ T warp_tot[kCumBlock / 32];
  const T id = CumT<T>::template ident<OP>();
  const T* x = static_cast<const T*>(cols.in[blockIdx.y]);
  T* out = static_cast<T*>(cols.out[blockIdx.y]);
  const long long base = (long long)blockIdx.x * kCumTile;
  cum_load_tile<T>(x, base, n, id, tile);
  __syncthreads();
  const int s0 = (int)threadIdx.x * (kCumPer + 1);
  T v[kCumPer];
  T tot = id;
#pragma unroll
  for (int k = 0; k < kCumPer; ++k) {
    v[k] = tile[s0 + k];
    tot = cum_step<OP, T>(tot, v[k]);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T incl = tot;
#pragma unroll
  for (int m = 1; m < 32; m <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, incl, m);
    if (lane >= m) incl = cum_comb<OP, T>(y, incl);
  }
  if (lane == 31) warp_tot[warp] = incl;
  const T prev = __shfl_up_sync(0xffffffffu, incl, 1);  // rows of this warp's earlier lanes
  __syncthreads();
  T run = prefix[(long long)blockIdx.y * ntiles + blockIdx.x];
  if (carry) run = cum_comb<OP, T>(carry[blockIdx.y], run);
  for (int w = 0; w < warp; ++w) run = cum_comb<OP, T>(run, warp_tot[w]);
  if (lane > 0) run = cum_comb<OP, T>(run, prev);
#pragma unroll
  for (int k = 0; k < kCumPer; ++k) {
    run = cum_step<OP, T>(run, v[k]);
    tile[s0 + k] = (CumT<T>::skip(v[k]) && OP != MB200_CUM_FFILL) ? v[k] : run;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kCumPer; ++k) {
    const int j = k * kCumBlock + threadIdx.x;
    const long long i = base + j;
    if (i < n) out[i] = tile[cum_slot(j)];
  }
}

// carry of rank r = totals of ranks 0 .. r-1 combined in rank order (one thread per column)
template <typename T, int OP>
__global__ void cum_carry_kernel(const T* __restrict__ gathered, int ncols, int rank, T* __restrict__ carry) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ncols) return;
  T run = CumT<T>::template ident<OP>();
  for (int r = 0; r < rank; ++r) run = cum_comb<OP, T>(run, gathered[(long long)r * ncols + c]);
  carry[c] = run;
}

inline int cum_launched(const char* name) {
  MB_LAUNCH_CHECK(name);
  return 0;
}

inline long long cum_ntiles(long long n) { return n < 1 ? 1 : (n + kCumTile - 1) / kCumTile; }

template <typename T, int OP>
int cum_partials_impl(int ncols, const void* const* in, long long n, T* agg, T* totals, cudaStream_t st) {
  const long long ntiles = cum_ntiles(n);
  for (int c0 = 0; c0 < ncols; c0 += kCumCols) {
    const int m = (ncols - c0) < kCumCols ? (ncols - c0) : kCumCols;
    CumCols cols;
    memset(&cols, 0, sizeof(cols));
    for (int j = 0; j < m; ++j) cols.in[j] = in[c0 + j];
    T* a = agg + (long long)c0 * ntiles;
    cum_tile_reduce_kernel<T, OP><<<dim3((unsigned)ntiles, (unsigned)m), kCumBlock, 0, st>>>(cols, n, ntiles, a);
    MB_LAUNCH_CHECK("cum_tile_reduce_kernel");
    cum_scan_tiles_kernel<T, OP><<<(unsigned)m, 1024, 0, st>>>(a, ntiles, totals ? totals + c0 : nullptr);
    MB_LAUNCH_CHECK("cum_scan_tiles_kernel");
  }
  return 0;
}

template <typename T, int OP>
int cum_apply_impl(int ncols, const void* const* in, void* const* out, long long n, const T* prefix, const T* carry,
                   cudaStream_t st) {
  const long long ntiles = cum_ntiles(n);
  for (int c0 = 0; c0 < ncols; c0 += kCumCols) {
    const int m = (ncols - c0) < kCumCols ? (ncols - c0) : kCumCols;
    CumCols cols;
    memset(&cols, 0, sizeof(cols));
    for (int j = 0; j < m; ++j) {
      cols.in[j] = in[c0 + j];
      cols.out[j] = out[c0 + j];
    }
    cum_tile_scan_kernel<T, OP><<<dim3((unsigned)ntiles, (unsigned)m), kCumBlock, 0, st>>>(
        cols, n, ntiles, prefix + (long long)c0 * ntiles, carry ? carry + c0 : nullptr);
    MB_LAUNCH_CHECK("cum_tile_scan_kernel");
  }
  return 0;
}

// op / dtype dispatch: CALL is a macro taking (T, OP)
#define MB_CUM_DISPATCH(op, dtype, CALL)                                                        \
  do {                                                                                          \
    if ((dtype) == MB200_F64) {                                                                 \
      switch (op) {                                                                             \
        case MB200_CUM_SUM: return CALL(double, MB200_CUM_SUM);                                 \
        case MB200_CUM_MAX: return CALL(double, MB200_CUM_MAX);                                 \
        case MB200_CUM_MIN: return CALL(double, MB200_CUM_MIN);                                 \
        case MB200_CUM_FFILL: return CALL(double, MB200_CUM_FFILL);                             \
      }                                                                                         \
    } else if ((dtype) == MB200_I64) {                                                          \
      switch (op) {                                                                             \
        case MB200_CUM_SUM: return CALL(long long, MB200_CUM_SUM);                              \
        case MB200_CUM_MAX: return CALL(long long, MB200_CUM_MAX);                              \
        case MB200_CUM_MIN: return CALL(long long, MB200_CUM_MIN);                              \
      }                                                                                         \
    }                                                                                           \
  } while (0)

}  // namespace mb200

using namespace mb200;

extern "C" size_t mb200_cum_scratch_bytes(int ncols, int64_t nrows) {
  if (ncols < 1) ncols = 1;
  return (size_t)ncols * (size_t)cum_ntiles(nrows) * 8 + 256;
}

static int cum_check(const char* what, int op, int dtype, int ncols, const void* const* in, int64_t nrows) {
  if (ncols < 0 || nrows < 0) return fail(what, "negative size");
  if (dtype != MB200_F64 && dtype != MB200_I64) return fail(what, "dtype must be MB200_F64 or MB200_I64");
  if (op < MB200_CUM_SUM || op > MB200_CUM_FFILL || (op == MB200_CUM_FFILL && dtype != MB200_F64))
    return fail(what, "op must be MB200_CUM_SUM / MAX / MIN (or FFILL on float64)");
  if (ncols > 0 && nrows > 0) {
    if (!in) return fail(what, "null column array");
    for (int j = 0; j < ncols; ++j)
      if (!in[j] || ((uintptr_t)in[j] & 7u)) return fail(what, "null or misaligned column");
  }
  return 0;
}

extern "C" int mb200_cum_partials(int op, int dtype, int ncols, const void* const* in, int64_t nrows, void* scratch,
                                  size_t scratch_bytes, void* totals_dev, mb200_stream_t stream) {
  if (int rc = cum_check("mb200_cum_partials", op, dtype, ncols, in, nrows)) return rc;
  if (ncols == 0) return 0;
  if (!scratch || scratch_bytes < mb200_cum_scratch_bytes(ncols, nrows))
    return fail("mb200_cum_partials", "scratch missing or too small");
  DevProps dp;
  if (int rc = dev_props(&dp)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (nrows == 0) {
    // one tile of nothing per column: the aggregates are the identity; run the kernels on an empty range so the
    // totals still come out (the input pointers are never dereferenced: every row index is past the end)
    static const void* const none[kCumCols] = {};
    if (ncols > kCumCols) return fail("mb200_cum_partials", "empty block with more than 32 columns");
    in = none;
  }
#define MB_CUM_PARTIALS(T, OP) cum_partials_impl<T, OP>(ncols, in, nrows, static_cast<T*>(scratch), static_cast<T*>(totals_dev), st)
  MB_CUM_DISPATCH(op, dtype, MB_CUM_PARTIALS);
#undef MB_CUM_PARTIALS
  return fail("mb200_cum_partials", "unsupported op / dtype");
}

extern "C" int mb200_cum_apply(int op, int dtype, int ncols, const void* const* in, void* const* out, int64_t nrows,
                               const void* scratch, const void* carry_dev, mb200_stream_t stream) {
  if (int rc = cum_check("mb200_cum_apply", op, dtype, ncols, in, nrows)) return rc;
  if (ncols == 0 || nrows == 0) return 0;
  if (!scratch || !out) return fail("mb200_cum_apply", "null argument");
  for (int j = 0; j < ncols; ++j)
    if (!out[j] || ((uintptr_t)out[j] & 7u)) return fail("mb200_cum_apply", "null or misaligned output column");
  DevProps dp;
  if (int rc = dev_props(&dp)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
#define MB_CUM_APPLY(T, OP) cum_apply_impl<T, OP>(ncols, in, out, nrows, static_cast<const T*>(scratch), static_cast<const T*>(carry_dev), st)
  MB_CUM_DISPATCH(op, dtype, MB_CUM_APPLY);
#undef MB_CUM_APPLY
  return fail("mb200_cum_apply", "unsupported op / dtype");
}

extern "C" int mb200_cum_carry(int op, int dtype, int ncols, const void* gathered_totals_dev, int rank, void* carry_dev,
                               mb200_stream_t stream) {
  if (ncols < 0 || rank < 0) return fail("mb200_cum_carry", "negative size");
  if (ncols == 0) return 0;
  if (!carry_dev || (rank > 0 && !gathered_totals_dev)) return fail("mb200_cum_carry", "null argument");
  DevProps dp;
  if (int rc = dev_props(&dp)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned g = (unsigned)((ncols + 127) / 128);
#define MB_CUM_CARRY(T, OP)                                                                                         \
  (cum_carry_kernel<T, OP><<<g, 128, 0, st>>>(static_cast<const T*>(gathered_totals_dev), ncols, rank,              \
                                              static_cast<T*>(carry_dev)),                                          \
   cum_launched("cum_carry_kernel"))
  MB_CUM_DISPATCH(op, dtype, MB_CUM_CARRY);
#undef MB_CUM_CARRY
  return fail("mb200_cum_carry", "unsupported op / dtype");
}
