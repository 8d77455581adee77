// reduce.cu — TreeReduce map phase: column-wise sum / count / min / max of one block.
//
// Replaces per-block `pandas.DataFrame.sum/count/min/max(axis=0, skipna=...)` called from
// PandasDataframe.tree_reduce (df.py:2208-2250) through TreeReduce.register (qc.py:976-1096);
// pandas computes these with nanops.nansum etc. (NaN -> 0 fill, numpy pairwise summation).
//
// Layout: grid = (ctas_per_col, ncols); CTA (x, c) owns row tiles x, x+gridDim.x, ... of
// column c (fixed map => deterministic result).  Two variants:
//   variant 0: 6-stage ring of 16 KiB shared-memory tiles filled by 1-D TMA bulk copies
//       (cp.async.bulk + mbarrier complete_tx; UBLKCP in SASS) issued by a dedicated producer
//       warp, consumed by 8 warps with conflict-free 128-bit LDS, warp-shuffle + shared-memory
//       block reduction;
//   variant 1: direct 128-bit streaming loads (LDG.E.128), same reduction tree.
// Per-thread float sums are Kahan-compensated (error O(eps)*sum|x| independent of n; the
// compensation is dropped while the running sum is not finite, so +-inf inputs and sums that
// overflow to +-inf behave like pandas/numpy).
// Stage 2 (reduce_finalize) combines the per-CTA partials in fixed order.
// Algorithmic traffic: 8 B read per element; output ncols * 16 B.
#include <math.h>
#include <type_traits>

#include "common.cuh"

namespace mb200 {

constexpr int kRThreads = 256;
constexpr int kMaxCtasPerCol = 2048;
// TMA ring
constexpr int kStages = 6;
constexpr int kTmaTileElems = 2048;  // 16 KiB
constexpr int kTmaTileBytes = kTmaTileElems * 8;
// direct-load variant
constexpr int kLdgUnroll = 4;
constexpr int kLdgTile = kRThreads * kLdgUnroll * 4;

struct RedParams {
  const void* in[MB200_MAX_COLS];
  int ncols;
  long long nrows;
  int skipna;
  void* part_val;       // [ncols][gridDim.x]
  long long* part_cnt;  // [ncols][gridDim.x]
  const double* centers;  // SSD only: per-column centre (device array [ncols])
};

// ---------------------------------------------------------------- accumulators
template <int OP, typename T>
struct Acc;

template <>
struct Acc<MB200_RED_SUM, double> {
  double s = 0.0, c = 0.0;
  long long n = 0;
  __device__ __forceinline__ void add(double x, int skipna) {
    const bool ok = (x == x);
    n += ok;
    const double v = (ok || !skipna) ? x : 0.0;
    const double y = v - c;
    const double t = s + y;
    // a running sum that is +-inf (an inf input, or overflow) or NaN carries no compensation: (t - s) - y would be
    // inf or NaN, and value() = s - c would turn an overflowed sum into inf - inf = NaN
    c = isfinite(t) ? (t - s) - y : 0.0;
    s = t;
  }
  __device__ __forceinline__ void merge(const Acc& o) {
    add_raw(o.s);
    add_raw(-o.c);
    n += o.n;
  }
  __device__ __forceinline__ void add_raw(double v) {
    const double y = v - c;
    const double t = s + y;
    c = isfinite(t) ? (t - s) - y : 0.0;
    s = t;
  }
  __device__ __forceinline__ double value() const { return s - c; }
  static __device__ __forceinline__ double combine(double a, double b) { return a + b; }
};
// Sum of squared deviations from a per-column centre: the second pass of pandas' two-pass variance
// (nanops.nanvar: avg = sum / count; sqr = (avg - values) ** 2; NaNs dropped; result = sqr.sum() / (count - ddof)).
// One rounding for the difference, one for the square, compensated summation like SUM.  skipna drops the rows whose
// VALUE is NaN, not the deviations that are: a column holding inf has centre inf and inf - inf = NaN, and pandas'
// variance of it is NaN.
template <>
struct Acc<MB200_RED_SSD, double> : Acc<MB200_RED_SUM, double> {
  double center = 0.0;
  __device__ __forceinline__ void add(double x, int skipna) {
    const double d = __dsub_rn(center, x);
    const bool nan = x != x;
    Acc<MB200_RED_SUM, double>::add(nan ? x : __dmul_rn(d, d), nan ? skipna : 0);
  }
};
template <>
struct Acc<MB200_RED_SUM, long long> {
  unsigned long long s = 0;
  long long n = 0;
  __device__ __forceinline__ void add(long long x, int) {
    s += (unsigned long long)x;
    n += 1;
  }
  __device__ __forceinline__ void merge(const Acc& o) {
    s += o.s;
    n += o.n;
  }
  __device__ __forceinline__ long long value() const { return (long long)s; }
  static __device__ __forceinline__ long long combine(long long a, long long b) {
    return (long long)((unsigned long long)a + (unsigned long long)b);
  }
};
template <>
struct Acc<MB200_RED_MIN, double> {
  double m = (double)INFINITY;
  long long n = 0;
  __device__ __forceinline__ void add(double x, int) {
    n += (x == x);
    m = fmin(m, x);  // fmin ignores NaN operands
  }
  __device__ __forceinline__ void merge(const Acc& o) {
    m = fmin(m, o.m);
    n += o.n;
  }
  __device__ __forceinline__ double value() const { return m; }
  static __device__ __forceinline__ double combine(double a, double b) { return fmin(a, b); }
};
template <>
struct Acc<MB200_RED_MAX, double> {
  double m = -(double)INFINITY;
  long long n = 0;
  __device__ __forceinline__ void add(double x, int) {
    n += (x == x);
    m = fmax(m, x);
  }
  __device__ __forceinline__ void merge(const Acc& o) {
    m = fmax(m, o.m);
    n += o.n;
  }
  __device__ __forceinline__ double value() const { return m; }
  static __device__ __forceinline__ double combine(double a, double b) { return fmax(a, b); }
};
template <>
struct Acc<MB200_RED_MIN, long long> {
  long long m = 0x7fffffffffffffffLL;
  long long n = 0;
  __device__ __forceinline__ void add(long long x, int) {
    m = x < m ? x : m;
    n += 1;
  }
  __device__ __forceinline__ void merge(const Acc& o) {
    m = o.m < m ? o.m : m;
    n += o.n;
  }
  __device__ __forceinline__ long long value() const { return m; }
  static __device__ __forceinline__ long long combine(long long a, long long b) { return a < b ? a : b; }
};
template <>
struct Acc<MB200_RED_MAX, long long> {
  long long m = (long long)0x8000000000000000ULL;
  long long n = 0;
  __device__ __forceinline__ void add(long long x, int) {
    m = x > m ? x : m;
    n += 1;
  }
  __device__ __forceinline__ void merge(const Acc& o) {
    m = o.m > m ? o.m : m;
    n += o.n;
  }
  __device__ __forceinline__ long long value() const { return m; }
  static __device__ __forceinline__ long long combine(long long a, long long b) { return a > b ? a : b; }
};
template <>
struct Acc<MB200_RED_PROD, double> {
  double m = 1.0;
  long long n = 0;
  __device__ __forceinline__ void add(double x, int skipna) {
    const bool ok = (x == x);
    n += ok;
    m *= (ok || !skipna) ? x : 1.0;
  }
  __device__ __forceinline__ void merge(const Acc& o) {
    m *= o.m;
    n += o.n;
  }
  __device__ __forceinline__ double value() const { return m; }
  static __device__ __forceinline__ double combine(double a, double b) { return a * b; }
};
template <>
struct Acc<MB200_RED_PROD, long long> {
  unsigned long long m = 1;
  long long n = 0;
  __device__ __forceinline__ void add(long long x, int) {
    m *= (unsigned long long)x;
    n += 1;
  }
  __device__ __forceinline__ void merge(const Acc& o) {
    m *= o.m;
    n += o.n;
  }
  __device__ __forceinline__ long long value() const { return (long long)m; }
  static __device__ __forceinline__ long long combine(long long a, long long b) {
    return (long long)((unsigned long long)a * (unsigned long long)b);
  }
};
template <>
struct Acc<MB200_RED_COUNT, double> {
  long long n = 0;
  __device__ __forceinline__ void add(double x, int) { n += (x == x); }
  __device__ __forceinline__ void merge(const Acc& o) { n += o.n; }
  __device__ __forceinline__ double value() const { return 0.0; }
  static __device__ __forceinline__ double combine(double a, double) { return a; }
};
template <>
struct Acc<MB200_RED_COUNT, long long> {
  long long n = 0;
  __device__ __forceinline__ void add(long long, int) { n += 1; }
  __device__ __forceinline__ void merge(const Acc& o) { n += o.n; }
  __device__ __forceinline__ long long value() const { return 0; }
  static __device__ __forceinline__ long long combine(long long a, long long) { return a; }
};

template <typename T>
__device__ __forceinline__ T shfl_xor(T v, int m) {
  return __shfl_xor_sync(0xffffffffu, v, m);
}

// block-wide combine of (value, count); result valid in thread 0.  Fixed tree => deterministic.
// Works for any block of <= 32 warps (the TMA variant carries a 9th, producer-only warp that
// contributes the identity).
template <int OP, typename T>
__device__ __forceinline__ void block_combine(T& val, long long& cnt) {
  __shared__ T s_val[32];
  __shared__ long long s_cnt[32];
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    val = Acc<OP, T>::combine(val, shfl_xor(val, m));
    cnt += shfl_xor(cnt, m);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nw = (blockDim.x + 31) >> 5;
  if (lane == 0) {
    s_val[warp] = val;
    s_cnt[warp] = cnt;
  }
  __syncthreads();
  if (warp == 0) {
    Acc<OP, T> ident;
    T v = lane < nw ? s_val[lane] : ident.value();
    long long n = lane < nw ? s_cnt[lane] : 0;
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) {
      v = Acc<OP, T>::combine(v, shfl_xor(v, m));
      n += shfl_xor(n, m);
    }
    val = v;
    cnt = n;
  }
}

template <int OP, typename T>
__device__ __forceinline__ void write_partial(const RedParams& p, T val, long long cnt) {
  if (threadIdx.x == 0) {
    const size_t idx = (size_t)blockIdx.y * gridDim.x + blockIdx.x;
    static_cast<T*>(p.part_val)[idx] = val;
    p.part_cnt[idx] = cnt;
  }
}

// ---------------------------------------------------------------- variant 1: direct LDG.256
template <int OP, typename T, bool VEC>
__global__ void __launch_bounds__(kRThreads) reduce_ldg_kernel(const __grid_constant__ RedParams p) {
  const T* __restrict__ a = static_cast<const T*>(p.in[blockIdx.y]);
  const long long n = p.nrows;
  const long long ntiles = (n + kLdgTile - 1) / kLdgTile;
  const int tid = threadIdx.x;
  Acc<OP, T> acc[4];
  if constexpr (OP == MB200_RED_SSD) {
    const double c = p.centers[blockIdx.y];
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i].center = c;
  }
  for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const long long base = t * kLdgTile;
    if (VEC && base + kLdgTile <= n) {
      if constexpr (std::is_same<T, double>::value) {
        f64x4 v[kLdgUnroll];
#pragma unroll
        for (int u = 0; u < kLdgUnroll; ++u) v[u] = ldg_stream_f64x4(a + base + (long long)(u * kRThreads + tid) * 4);
#pragma unroll
        for (int u = 0; u < kLdgUnroll; ++u) {
          acc[0].add(v[u].x, p.skipna);
          acc[1].add(v[u].y, p.skipna);
          acc[2].add(v[u].z, p.skipna);
          acc[3].add(v[u].w, p.skipna);
        }
      } else {
        i64x4 v[kLdgUnroll];
#pragma unroll
        for (int u = 0; u < kLdgUnroll; ++u) v[u] = ldg_stream_i64x4(a + base + (long long)(u * kRThreads + tid) * 4);
#pragma unroll
        for (int u = 0; u < kLdgUnroll; ++u) {
          acc[0].add(v[u].x, p.skipna);
          acc[1].add(v[u].y, p.skipna);
          acc[2].add(v[u].z, p.skipna);
          acc[3].add(v[u].w, p.skipna);
        }
      }
    } else {
      const long long end = (base + kLdgTile < n) ? base + kLdgTile : n;
      for (long long i = base + tid; i < end; i += kRThreads) acc[0].add(a[i], p.skipna);
    }
  }
  acc[0].merge(acc[1]);
  acc[2].merge(acc[3]);
  acc[0].merge(acc[2]);
  T val = acc[0].value();
  long long cnt = acc[0].n;
  block_combine<OP, T>(val, cnt);
  write_partial<OP, T>(p, val, cnt);
}

// ---------------------------------------------------------------- variant 0: TMA-staged tiles
// Warp-specialised: warps 0..7 consume, warp 8 (one elected lane) is the TMA producer.  A ring of
// kStages 16 KiB tiles with a full[] (TMA complete_tx) and an empty[] (one arrive per consumer
// warp) mbarrier per stage lets the producer run kStages tiles ahead without any block-wide sync.
constexpr int kTmaThreads = kRThreads + 32;
constexpr int kConsumerWarps = kRThreads / 32;

template <int OP, typename T>
__global__ void __launch_bounds__(kTmaThreads) reduce_tma_kernel(const __grid_constant__ RedParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T* tiles = reinterpret_cast<T*>(smem_raw);  // kStages x 16 KiB
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + kStages * kTmaTileBytes);
  uint64_t* empty = full + kStages;

  const T* __restrict__ a = static_cast<const T*>(p.in[blockIdx.y]);
  const long long n = p.nrows;
  const long long ntiles = (n + kTmaTileElems - 1) / kTmaTileElems;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  // tiles owned by this CTA: blockIdx.x + k * gridDim.x
  const long long first = blockIdx.x;
  const long long nmine = first < ntiles ? (ntiles - first + gridDim.x - 1) / gridDim.x : 0;

  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kConsumerWarps);
    }
    mbar_fence_init();
  }
  __syncthreads();

  auto tile_elems = [&](long long k) -> int {
    const long long base = (first + k * gridDim.x) * kTmaTileElems;
    const long long rem = n - base;
    return rem >= kTmaTileElems ? kTmaTileElems : (int)rem;
  };

  Acc<OP, T> acc[4];
  if constexpr (OP == MB200_RED_SSD) {
    const double c = p.centers[blockIdx.y];
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i].center = c;
  }
  if (warp == kConsumerWarps) {
    // ---------------- producer warp
    if (lane == 0) {
      const uint64_t policy = l2_policy_evict_first();
      for (long long k = 0; k < nmine; ++k) {
        const int s = (int)(k % kStages);
        if (k >= kStages) mbar_wait(&empty[s], (uint32_t)(((k / kStages) - 1) & 1));
        const long long base = (first + k * gridDim.x) * kTmaTileElems;
        // elements that arrive through the bulk copy: even count (16-byte granularity)
        const uint32_t bytes = (uint32_t)((tile_elems(k) & ~1) * 8);
        mbar_expect_tx(&full[s], bytes);
        if (bytes) tma_bulk_g2s(tiles + (size_t)s * kTmaTileElems, a + base, bytes, &full[s], policy);
      }
    }
  } else {
    // ---------------- consumer warps
    for (long long k = 0; k < nmine; ++k) {
      const int s = (int)(k % kStages);
      mbar_wait(&full[s], (uint32_t)((k / kStages) & 1));
      const T* tile = tiles + (size_t)s * kTmaTileElems;
      const int ne = tile_elems(k);
      if (ne == kTmaTileElems) {
#pragma unroll
        for (int j = 0; j < kTmaTileElems / (2 * kRThreads); ++j) {
          const int e = (j * kRThreads + tid) * 2;
          if constexpr (std::is_same<T, double>::value) {
            const double2 v = *reinterpret_cast<const double2*>(tile + e);
            acc[(2 * j) & 3].add(v.x, p.skipna);
            acc[(2 * j + 1) & 3].add(v.y, p.skipna);
          } else {
            const longlong2 v = *reinterpret_cast<const longlong2*>(tile + e);
            acc[(2 * j) & 3].add(v.x, p.skipna);
            acc[(2 * j + 1) & 3].add(v.y, p.skipna);
          }
        }
      } else {
        const int ne_even = ne & ~1;
        for (int e = tid; e < ne_even; e += kRThreads) acc[0].add(tile[e], p.skipna);
        if ((ne & 1) && tid == 0) {  // odd tail element never went through the 16-byte bulk copy
          const long long base = (first + k * gridDim.x) * kTmaTileElems;
          acc[1].add(a[base + ne - 1], p.skipna);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);  // this warp is done reading stage s
    }
  }
  acc[0].merge(acc[1]);
  acc[2].merge(acc[3]);
  acc[0].merge(acc[2]);
  T val = acc[0].value();
  long long cnt = acc[0].n;
  block_combine<OP, T>(val, cnt);
  write_partial<OP, T>(p, val, cnt);
}

// ---------------------------------------------------------------- stage 2
// One warp per column: lane-strided fixed-order pass over the per-CTA partials, then shuffle tree.
template <int OP, typename T>
__global__ void reduce_finalize_kernel(const void* part_val, const long long* part_cnt, int nparts,
                                       long long nrows, int skipna, void* out_val, long long* out_cnt) {
  const int col = blockIdx.x;
  const int lane = threadIdx.x;
  const T* pv = static_cast<const T*>(part_val) + (size_t)col * nparts;
  const long long* pc = part_cnt + (size_t)col * nparts;
  Acc<OP, T> ident;
  T v = ident.value();
  long long n = 0;
  if constexpr ((OP == MB200_RED_SUM || OP == MB200_RED_SSD) && std::is_same<T, double>::value) {
    // compensated combine of the CTA partials
    Acc<MB200_RED_SUM, double> a;
    for (int i = lane; i < nparts; i += 32) {
      a.add_raw(pv[i]);
      n += pc[i];
    }
    v = a.value();
  } else {
    for (int i = lane; i < nparts; i += 32) {
      v = Acc<OP, T>::combine(v, pv[i]);
      n += pc[i];
    }
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    v = Acc<OP, T>::combine(v, shfl_xor(v, m));
    n += shfl_xor(n, m);
  }
  if (lane == 0) {
    if constexpr (std::is_same<T, double>::value && (OP == MB200_RED_MIN || OP == MB200_RED_MAX)) {
      // pandas: all-NaN column -> NaN; skipna=False with any NaN -> NaN
      if (n == 0 || (!skipna && n < nrows)) v = __longlong_as_double(0x7ff8000000000000LL);
    }
    if (out_val && OP != MB200_RED_COUNT) static_cast<T*>(out_val)[col] = v;
    if (out_cnt) out_cnt[col] = n;
  }
}

template <int OP, typename T>
static int run_reduce(const RedParams& p0, int variant, void* out_val, long long* out_cnt, void* scratch,
                      cudaStream_t st) {
  DevProps dp;
  if (int rc = dev_props(&dp)) return rc;
  RedParams p = p0;
  bool a32 = true, a16 = true;
  for (int c = 0; c < p.ncols; ++c) {
    a32 = a32 && aligned32(p.in[c]);
    a16 = a16 && aligned16(p.in[c]);
  }
  if (variant == 0 && !a16) variant = 1;  // bulk copies need 16-byte aligned sources

  const size_t smem = (size_t)kStages * kTmaTileBytes + 2 * kStages * sizeof(uint64_t);
  int occ = 0;
  long long ntiles;
  if (variant == 0) {
    MB_CUDA(cudaFuncSetAttribute(reduce_tma_kernel<OP, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    MB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, reduce_tma_kernel<OP, T>, kTmaThreads, smem));
    ntiles = (p.nrows + kTmaTileElems - 1) / kTmaTileElems;
  } else {
    MB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, reduce_ldg_kernel<OP, T, true>, kRThreads, 0));
    ntiles = (p.nrows + kLdgTile - 1) / kLdgTile;
  }
  if (occ < 1) occ = 1;
  // resident CTAs are shared between the columns; every column gets the same count
  long long per_col = ((long long)dp.sm_count * occ + p.ncols - 1) / p.ncols;
  if (per_col > ntiles) per_col = ntiles;
  if (per_col > kMaxCtasPerCol) per_col = kMaxCtasPerCol;
  if (per_col < 1) per_col = 1;

  p.part_val = scratch;
  p.part_cnt = reinterpret_cast<long long*>(static_cast<char*>(scratch) +
                                            (size_t)MB200_MAX_COLS * kMaxCtasPerCol * 8);
  dim3 grid((unsigned)per_col, (unsigned)p.ncols);
  if (variant == 0) {
    reduce_tma_kernel<OP, T><<<grid, kTmaThreads, smem, st>>>(p);
    MB_LAUNCH_CHECK("reduce_tma_kernel");
  } else {
    if (a32)
      reduce_ldg_kernel<OP, T, true><<<grid, kRThreads, 0, st>>>(p);
    else
      reduce_ldg_kernel<OP, T, false><<<grid, kRThreads, 0, st>>>(p);
    MB_LAUNCH_CHECK("reduce_ldg_kernel");
  }
  reduce_finalize_kernel<OP, T><<<p.ncols, 32, 0, st>>>(p.part_val, p.part_cnt, (int)per_col, p.nrows, p.skipna,
                                                        out_val, out_cnt);
  MB_LAUNCH_CHECK("reduce_finalize_kernel");
  return 0;
}

}  // namespace mb200

using namespace mb200;

extern "C" size_t mb200_reduce_scratch_bytes(int ncols) {
  (void)ncols;
  return (size_t)MB200_MAX_COLS * kMaxCtasPerCol * 16;
}

static int reduce_columns_impl(int op, int dtype, int ncols, const void* const* in, int64_t nrows, int skipna,
                               const double* centers_dev, void* out_val, int64_t* out_cnt, void* scratch, int variant,
                               mb200_stream_t stream);

extern "C" int mb200_reduce_columns(int op, int dtype, int ncols, const void* const* in, int64_t nrows,
                                    int skipna, void* out_val, int64_t* out_cnt, void* scratch, int variant,
                                    mb200_stream_t stream) {
  if (op == MB200_RED_SSD) return fail("mb200_reduce_columns", "MB200_RED_SSD needs mb200_reduce_columns_centered");
  return reduce_columns_impl(op, dtype, ncols, in, nrows, skipna, nullptr, out_val, out_cnt, scratch, variant, stream);
}

extern "C" int mb200_reduce_columns_centered(int op, int dtype, int ncols, const void* const* in, int64_t nrows,
                                             int skipna, const double* centers_dev, void* out_val, int64_t* out_cnt,
                                             void* scratch, int variant, mb200_stream_t stream) {
  if (op != MB200_RED_SSD || dtype != MB200_F64)
    return fail("mb200_reduce_columns_centered", "only MB200_RED_SSD over float64 columns takes centres");
  if (!centers_dev && ncols > 0) return fail("mb200_reduce_columns_centered", "null centres");
  return reduce_columns_impl(op, dtype, ncols, in, nrows, skipna, centers_dev, out_val, out_cnt, scratch, variant,
                             stream);
}

static int reduce_columns_impl(int op, int dtype, int ncols, const void* const* in, int64_t nrows, int skipna,
                               const double* centers_dev, void* out_val, int64_t* out_cnt, void* scratch, int variant,
                               mb200_stream_t stream) {
  if (ncols < 0 || ncols > MB200_MAX_COLS) return fail("mb200_reduce_columns", "ncols out of range (0..32)");
  if (nrows < 0) return fail("mb200_reduce_columns", "negative nrows");
  if (ncols == 0) return 0;
  if (!in || !scratch) return fail("mb200_reduce_columns", "null argument");
  RedParams p;
  memset(&p, 0, sizeof(p));
  for (int c = 0; c < ncols; ++c) {
    if (!in[c] && nrows > 0) return fail("mb200_reduce_columns", "null column pointer");
    p.in[c] = in[c];
  }
  p.ncols = ncols;
  p.nrows = nrows;
  p.skipna = skipna ? 1 : 0;
  p.centers = centers_dev;
  cudaStream_t st = (cudaStream_t)stream;
  long long* oc = reinterpret_cast<long long*>(out_cnt);
#define MB_RED(OPC, T) return run_reduce<OPC, T>(p, variant, out_val, oc, scratch, st);
  if (dtype == MB200_F64) {
    switch (op) {
      case MB200_RED_SUM: MB_RED(MB200_RED_SUM, double)
      case MB200_RED_MIN: MB_RED(MB200_RED_MIN, double)
      case MB200_RED_MAX: MB_RED(MB200_RED_MAX, double)
      case MB200_RED_COUNT: MB_RED(MB200_RED_COUNT, double)
      case MB200_RED_PROD: MB_RED(MB200_RED_PROD, double)
      case MB200_RED_SSD: MB_RED(MB200_RED_SSD, double)
    }
  } else if (dtype == MB200_I64) {
    switch (op) {
      case MB200_RED_SUM: MB_RED(MB200_RED_SUM, long long)
      case MB200_RED_MIN: MB_RED(MB200_RED_MIN, long long)
      case MB200_RED_MAX: MB_RED(MB200_RED_MAX, long long)
      case MB200_RED_COUNT: MB_RED(MB200_RED_COUNT, long long)
      case MB200_RED_PROD: MB_RED(MB200_RED_PROD, long long)
    }
  }
#undef MB_RED
  return fail("mb200_reduce_columns", "unsupported op/dtype");
}
