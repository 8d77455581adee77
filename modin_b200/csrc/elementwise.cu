// elementwise.cu — Map / Binary operator templates as coalesced 128-bit column sweeps.
//
// One launch covers every column of a block (Modin partition): one CTA per (4096-row tile, column).
// The tile is 8 slabs of 512 rows; in each slab thread t moves rows 2t and 2t + 1 with one access
// per operand (LDG.E.128 / STG.E.128 for 8-byte types, 16-bit for bool columns), so every warp
// instruction covers whole contiguous sectors.  All loads of a tile are issued before the first
// store (L1 bypass, L2 evict-first).  The path is HBM-bound: algorithmic traffic is 8 B read per
// operand element + 8 B written (1 B for predicates).
//
// pandas semantics restated here (reference call sites):
//   abs/neg/isna/notna  Map.register(pandas.DataFrame.abs ...)   qc.py:2036, 2063-2106
//   fillna(scalar)      qc.fillna -> frame.map                    qc.py:2710-2813
//   a OP b, a OP s      Binary.register(pandas.DataFrame.add ...) qc.py:535-624
//   a*b+c               two Binary passes in the reference (alg/binary.py:420-430) -- fused here
//                       but with TWO IEEE roundings (__dmul_rn then __dadd_rn), never an FMA,
//                       so results are bit-identical to pandas.
#include <type_traits>

#include "common.cuh"

namespace mb200 {

constexpr int kThreads = 256;
constexpr int kPair = 2;                  // elements per thread and access
constexpr int kSlab = kThreads * kPair;   // 512 elements
constexpr int kSlabs = 8;
constexpr int kTile = kSlab * kSlabs;     // 4096 elements = 32 KiB of f64 per operand

struct MapParams {
  const void* in0[MB200_MAX_COLS];
  const void* in1[MB200_MAX_COLS];
  const void* in2[MB200_MAX_COLS];
  void* out[MB200_MAX_COLS];
  uint64_t s0[MB200_MAX_COLS];
  uint64_t s1[MB200_MAX_COLS];
  long long nrows;
};

template <typename T>
__device__ __forceinline__ T from_bits(uint64_t b);
template <>
__device__ __forceinline__ double from_bits<double>(uint64_t b) {
  return __longlong_as_double((long long)b);
}
template <>
__device__ __forceinline__ long long from_bits<long long>(uint64_t b) {
  return (long long)b;
}
template <>
__device__ __forceinline__ uint8_t from_bits<uint8_t>(uint64_t b) {
  return (uint8_t)(b != 0);
}

constexpr __host__ __device__ int op_nin(int op) { return op >= 64 ? 3 : (op >= 32 ? 2 : 1); }
constexpr __host__ __device__ bool op_is_pred(int op) {
  return op == MB200_OP_ISNA || op == MB200_OP_NOTNA || (op >= MB200_OP_EQ_S && op <= MB200_OP_GE_S) ||
         (op >= MB200_OP_EQ && op <= MB200_OP_GE);
}

// ---- the arithmetic.  TI in {double, long long}; TO in {double, long long, uint8_t}.
template <int OP, typename TI, typename TO>
__device__ __forceinline__ TO apply(TI a, TI b, TI c, TI s0, TI s1) {
  constexpr bool F = std::is_same<TI, double>::value;  // floating input?
  if constexpr (OP == MB200_OP_ABS) {
    if constexpr (F) return (TO)fabs(a);
    else return (TO)(a < 0 ? (TI)(0ULL - (unsigned long long)a) : a);
  } else if constexpr (OP == MB200_OP_NEG) {
    // sign-bit flip (like numpy/x86 xorpd): `-a` as arithmetic would not flip the sign of a NaN
    if constexpr (F) return (TO)__longlong_as_double(__double_as_longlong(a) ^ (long long)0x8000000000000000ULL);
    else return (TO)(TI)(0ULL - (unsigned long long)a);
  } else if constexpr (OP == MB200_OP_ISNA) {
    return (TO)(a != a);
  } else if constexpr (OP == MB200_OP_NOTNA) {
    return (TO)(a == a);
  } else if constexpr (OP == MB200_OP_FILLNA_S) {
    return (TO)((a != a) ? s0 : a);
  } else if constexpr (OP == MB200_OP_AFFINE) {
    if constexpr (F) return (TO)__dadd_rn(__dmul_rn(a, s0), s1);
    else return (TO)(TI)((unsigned long long)a * (unsigned long long)s0 + (unsigned long long)s1);
  } else if constexpr (OP == MB200_OP_ADD_S || OP == MB200_OP_ADD) {
    TI r = (OP == MB200_OP_ADD) ? b : s0;
    if constexpr (F) return (TO)__dadd_rn(a, r);
    else return (TO)(TI)((unsigned long long)a + (unsigned long long)r);
  } else if constexpr (OP == MB200_OP_SUB_S || OP == MB200_OP_SUB) {
    TI r = (OP == MB200_OP_SUB) ? b : s0;
    if constexpr (F) return (TO)__dsub_rn(a, r);
    else return (TO)(TI)((unsigned long long)a - (unsigned long long)r);
  } else if constexpr (OP == MB200_OP_RSUB_S) {
    if constexpr (F) return (TO)__dsub_rn(s0, a);
    else return (TO)(TI)((unsigned long long)s0 - (unsigned long long)a);
  } else if constexpr (OP == MB200_OP_MUL_S || OP == MB200_OP_MUL) {
    TI r = (OP == MB200_OP_MUL) ? b : s0;
    if constexpr (F) return (TO)__dmul_rn(a, r);
    else return (TO)(TI)((unsigned long long)a * (unsigned long long)r);
  } else if constexpr (OP == MB200_OP_DIV_S || OP == MB200_OP_DIV) {
    TI r = (OP == MB200_OP_DIV) ? b : s0;
    return (TO)__ddiv_rn((double)a, (double)r);  // true division: int64 inputs promote to f64
  } else if constexpr (OP == MB200_OP_RDIV_S) {
    return (TO)__ddiv_rn((double)s0, (double)a);
  } else if constexpr (OP == MB200_OP_EQ_S || OP == MB200_OP_EQ) {
    return (TO)(a == ((OP == MB200_OP_EQ) ? b : s0));
  } else if constexpr (OP == MB200_OP_NE_S || OP == MB200_OP_NE) {
    return (TO)(a != ((OP == MB200_OP_NE) ? b : s0));
  } else if constexpr (OP == MB200_OP_LT_S || OP == MB200_OP_LT) {
    return (TO)(a < ((OP == MB200_OP_LT) ? b : s0));
  } else if constexpr (OP == MB200_OP_LE_S || OP == MB200_OP_LE) {
    return (TO)(a <= ((OP == MB200_OP_LE) ? b : s0));
  } else if constexpr (OP == MB200_OP_GT_S || OP == MB200_OP_GT) {
    return (TO)(a > ((OP == MB200_OP_GT) ? b : s0));
  } else if constexpr (OP == MB200_OP_GE_S || OP == MB200_OP_GE) {
    return (TO)(a >= ((OP == MB200_OP_GE) ? b : s0));
  } else if constexpr (OP == MB200_OP_CLIP_S) {
    // pandas clip = where(x >= lower, lower) / where(x <= upper, upper) with NaN kept: comparisons, not
    // fmin / fmax (which would turn a -0.0 at lower = 0.0 into +0.0); absent bounds are passed as -inf / +inf
    return (TO)(a < s0 ? s0 : (a > s1 ? s1 : a));
  } else if constexpr (OP == MB200_OP_ROUND_S) {
    // numpy.round(x, d) (pandas DataFrame.round): d >= 0: rint(x * 10^d) / 10^d, d < 0: rint(x / 10^-d) * 10^-d;
    // s0 = 10^|d| (exact in float64 for |d| <= 22), s1 = sign of d.  rint = round-half-to-even.  Like numpy,
    // no guard against the scaled value overflowing (round(1e308, 2) = inf).
    if constexpr (F) {
      if (s1 >= (TI)0) return (TO)__ddiv_rn(rint(__dmul_rn(a, s0)), s0);
      return (TO)__dmul_rn(rint(__ddiv_rn(a, s0)), s0);
    } else {
      return (TO)a;  // integers: decimals >= 0 is the identity (negative decimals are not on this path)
    }
  } else if constexpr (OP == MB200_OP_NOT) {
    return (TO)(a == (TI)0);
  } else if constexpr (OP == MB200_OP_AND) {
    return (TO)((a != (TI)0) && (b != (TI)0));
  } else if constexpr (OP == MB200_OP_OR) {
    return (TO)((a != (TI)0) || (b != (TI)0));
  } else if constexpr (OP == MB200_OP_XOR) {
    return (TO)((a != (TI)0) != (b != (TI)0));
  } else if constexpr (OP == MB200_OP_ORDERED_S) {
    // sort key: an int64 whose signed order is the order sort_values wants.  float64: flip the magnitude bits
    // of negatives (total order of IEEE doubles), NaN -> INT64_MAX (na_position="last" in either direction);
    // s0 != 0 = descending: bitwise NOT reverses the order without overflow and keeps ties stable.
    long long o;
    if constexpr (F) {
      if (a != a) return (TO)0x7fffffffffffffffLL;
      const long long b = __double_as_longlong(a);
      o = b ^ ((b >> 63) & 0x7fffffffffffffffLL);
    } else {
      o = (long long)a;
    }
    return (TO)(s0 != (TI)0 ? ~o : o);
  } else if constexpr (OP == MB200_OP_COPY) {
    return (TO)a;
  } else if constexpr (OP == MB200_OP_FILLNA) {
    return (TO)((a != a) ? b : a);
  } else if constexpr (OP == MB200_OP_FMA3) {
    if constexpr (F) return (TO)__dadd_rn(__dmul_rn(a, b), c);
    else return (TO)(TI)((unsigned long long)a * (unsigned long long)b + (unsigned long long)c);
  } else {
    return (TO)a;
  }
}

// One element pair per thread and slab: a 16-byte access for the 8-byte types, 2 bytes for bool (uint8) columns.
template <typename T>
struct Pair;
template <>
struct Pair<double> {
  using type = double2;
  static __device__ __forceinline__ double2 load(const double* p) { return ldg_stream_f64x2(p); }
  static __device__ __forceinline__ void store(double* p, const double2& v) { stg_stream_f64x2(p, v); }
};
template <>
struct Pair<long long> {
  using type = longlong2;
  static __device__ __forceinline__ longlong2 load(const long long* p) { return ldg_stream_i64x2(p); }
  static __device__ __forceinline__ void store(long long* p, const longlong2& v) { stg_stream_i64x2(p, v); }
};
template <>
struct Pair<uint8_t> {
  using type = uchar2;
  static __device__ __forceinline__ uchar2 load(const uint8_t* p) { return __ldg(reinterpret_cast<const uchar2*>(p)); }
  static __device__ __forceinline__ void store(uint8_t* p, const uchar2& v) { *reinterpret_cast<uchar2*>(p) = v; }
};

// VEC=true: every operand pointer is 16-byte aligned -> vector path; else scalar sweep.
template <int OP, typename TI, typename TO, bool VEC>
__global__ void __launch_bounds__(kThreads) map_kernel(const __grid_constant__ MapParams p) {
  constexpr int NIN = op_nin(OP);
  const int tid = threadIdx.x;
  // one CTA per (row tile, column), as the Fold kernels: no per-tile index arithmetic, no tile loop
  const int col = blockIdx.y;
  const long long base = (long long)blockIdx.x * kTile;
  const TI* __restrict__ a = static_cast<const TI*>(p.in0[col]);
  const TI* __restrict__ b = NIN >= 2 ? static_cast<const TI*>(p.in1[col]) : nullptr;
  const TI* __restrict__ c = NIN >= 3 ? static_cast<const TI*>(p.in2[col]) : nullptr;
  TO* __restrict__ o = static_cast<TO*>(p.out[col]);
  const TI s0 = from_bits<TI>(p.s0[col]);
  const TI s1 = from_bits<TI>(p.s1[col]);
  if (VEC && base + kTile <= p.nrows) {
    // slab k, thread t: elements base + k * kSlab + 2 t and + 1, so each warp instruction covers whole sectors
    typename Pair<TI>::type va[kSlabs], vb[kSlabs], vc[kSlabs];
#pragma unroll
    for (int k = 0; k < kSlabs; ++k) {
      const long long i = base + k * kSlab + kPair * tid;
      va[k] = Pair<TI>::load(a + i);
      if constexpr (NIN >= 2) vb[k] = Pair<TI>::load(b + i);
      if constexpr (NIN >= 3) vc[k] = Pair<TI>::load(c + i);
    }
#pragma unroll
    for (int k = 0; k < kSlabs; ++k) {
      const long long i = base + k * kSlab + kPair * tid;
      TI bx = 0, by = 0, cx = 0, cy = 0;
      if constexpr (NIN >= 2) bx = vb[k].x, by = vb[k].y;
      if constexpr (NIN >= 3) cx = vc[k].x, cy = vc[k].y;
      typename Pair<TO>::type r;
      r.x = apply<OP, TI, TO>(va[k].x, bx, cx, s0, s1);
      r.y = apply<OP, TI, TO>(va[k].y, by, cy, s0, s1);
      Pair<TO>::store(o + i, r);
    }
  } else {
    const long long end = (base + kTile < p.nrows) ? base + kTile : p.nrows;
    for (long long i = base + tid; i < end; i += kThreads) {
      TI x = a[i];
      TI y = NIN >= 2 ? b[i] : (TI)0;
      TI z = NIN >= 3 ? c[i] : (TI)0;
      o[i] = apply<OP, TI, TO>(x, y, z, s0, s1);
    }
  }
}

#define MB_CASE(OPC, TI, TO)                                     \
  case OPC:                                                      \
    if (vec)                                                     \
      map_kernel<OPC, TI, TO, true><<<grid, kThreads, 0, st>>>(p);  \
    else                                                         \
      map_kernel<OPC, TI, TO, false><<<grid, kThreads, 0, st>>>(p); \
    MB_LAUNCH_CHECK("map_kernel");                               \
    return 0;

}  // namespace mb200

using namespace mb200;

extern "C" int mb200_map(int op, int dtype, int ncols, const void* const* in0, const void* const* in1,
                         const void* const* in2, void* const* out, int64_t nrows, const uint64_t* s0,
                         const uint64_t* s1, mb200_stream_t stream) {
  if (ncols < 0 || ncols > MB200_MAX_COLS) return fail("mb200_map", "ncols out of range (0..32)");
  if (nrows < 0) return fail("mb200_map", "negative nrows");
  if (ncols == 0 || nrows == 0) return 0;
  if (!in0 || !out) return fail("mb200_map", "null column array");
  const int nin = op_nin(op);
  if (nin >= 2 && !in1) return fail("mb200_map", "binary op needs in1");
  if (nin >= 3 && !in2) return fail("mb200_map", "ternary op needs in2");
  MapParams p;
  memset(&p, 0, sizeof(p));
  bool vec = true;
  for (int c = 0; c < ncols; ++c) {
    p.in0[c] = in0[c];
    p.in1[c] = nin >= 2 ? in1[c] : nullptr;
    p.in2[c] = nin >= 3 ? in2[c] : nullptr;
    p.out[c] = out[c];
    p.s0[c] = s0 ? s0[c] : 0;
    p.s1[c] = s1 ? s1[c] : 0;
    if (!in0[c] || !out[c]) return fail("mb200_map", "null column pointer");
    vec = vec && aligned16(in0[c]) && aligned16(out[c]);
    if (nin >= 2) vec = vec && in1[c] && aligned16(in1[c]);
    if (nin >= 3) vec = vec && in2[c] && aligned16(in2[c]);
    if ((nin >= 2 && !in1[c]) || (nin >= 3 && !in2[c])) return fail("mb200_map", "null column pointer");
  }
  p.nrows = nrows;
  const long long tiles_per_col = (nrows + kTile - 1) / kTile;
  if (tiles_per_col > 0x7fffffffLL) return fail("mb200_map", "too many rows for one launch");
  const dim3 grid((unsigned)tiles_per_col, (unsigned)ncols);
  cudaStream_t st = (cudaStream_t)stream;

  if (dtype == MB200_F64) {
    switch (op) {
      MB_CASE(MB200_OP_ABS, double, double)
      MB_CASE(MB200_OP_NEG, double, double)
      MB_CASE(MB200_OP_ISNA, double, uint8_t)
      MB_CASE(MB200_OP_NOTNA, double, uint8_t)
      MB_CASE(MB200_OP_FILLNA_S, double, double)
      MB_CASE(MB200_OP_AFFINE, double, double)
      MB_CASE(MB200_OP_ADD_S, double, double)
      MB_CASE(MB200_OP_SUB_S, double, double)
      MB_CASE(MB200_OP_RSUB_S, double, double)
      MB_CASE(MB200_OP_MUL_S, double, double)
      MB_CASE(MB200_OP_DIV_S, double, double)
      MB_CASE(MB200_OP_RDIV_S, double, double)
      MB_CASE(MB200_OP_EQ_S, double, uint8_t)
      MB_CASE(MB200_OP_NE_S, double, uint8_t)
      MB_CASE(MB200_OP_LT_S, double, uint8_t)
      MB_CASE(MB200_OP_LE_S, double, uint8_t)
      MB_CASE(MB200_OP_GT_S, double, uint8_t)
      MB_CASE(MB200_OP_GE_S, double, uint8_t)
      MB_CASE(MB200_OP_CLIP_S, double, double)
      MB_CASE(MB200_OP_COPY, double, double)
      MB_CASE(MB200_OP_ROUND_S, double, double)
      MB_CASE(MB200_OP_ORDERED_S, double, long long)
      MB_CASE(MB200_OP_ADD, double, double)
      MB_CASE(MB200_OP_SUB, double, double)
      MB_CASE(MB200_OP_MUL, double, double)
      MB_CASE(MB200_OP_DIV, double, double)
      MB_CASE(MB200_OP_EQ, double, uint8_t)
      MB_CASE(MB200_OP_NE, double, uint8_t)
      MB_CASE(MB200_OP_LT, double, uint8_t)
      MB_CASE(MB200_OP_LE, double, uint8_t)
      MB_CASE(MB200_OP_GT, double, uint8_t)
      MB_CASE(MB200_OP_GE, double, uint8_t)
      MB_CASE(MB200_OP_FILLNA, double, double)
      MB_CASE(MB200_OP_FMA3, double, double)
      default:
        return fail("mb200_map", "unsupported op for float64");
    }
  } else if (dtype == MB200_I64) {
    switch (op) {
      MB_CASE(MB200_OP_ABS, long long, long long)
      MB_CASE(MB200_OP_NEG, long long, long long)
      MB_CASE(MB200_OP_AFFINE, long long, long long)
      MB_CASE(MB200_OP_ADD_S, long long, long long)
      MB_CASE(MB200_OP_SUB_S, long long, long long)
      MB_CASE(MB200_OP_RSUB_S, long long, long long)
      MB_CASE(MB200_OP_MUL_S, long long, long long)
      MB_CASE(MB200_OP_DIV_S, long long, double)
      MB_CASE(MB200_OP_RDIV_S, long long, double)
      MB_CASE(MB200_OP_EQ_S, long long, uint8_t)
      MB_CASE(MB200_OP_NE_S, long long, uint8_t)
      MB_CASE(MB200_OP_LT_S, long long, uint8_t)
      MB_CASE(MB200_OP_LE_S, long long, uint8_t)
      MB_CASE(MB200_OP_GT_S, long long, uint8_t)
      MB_CASE(MB200_OP_GE_S, long long, uint8_t)
      MB_CASE(MB200_OP_CLIP_S, long long, long long)
      MB_CASE(MB200_OP_COPY, long long, long long)
      MB_CASE(MB200_OP_ROUND_S, long long, long long)
      MB_CASE(MB200_OP_ORDERED_S, long long, long long)
      MB_CASE(MB200_OP_ADD, long long, long long)
      MB_CASE(MB200_OP_SUB, long long, long long)
      MB_CASE(MB200_OP_MUL, long long, long long)
      MB_CASE(MB200_OP_DIV, long long, double)
      MB_CASE(MB200_OP_EQ, long long, uint8_t)
      MB_CASE(MB200_OP_NE, long long, uint8_t)
      MB_CASE(MB200_OP_LT, long long, uint8_t)
      MB_CASE(MB200_OP_LE, long long, uint8_t)
      MB_CASE(MB200_OP_GT, long long, uint8_t)
      MB_CASE(MB200_OP_GE, long long, uint8_t)
      MB_CASE(MB200_OP_FMA3, long long, long long)
      default:
        return fail("mb200_map", "unsupported op for int64");
    }
  } else if (dtype == MB200_U8) {
    // bool columns: logical ops stay bool; COPY widens to int64 (what a reduction over booleans consumes)
    switch (op) {
      MB_CASE(MB200_OP_COPY, uint8_t, long long)
      MB_CASE(MB200_OP_NOT, uint8_t, uint8_t)
      MB_CASE(MB200_OP_AND, uint8_t, uint8_t)
      MB_CASE(MB200_OP_OR, uint8_t, uint8_t)
      MB_CASE(MB200_OP_XOR, uint8_t, uint8_t)
      default:
        return fail("mb200_map", "unsupported op for bool");
    }
  }
  return fail("mb200_map", "unsupported dtype");
}
