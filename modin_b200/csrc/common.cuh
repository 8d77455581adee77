// common.cuh — shared helpers for the sm_90a kernels of libmodin_b200.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>

#include "../../include/modin_b200.h"

namespace mb200 {

// ---------------------------------------------------------------- error plumbing
extern thread_local char g_err[512];
extern std::atomic<long long> g_launches;

inline int fail(const char* what, const char* detail) {
  snprintf(g_err, sizeof(g_err), "%s: %s", what, detail ? detail : "");
  return 1;
}
inline int cuda_fail(const char* what, cudaError_t e) {
  snprintf(g_err, sizeof(g_err), "%s: CUDA error %d (%s)", what, (int)e, cudaGetErrorString(e));
  return 2;
}
#define MB_CUDA(call)                                   \
  do {                                                  \
    cudaError_t _e = (call);                            \
    if (_e != cudaSuccess) return cuda_fail(#call, _e); \
  } while (0)
#define MB_LAUNCH_CHECK(name)                              \
  do {                                                     \
    cudaError_t _e = cudaGetLastError();                   \
    if (_e != cudaSuccess) return cuda_fail(name, _e);     \
    g_launches.fetch_add(1, std::memory_order_relaxed);    \
  } while (0)

struct DevProps {
  int sm_count;
  size_t l2_bytes;
  int cc_major, cc_minor;
  size_t smem_optin;
};
// cached per-device properties; returns non-zero (error set) if no usable sm_90 device.
int dev_props(DevProps* out);
// Reference-counted persisting-L2 carve-out (runtime.cu): acquire returns the carve-out size in bytes (0 =
// unsupported) and the largest access-policy window; the last release hands the whole L2 back.
size_t l2_carveout_acquire(size_t* max_window_bytes);
void l2_carveout_release();
// hand an unused carve-out back to normally managed L2 (a device-synchronising call: done lazily, by kernels that want
// the whole L2 for themselves, never per group table)
void l2_carveout_drop_idle();

// ---------------------------------------------------------------- streaming loads/stores
// Streaming data is read once, so it bypasses L1 allocation and is marked evict-first in
// L2: this keeps the L2-resident hash tables of the groupby/join kernels from being flushed
// by the sweep.  sm_90 has no 256-bit global access and no `.L2::evict_first` qualifier on
// a plain load, so the evict-first priority goes through the cache-policy operand form.
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t pol;
  // not volatile: every call yields the same policy, so the compiler may hoist it out of loops
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

// Deliberately NOT `.nc`: ptxas sinks non-coherent loads below independent stores to save
// registers, which serialises the unrolled loads; plain ld.global keeps every load of a
// tile ahead of the first store.
//
// Two-element pairs, one 128-bit access each (LDG.E.128 / STG.E.128 on sm_90a).  With lane i
// at p + 2 i, one warp instruction covers 512 contiguous bytes: 16 whole 32-byte sectors.
__device__ __forceinline__ double2 ldg_stream_f64x2(const double* p) {
  double2 v;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.f64 {%0,%1}, [%2], %3;"
               : "=d"(v.x), "=d"(v.y)
               : "l"(p), "l"(l2_policy_evict_first()));
  return v;
}
__device__ __forceinline__ longlong2 ldg_stream_i64x2(const long long* p) {
  longlong2 v;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.s64 {%0,%1}, [%2], %3;"
               : "=l"(v.x), "=l"(v.y)
               : "l"(p), "l"(l2_policy_evict_first()));
  return v;
}
__device__ __forceinline__ void stg_stream_f64x2(double* p, const double2& v) {
  asm volatile("st.global.L1::no_allocate.v2.f64 [%0], {%1,%2};" ::"l"(p), "d"(v.x), "d"(v.y) : "memory");
}
__device__ __forceinline__ void stg_stream_i64x2(long long* p, const longlong2& v) {
  asm volatile("st.global.L1::no_allocate.v2.s64 [%0], {%1,%2};" ::"l"(p), "l"(v.x), "l"(v.y) : "memory");
}

// Four-element tiles, moved as two 128-bit accesses 16 B apart, at p and p + 2.  Lane i at p + 4 i
// therefore uses half of every sector per warp instruction; only reduce_ldg_kernel and
// key_range_kernel use these, because which element a lane reads fixes their summation order and
// their key sample.
struct __align__(32) f64x4 {
  double x, y, z, w;
};
struct __align__(32) i64x4 {
  long long x, y, z, w;
};

__device__ __forceinline__ f64x4 ldg_stream_f64x4(const double* p) {
  f64x4 v;
  const uint64_t pol = l2_policy_evict_first();
  asm volatile(
      "ld.global.L1::no_allocate.L2::cache_hint.v2.f64 {%0,%1}, [%4], %6;\n\t"
      "ld.global.L1::no_allocate.L2::cache_hint.v2.f64 {%2,%3}, [%5], %6;"
      : "=d"(v.x), "=d"(v.y), "=d"(v.z), "=d"(v.w)
      : "l"(p), "l"(p + 2), "l"(pol));
  return v;
}
__device__ __forceinline__ i64x4 ldg_stream_i64x4(const long long* p) {
  i64x4 v;
  const uint64_t pol = l2_policy_evict_first();
  asm volatile(
      "ld.global.L1::no_allocate.L2::cache_hint.v2.s64 {%0,%1}, [%4], %6;\n\t"
      "ld.global.L1::no_allocate.L2::cache_hint.v2.s64 {%2,%3}, [%5], %6;"
      : "=l"(v.x), "=l"(v.y), "=l"(v.z), "=l"(v.w)
      : "l"(p), "l"(p + 2), "l"(pol));
  return v;
}
// Scalar streaming loads take the same cache-policy operand.
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ double ldg_stream_f64(const double* p, uint64_t pol) {
  double v;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ long long ldg_stream_i64(const long long* p, uint64_t pol) {
  long long v;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.s64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
  return v;
}

// ---------------------------------------------------------------- mbarrier + TMA bulk copy
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// 1-D TMA bulk copy global -> shared, completion signalled on an mbarrier (UBLKCP in SASS).
__device__ __forceinline__ void tma_bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes,
                                             uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
      "[%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}

// ---------------------------------------------------------------- misc device helpers
__device__ __forceinline__ uint64_t mix64(uint64_t z) {  // splitmix64 finaliser
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
__device__ __forceinline__ uint32_t hash_key(long long k) {
  // murmur3 fmix64 -> 32 bits; must match oracle-independent host code nowhere (device only)
  uint64_t z = (uint64_t)k;
  z ^= z >> 33;
  z *= 0xff51afd7ed558ccdULL;
  z ^= z >> 33;
  z *= 0xc4ceb9fe1a85ec53ULL;
  z ^= z >> 33;
  return (uint32_t)z;
}

// ---------------------------------------------------------------- key statistics {min, max, sampled, duplicated}
// The statistics a groupby needs about its int64 key column to pick a table (dense range? skewed?).  They are
// column METADATA: computed by whichever kernel produces the column (gen_i64*, the ingest pass after an H2D
// copy) or, for a column of unknown origin, once by key_range_kernel -- never per query.
//   stats[0] = min, stats[1] = max, stats[2] = keys sampled, stats[3] = of those, how many shared their value
//   with another of the 32 keys sampled in the same warp instruction.
struct KeyStatsAcc {
  long long lo = 0x7fffffffffffffffLL, hi = (long long)0x8000000000000000ULL;
  unsigned int sampled = 0, dups = 0;
  __device__ __forceinline__ void add(long long k) {
    lo = k < lo ? k : lo;
    hi = k > hi ? k : hi;
  }
  // all 32 lanes of the warp must call this together
  __device__ __forceinline__ void sample_warp(long long k) {
    const unsigned int peers = __match_any_sync(0xffffffffu, (unsigned long long)k);
    dups += __popc(__ballot_sync(0xffffffffu, __popc(peers) > 1));
    sampled += 32;
  }
  // block-wide fold + one atomic quadruple per block; blockDim.x <= 1024, every thread of the block calls it
  __device__ __forceinline__ void flush(long long* stats) {
    __shared__ long long s_min[32], s_max[32];
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) {
      const long long a = __shfl_xor_sync(0xffffffffu, lo, m), b = __shfl_xor_sync(0xffffffffu, hi, m);
      lo = a < lo ? a : lo;
      hi = b > hi ? b : hi;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = (blockDim.x + 31) >> 5;
    if (lane == 0) {
      s_min[warp] = lo;
      s_max[warp] = hi;
      if (sampled) {  // every lane of a warp holds the same two counters
        atomicAdd(reinterpret_cast<unsigned long long*>(&stats[2]), (unsigned long long)sampled);
        atomicAdd(reinterpret_cast<unsigned long long*>(&stats[3]), (unsigned long long)dups);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < nwarps; ++w) {
        lo = s_min[w] < lo ? s_min[w] : lo;
        hi = s_max[w] > hi ? s_max[w] : hi;
      }
      if (lo <= hi) {
        atomicMin(&stats[0], lo);
        atomicMax(&stats[1], hi);
      }
    }
  }
};

// stats_dev[4] <- {INT64_MAX, INT64_MIN, 0, 0} (groupby.cu)
int key_stats_init(long long* stats_dev, cudaStream_t st);

inline bool aligned32(const void* p) { return (((uintptr_t)p) & 31u) == 0; }
inline bool aligned16(const void* p) { return (((uintptr_t)p) & 15u) == 0; }

}  // namespace mb200
