// groupby.cu — GroupByReduce: open-addressed hash aggregation of one block into an
// L2-resident table, plus the sorted emit.
//
// Reference path: GroupByReduce.map (alg/groupby.py:124-208) runs `df.groupby(by).sum()` per
// row block (pandas: factorize = hash of the key column, then _libs.groupby.group_sum);
// GroupByReduce.reduce (alg/groupby.py:211-300) concatenates the partial tables and regroups.
// Here one table per GPU absorbs every row block resident on that GPU (map + local reduce
// fused), and partial tables from other GPUs are merged with the same kernel.
//
// Data structure (all device resident):
//   slots[cap]   16-byte {int64 key, int32 gid, pad}; cap = pow2 >= 2 * group_capacity.
//                gid: -1 empty, -2 claimed (being published), [0, gcap) dense id, gcap = overflowed.
//                A slot is published with ONE 128-bit store {key, gid} and read with ONE 128-bit load.
//   acc[gcap][vstride]  float64 sums, row-major so one group's V sums share 64-byte segments.
//   cnt[gcap][vstride]  int64 non-NaN counts (optional), size[gcap] int64 rows (optional).
// For G = 1e6, V = 8 the table is 32 MiB of slots + 64 MiB of sums, more than the 50 MB L2 of an H100,
// so the streamed 72 B/row input is loaded with an L2 evict-first policy to leave the L2 to the table.
// A table that misses L2 makes the kernel bound by random 32-byte-sector DRAM traffic rather than by
// the atomics or the stream.
//
// Kernels
//   gb_accumulate_tma_kernel (every table size; V <= 8, 16-byte aligned columns): a producer warp streams
//     256-row tiles of the key + value columns into a shared-memory ring with 1-D TMA bulk copies
//     (full/empty mbarriers), so DRAM latency is out of the per-row dependency chain and no
//     registers hold in-flight rows; 8 consumer warps each take 32 rows of a tile.
//   gb_accumulate_kernel (ragged tails, unaligned views, V > 8, partial-table merges, or MB200_GB_VARIANT=1):
//     the same per-warp algorithm with direct coalesced loads and 40 resident warps per SM.
// Per warp (32 rows):
//   1. warp-cooperative probe: __match_any_sync groups lanes holding the same key; the lowest lane
//      of each group looks the key up (read-only linear probing).  Missing keys are inserted in
//      warp-convergent ROUNDS: claim the empty slot with a CAS, take dense ids with one atomicAdd
//      per warp per round, publish {key, gid} with a 128-bit store; a lane that meets a slot
//      claimed by someone else simply retries next round -- no lane ever spins on another lane;
//   2. accumulate with RED.ADD.F64, 8 consecutive lanes updating the 8 sums of ONE group (one
//      64-byte segment, one L2 request per row); the value tile is read transposed from shared memory.
// Float atomics make the summation order run-dependent: results agree with pandas to the
// tolerance stated in tests (|err| <= 4 log2(n) eps sum|x|), not bit for bit; counts/sizes
// and keys are exact.
#include "common.cuh"

namespace mb200 {

int sort_pairs_device(long long* keys, long long* pay, long long* tmp_keys, long long* tmp_pay,
                      unsigned int* counts, long long n, unsigned long long bias, int nbits, cudaStream_t st);
size_t sort_scratch_bytes(long long n);

struct __align__(16) Slot {
  long long key;
  int gid;
  int pad;
};

struct GbMeta {  // device-side bookkeeping
  int ngroups;
  int overflow;
  long long kmin;  // filled by gb_collect_kernel
  long long kmax;
};

}  // namespace mb200

struct mb200_gb_table {
  mb200::Slot* slots;
  long long cap;  // power of two
  double* acc;
  long long* cnt;
  long long* size;
  long long gcap;
  int nvals;
  int vstride;
  int flags;
  mb200::GbMeta* meta;
  // dense (direct-addressed) tables: gid = key - kbase, no slots; one presence byte per key
  int dense;
  long long kbase;
  unsigned int* present;   // [nwords] words of 4 presence bytes
  long long nwords;
  unsigned int* blockoff;  // [nwords / 256 + 1] per-block popcounts -> exclusive offsets (emit)
  int borrowed;            // acc / cnt / size / present belong to the caller
  int skewed;              // mb200_gb_hint_skew: use the per-CTA hot-group cache
  int persisted;           // holds a reference on the persisting L2 carve-out (accumulators pinned)
  size_t carve_bytes, window_bytes;
  long long win_lo, win_hi;  // gid window that ngroups / emit report (default: the whole range)
  // hashed tables: slots | acc | cnt | size live in ONE allocation so that one persisting-L2 access window
  // can cover the probe slots AND the accumulators (a stream carries a single window)
  void* arena;
  size_t arena_bytes;
  long long rows;  // rows accumulated so far: the position of the next accumulate call's first row (FIRST / LAST)
  int arg_filled;  // ARGMIN / ARGMAX: mb200_gb_accumulate_arg has run (it runs once per table)
};

namespace mb200 {

constexpr int kGbThreads = 256;
constexpr int kGbWarps = kGbThreads / 32;
constexpr int kGbArg = MB200_GB_ARGMIN | MB200_GB_ARGMAX;  // groupby.idxmin / idxmax tables
constexpr int kColStride = 34;  // doubles; 34 = 2 (mod 16) -> conflict-free transposed reads
// TMA-staged kernel
constexpr int kTileRows = 256;
constexpr int kTileColStride = 258;  // doubles; 258 = 2 (mod 16), and 258 * 8 is a multiple of 16 bytes
constexpr int kGbStages = 3;
constexpr int kGbTmaThreads = kGbThreads + 32;
constexpr int kStageBytes = ((9 * kTileColStride * 8 + 127) / 128) * 128;

struct GbParams {
  Slot* slots;
  unsigned int mask;
  long long cap;
  double* acc;
  long long* cnt;
  long long* size;
  long long gcap;
  int nvals;
  int vstride;
  int flags;
  GbMeta* meta;
  const long long* keys;
  const void* vals[MB200_MAX_COLS];   // raw values, or partial sums when PARTIAL
  const void* pcnt[MB200_MAX_COLS];   // partial counts (PARTIAL only)
  union {                             // PARTIAL and FIRST / LAST tables exclude each other
    const long long* psize;           // partial sizes (PARTIAL only)
    long long row0;                   // FIRST / LAST: table position of row 0 of this launch (earlier calls' rows)
  };
  long long nrows;
  int dense;              // direct-addressed table: gid = key - kbase
  long long kbase;
  unsigned int* present;  // dense: one byte per key of [kbase, kbase + gcap)
};

// ---- table accesses: relaxed GPU-scope
__device__ __forceinline__ void red_add_f64(double* p, double v) {
  asm volatile("red.relaxed.gpu.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
__device__ __forceinline__ void red_add_u64(long long* p, long long v) {
  asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_slot(Slot* s, long long key, int gid) {
  const unsigned long long b = (unsigned long long)(unsigned int)gid;
  asm volatile("st.relaxed.gpu.global.v2.u64 [%0], {%1,%2};" ::"l"(s), "l"((unsigned long long)key), "l"(b)
               : "memory");
}

// min / max accumulators share the `acc` array: doubles are stored through an order-preserving map to
// int64 (flip the magnitude bits of negatives) so that RED.MIN.S64 / RED.MAX.S64 order them like
// floating-point comparison.  NaNs are skipped by the callers; INT64_MAX / INT64_MIN (the images of
// all-ones NaNs) mark "no value yet" for min / max and decode to NaN.
__device__ __forceinline__ long long f64_to_ordered(double x) {
  const long long b = __double_as_longlong(x);
  return b ^ ((b >> 63) & 0x7fffffffffffffffLL);
}
__device__ __forceinline__ double ordered_to_f64(long long o) {
  return __longlong_as_double(o ^ ((o >> 63) & 0x7fffffffffffffffLL));
}
__device__ __forceinline__ void red_min_s64(long long* p, long long v) {
  asm volatile("red.relaxed.gpu.global.min.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_max_s64(long long* p, long long v) {
  asm volatile("red.relaxed.gpu.global.max.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// value accumulator update of one (group, column): sum, or min / max on the ordered image
__device__ __forceinline__ void acc_update(const GbParams& p, size_t o, double xv) {
  if (p.flags & MB200_GB_SUM) red_add_f64(p.acc + o, xv);
  else if (p.flags & MB200_GB_MIN) red_min_s64(reinterpret_cast<long long*>(p.acc) + o, f64_to_ordered(xv));
  else if (p.flags & MB200_GB_MAX) red_max_s64(reinterpret_cast<long long*>(p.acc) + o, f64_to_ordered(xv));
}

// FIRST / LAST (the POS kernels): the accumulator of (group, column) is min / max of the positions of the rows whose
// value is not NaN -- the same RED.MIN.S64 / RED.MAX.S64 as min / max, on positions instead of ordered values
__device__ __forceinline__ void pos_update(const GbParams& p, size_t o, long long pos) {
  if (p.flags & MB200_GB_FIRST) red_min_s64(reinterpret_cast<long long*>(p.acc) + o, pos);
  else red_max_s64(reinterpret_cast<long long*>(p.acc) + o, pos);
}

// does adding / min-ing / max-ing / counting `xv` leave a trace in a DENSE table's accumulators?
// (POS: every non-NaN value moves its position accumulator off the sentinel)
template <bool POS = false>
__device__ __forceinline__ bool dense_visible(const GbParams& p, double xv) {
  if (xv != xv) return false;                                                   // NaNs are skipped everywhere
  if (POS) return true;
  if (p.flags & (MB200_GB_COUNT | MB200_GB_MIN | MB200_GB_MAX)) return true;  // cnt > 0 / acc != sentinel
  return __double_as_longlong(xv) != (long long)0x8000000000000000ULL;          // -0.0 + -0.0 stays -0.0
}
__device__ __forceinline__ void dense_mark(const GbParams& p, int g) {
  asm volatile("st.relaxed.gpu.global.u8 [%0], %1;" ::"l"(reinterpret_cast<unsigned char*>(p.present) + g), "r"(1u)
               : "memory");
}

// Probing works on BUCKETS of two slots = one 32-byte sector, fetched with two back-to-back 128-bit loads
// (sm_90 has no 256-bit load; each slot is still read whole, as it is published with one 128-bit store):
// a probe round costs the same sector as a single-slot probe but the chain of rounds is about half as long
// (with single-slot linear probing at load factor 0.48 the longest of a warp's 32 chains averaged 5.6
// dependent round trips per 32 rows -- 29 % of all stall samples sat on that load).
// All probe loops have WARP-UNIFORM trip counts (the continue condition is a __any_sync vote), so
// every lane leaves a loop together.  A data-dependent `break` per lane is legal under independent
// thread scheduling but nvcc then lets the early finishers run ahead, and the warp executes the
// accumulate phase in diverged groups (more RED instructions for the same rows).
__device__ __forceinline__ void ld_bucket(const Slot* b, long long& k0, int& g0, long long& k1, int& g1) {
  unsigned long long a, x, c, d;
  asm volatile(
      "ld.relaxed.gpu.global.v2.u64 {%0,%1}, [%4];\n\t"
      "ld.relaxed.gpu.global.v2.u64 {%2,%3}, [%5];"
      : "=l"(a), "=l"(x), "=l"(c), "=l"(d)
      : "l"(b), "l"(b + 1)
      : "memory");
  k0 = (long long)a;
  g0 = (int)(unsigned int)(x & 0xffffffffULL);
  k1 = (long long)c;
  g1 = (int)(unsigned int)(d & 0xffffffffULL);
}

// One probe round for key `k` at `bucket`.  Returns: >= 0 found gid; -1 the first non-foreign slot
// (index `sub`) is empty; -2 it is being published by someone; -3 both slots hold other keys.
__device__ __forceinline__ int probe_bucket(const GbParams& p, long long k, unsigned int bucket, int& sub) {
  long long k0, k1;
  int g0, g1;
  ld_bucket(p.slots + 2 * (size_t)bucket, k0, g0, k1, g1);
  sub = 0;
  if (g0 >= 0 && k0 == k) return g0;
  if (g0 < 0) return g0;  // -1 empty / -2 in flight
  sub = 1;
  if (g1 >= 0 && k1 == k) return g1;
  if (g1 < 0) return g1;
  return -3;
}

// Warp-wide lookup: dense group id of each leader's key, or -1 when its probe chain ends at an empty
// or in-flight slot (`bucket` is left at that position).  Read-only: the steady-state path.
__device__ __forceinline__ int probe_find(const GbParams& p, long long k, bool is_leader, unsigned int& bucket) {
  int found = -1;
  long long probes = 0;
  bool active = is_leader;
  const unsigned int bmask = p.mask >> 1;
  while (__any_sync(0xffffffffu, active)) {
    if (active) {
      int sub;
      const int r = probe_bucket(p, k, bucket, sub);
      if (r >= 0) found = r;
      if (r != -3 || ++probes > p.cap) active = false;
      else bucket = (bucket + 1) & bmask;
    }
  }
  return found;
}

// Slow path, entered by the WHOLE warp (uniform branch) when some leader's key is not in the table yet.
// Rounds: every pending leader walks its chain (uniform-trip loop) until it finds its key, claims an
// empty slot with a CAS, or meets a slot that somebody else is publishing (retry next round); the
// round's winners take consecutive dense ids from ONE atomicAdd and publish {key, gid} with a 128-bit
// store.  No lane ever spins on another lane of its own warp.
__device__ __noinline__ int insert_rounds(const GbParams& p, long long k, bool is_leader, int gid,
                                          unsigned int bucket) {
  const int lane = threadIdx.x & 31;
  const int gcap = (int)p.gcap;
  const unsigned int bmask = p.mask >> 1;
  long long probes = 0;
  while (__any_sync(0xffffffffu, is_leader && gid < 0)) {
    bool won = false;
    int sub = 0;
    bool walking = is_leader && gid < 0;
    while (__any_sync(0xffffffffu, walking)) {
      if (walking) {
        const int r = probe_bucket(p, k, bucket, sub);
        if (r >= 0) {
          gid = r;
          walking = false;
        } else if (r == -3) {
          if (++probes > p.cap) {  // table full of other keys
            p.meta->overflow = 1;
            gid = gcap;
            walking = false;
          } else {
            bucket = (bucket + 1) & bmask;
          }
        } else {
          if (r == -1) won = (atomicCAS(&p.slots[2 * (size_t)bucket + sub].gid, -1, -2) == -1);
          walking = false;  // claimed it, or someone else is publishing this slot: look again next round
        }
      }
    }
    // dense ids for this round's winners: one atomicAdd per warp
    const unsigned int winners = __ballot_sync(0xffffffffu, won);
    if (winners) {
      const int first = __ffs(winners) - 1;
      int base = 0;
      if (lane == first) base = atomicAdd(&p.meta->ngroups, __popc(winners));
      base = __shfl_sync(0xffffffffu, base, first);
      if (won) {
        int ng = base + __popc(winners & ((1u << lane) - 1u));
        if (ng >= gcap) {
          p.meta->overflow = 1;
          ng = gcap;
        }
        st_slot(&p.slots[2 * (size_t)bucket + sub], k, ng);
        gid = ng;
      }
    }
  }
  return gid;
}

// Dense group id of every lane's key (gcap = table overflowed).  Must be called by all 32 lanes.
__device__ __forceinline__ int resolve_gid(const GbParams& p, long long k) {
  if (p.dense) {
    // direct addressing (kernel-uniform branch): no probe, no slots, and normally no presence access either:
    // dense accumulators start from a value no update can leave behind (-0.0 for sums, the "no value yet"
    // sentinels for min / max, 0 for counts / sizes), so a key is present iff its row changed -- only a row
    // that changes nothing (all values NaN or -0.0, no size) marks the presence byte (mark_if_invisible).
    // A per-row presence check cost as many L1 tag lookups as all the REDs of the row together.
    const unsigned long long d = (unsigned long long)k - (unsigned long long)p.kbase;
    if (d >= (unsigned long long)p.gcap) {
      p.meta->overflow = 1;  // key outside the declared range
      return (int)p.gcap;
    }
    return (int)d;
  }
  const int lane = threadIdx.x & 31;
  const unsigned int peers = __match_any_sync(0xffffffffu, (unsigned long long)k);
  const int leader = __ffs(peers) - 1;
  const bool is_leader = (lane == leader);
  unsigned int bucket = hash_key(k) & (p.mask >> 1);
  int gid = probe_find(p, k, is_leader, bucket);
  if (__any_sync(0xffffffffu, is_leader && gid < 0)) gid = insert_rounds(p, k, is_leader, gid, bucket);
  return __shfl_sync(0xffffffffu, gid, leader);
}

// ---------------------------------------------------------------- fallback: direct loads
// POS: FIRST / LAST tables (raw rows only) -- positions go to the accumulators, and a NULL value column reads as
// "no NaN" without a load.  POS = false compiles to the code these kernels had before FIRST / LAST existed.
template <bool PARTIAL, bool POS>
__global__ void __launch_bounds__(kGbThreads, 5) gb_accumulate_kernel(const __grid_constant__ GbParams p) {
  static_assert(!(POS && PARTIAL), "FIRST / LAST tables take raw rows only");
  __shared__ double s_tile[kGbWarps][8 * kColStride];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long nchunks = (p.nrows + 31) >> 5;
  const long long wstride = (long long)gridDim.x * kGbWarps;
  const int gcap = (int)p.gcap;
  const uint64_t pol = l2_policy_evict_first();
  for (long long ch = (long long)blockIdx.x * kGbWarps + warp; ch < nchunks; ch += wstride) {
    const long long base = ch << 5;
    const long long row = base + lane;
    const bool valid = row < p.nrows;
    long long k = valid ? ldg_stream_i64(p.keys + row, pol) : 0;
    // value loads of the first 8 columns are issued before the (dependent, random) probe
    double x[8];
    {
      const int nc = p.nvals < 8 ? p.nvals : 8;
#pragma unroll
      for (int c = 0; c < 8; ++c)
        x[c] = (c < nc && valid && (!POS || p.vals[c])) ? ldg_stream_f64(static_cast<const double*>(p.vals[c]) + row, pol)
                                                        : 0.0;
    }
    {
      // rows past the end borrow lane 0's key (lane 0 is always valid in a live chunk) so that they join
      // its peer group and never become leaders; the shuffle is executed by ALL lanes.
      const long long k0 = __shfl_sync(0xffffffffu, k, 0);
      k = valid ? k : k0;
    }
    const int gid = resolve_gid(p, k);
    const bool live = valid && gid < gcap;

    if ((p.flags & MB200_GB_SIZE) && live) red_add_u64(p.size + gid, PARTIAL ? p.psize[row] : 1LL);
    if (p.dense && p.nvals == 0 && !(p.flags & MB200_GB_SIZE) && live) dense_mark(p, gid);  // keys only
    // ---- accumulate, 8 value columns at a time
    for (int c0 = 0; c0 < p.nvals; c0 += 8) {
      const int nc = (p.nvals - c0) < 8 ? (p.nvals - c0) : 8;
      if (c0 > 0) {
#pragma unroll
        for (int c = 0; c < 8; ++c)
          x[c] = (c < nc && valid && (!POS || p.vals[c0 + c]))
                     ? ldg_stream_f64(static_cast<const double*>(p.vals[c0 + c]) + row, pol)
                     : 0.0;
      }
      double* tile = s_tile[warp];
#pragma unroll
      for (int c = 0; c < 8; ++c) tile[c * kColStride + lane] = x[c];
      __syncwarp();
      const int c = lane & 7;
      unsigned int seen = 0, rowok = 0;
      int gs[8];
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const int r = 4 * kk + (lane >> 3);
        const int g = __shfl_sync(0xffffffffu, gid, r);
        const double xv = tile[c * kColStride + r];
        const bool ok = (base + r < p.nrows) && (c < nc) && (g < gcap);
        gs[kk] = g;
        if ((base + r < p.nrows) && g < gcap) rowok |= 1u << kk;
        if (ok) {
          const size_t o = (size_t)g * p.vstride + c0 + c;
          if (!PARTIAL && dense_visible<POS>(p, xv)) seen |= 1u << kk;
          if (POS) {
            if (xv == xv) pos_update(p, o, p.row0 + base + r);
          } else if (xv == xv) {
            acc_update(p, o, xv);
          }
          if (p.flags & MB200_GB_COUNT) {
            if (PARTIAL) red_add_u64(p.cnt + o, static_cast<const long long*>(p.pcnt[c0 + c])[base + r]);
            else if (xv == xv) red_add_u64(p.cnt + o, 1LL);
          }
        }
      }
      if (p.dense && !(p.flags & MB200_GB_SIZE)) {  // rows that left no trace mark their presence byte
        seen |= __shfl_xor_sync(0xffffffffu, seen, 1);
        seen |= __shfl_xor_sync(0xffffffffu, seen, 2);
        seen |= __shfl_xor_sync(0xffffffffu, seen, 4);
        const unsigned int unseen = ~seen & rowok;
        if (c == 0 && unseen) {
#pragma unroll
          for (int kk = 0; kk < 8; ++kk)
            if ((unseen >> kk) & 1u) dense_mark(p, gs[kk]);
        }
      }
      __syncwarp();
    }
  }
}

// ---------------------------------------------------------------- default: TMA-staged tiles
// Handles the first ntiles * 256 rows (full tiles only); nvals <= 8; raw rows (not partial tables).
//
// HOT = true (skewed keys, mb200_gb_hint_skew): each CTA keeps a direct-mapped cache of kHotSlots groups in
// shared memory (slot = gid mod kHotSlots, claimed by the first group that arrives and kept to the end: a
// group with a large share of the rows arrives within the first few rows).  Rows of a cached group are
// accumulated with shared-memory atomics and the cache is added to the table once per CTA; all other rows
// take the global REDs.  Without it every row of a hot key serialises on one 64-byte L2 line.  SUM / COUNT
// tables only.
constexpr int kHotSlots = 256;
constexpr int kHotStride = 9;  // doubles per cached group (8 sums + 1 pad against bank conflicts)
// The HOT variant runs a 2-stage ring (the plain one 3): its cache shares the SM's shared memory with the ring, and
// at 3 stages only 2 CTAs fit per SM -- 2 stages and no count array for pure sums fit 3-4.
constexpr int kHotStages = 2;
__host__ __device__ constexpr int hot_offset(int stages) {
  return ((stages * kStageBytes + 2 * stages * 8 + 63) / 64) * 64;
}
constexpr int kHotBytesSum = kHotSlots * 4 + kHotSlots * kHotStride * 8;                 // tags + sums
constexpr int kHotBytes = kHotBytesSum + kHotSlots * kHotStride * 4;                     // ... + counts
constexpr int kHotBit = 1 << 30;  // group ids are < 2^29

template <bool HOT, int STAGES, bool POS>
__global__ void __launch_bounds__(kGbTmaThreads) gb_accumulate_tma_kernel(const __grid_constant__ GbParams p,
                                                                          long long ntiles) {
  static_assert(!(HOT && POS), "FIRST / LAST tables do not take the hot-group cache");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + STAGES * kStageBytes);
  uint64_t* empty = full + STAGES;
  int* s_tag = reinterpret_cast<int*>(smem_raw + hot_offset(STAGES));
  double* s_hot = reinterpret_cast<double*>(smem_raw + hot_offset(STAGES) + kHotSlots * 4);
  unsigned int* s_hcnt = reinterpret_cast<unsigned int*>(smem_raw + hot_offset(STAGES) + kHotSlots * 4 + kHotSlots * kHotStride * 8);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nv = p.nvals;
  const int gcap = (int)p.gcap;
  const long long first = blockIdx.x;
  const long long nmine = first < ntiles ? (ntiles - first + gridDim.x - 1) / gridDim.x : 0;

  if (HOT) {
    for (int i = tid; i < kHotSlots; i += kGbTmaThreads) s_tag[i] = -1;
    for (int i = tid; i < kHotSlots * kHotStride; i += kGbTmaThreads) {
      s_hot[i] = 0.0;
      if (p.flags & MB200_GB_COUNT) s_hcnt[i] = 0u;  // the count array exists only for COUNT tables
    }
  }
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], kGbWarps);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == kGbWarps) {
    // ---------------- producer: (1 + nv) bulk copies of 2 KiB per tile
    if (lane == 0) {
      const uint64_t pol = l2_policy_evict_first();
      int ncopy = nv;  // POS: NULL value columns ("no NaN") are not copied
      if (POS)
        for (int c = 0; c < nv; ++c) ncopy -= p.vals[c] ? 0 : 1;
      for (long long k = 0; k < nmine; ++k) {
        const int s = (int)(k % STAGES);
        if (k >= STAGES) mbar_wait(&empty[s], (uint32_t)(((k / STAGES) - 1) & 1));
        const long long row0 = (first + k * gridDim.x) * kTileRows;
        double* stage = reinterpret_cast<double*>(smem_raw + (size_t)s * kStageBytes);
        mbar_expect_tx(&full[s], (uint32_t)((1 + ncopy) * kTileRows * 8));
        tma_bulk_g2s(stage, p.keys + row0, kTileRows * 8, &full[s], pol);
        for (int c = 0; c < nv; ++c)
          if (!POS || p.vals[c])
            tma_bulk_g2s(stage + (size_t)(1 + c) * kTileColStride, static_cast<const double*>(p.vals[c]) + row0,
                         kTileRows * 8, &full[s], pol);
      }
    }
    return;
  }
  // ---------------- consumers: warp w owns rows [32w, 32w + 32) of every tile
  const int c = lane & 7;
  const bool nullcol = POS && c < nv && !p.vals[c];  // POS: this lane's column has no NaN and no staged tile
  for (long long k = 0; k < nmine; ++k) {
    const int s = (int)(k % STAGES);
    mbar_wait(&full[s], (uint32_t)((k / STAGES) & 1));
    const double* stage = reinterpret_cast<const double*>(smem_raw + (size_t)s * kStageBytes);
    const long long key = reinterpret_cast<const long long*>(stage)[warp * 32 + lane];
    int gid = resolve_gid(p, key);
    if ((p.flags & MB200_GB_SIZE) && gid < gcap) red_add_u64(p.size + gid, 1LL);
    if (HOT && gid < gcap) {  // is this row's group in the CTA's hot cache (or can it claim its slot)?
      const int slot = gid & (kHotSlots - 1);
      int tag = *reinterpret_cast<volatile int*>(&s_tag[slot]);
      if (tag == -1) {
        const int old = atomicCAS(&s_tag[slot], -1, gid);
        tag = old == -1 ? gid : old;
      }
      if (tag == gid) gid |= kHotBit;
    }
    const double* vt = stage + kTileColStride + warp * 32;  // value column 0, this warp's rows
    unsigned int seen = 0;  // bit kk: this lane's (row 4 kk + lane / 8, column c) update leaves a trace
    int gs[8];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const int r = 4 * kk + (lane >> 3);
      const int pg = __shfl_sync(0xffffffffu, gid, r);
      const int g = HOT ? (pg & ~kHotBit) : pg;
      gs[kk] = g;
      if (c < nv && g < gcap) {
        const double xv = nullcol ? 0.0 : vt[c * kTileColStride + r];
        if (dense_visible<POS>(p, xv)) seen |= 1u << kk;
        if (POS) {
          if (xv == xv) pos_update(p, (size_t)g * p.vstride + c, p.row0 + (first + k * gridDim.x) * kTileRows + warp * 32 + r);
        } else if (xv == xv) {
          if (HOT && (pg & kHotBit)) {
            const int o = (g & (kHotSlots - 1)) * kHotStride + c;
            if (p.flags & MB200_GB_SUM) atomicAdd(&s_hot[o], xv);
            if (p.flags & MB200_GB_COUNT) atomicAdd(&s_hcnt[o], 1u);
          } else {
            const size_t o = (size_t)g * p.vstride + c;
            acc_update(p, o, xv);
            if (p.flags & MB200_GB_COUNT) red_add_u64(p.cnt + o, 1LL);
          }
        }
      }
    }
    if (p.dense && !(p.flags & MB200_GB_SIZE)) {
      // rows none of whose 8 columns left a trace mark their presence byte (rare).  OR over the 8 lanes of a
      // row with three shuffles AFTER the REDs: a vote per row inside the loop serialised the tile reads.
      seen |= __shfl_xor_sync(0xffffffffu, seen, 1);
      seen |= __shfl_xor_sync(0xffffffffu, seen, 2);
      seen |= __shfl_xor_sync(0xffffffffu, seen, 4);
      unsigned int unseen = ~seen & 0xffu;
      if (c == 0 && unseen) {
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)
          if (((unseen >> kk) & 1u) && gs[kk] < gcap) dense_mark(p, gs[kk]);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
  }
  if (HOT) {
    // the 8 consumer warps fold the cache into the table (the producer warp has returned: named barrier)
    asm volatile("bar.sync 1, %0;" ::"n"(kGbThreads) : "memory");
    for (int i = tid; i < kHotSlots * 8; i += kGbThreads) {
      const int slot = i >> 3, cc = i & 7;
      const int tag = s_tag[slot];
      if (tag < 0 || cc >= nv) continue;
      const size_t o = (size_t)tag * p.vstride + cc;
      if (p.flags & MB200_GB_SUM) red_add_f64(p.acc + o, s_hot[slot * kHotStride + cc]);
      if ((p.flags & MB200_GB_COUNT) && s_hcnt[slot * kHotStride + cc])
        red_add_u64(p.cnt + o, (long long)s_hcnt[slot * kHotStride + cc]);
    }
  }
}

// ---------------------------------------------------------------- low-cardinality keys: table in shared memory
// Dense tables small enough for shared memory (R <= ~3100 at V = 8) are PRIVATISED per CTA: rows are
// accumulated with shared-memory atomics and each CTA adds its table to the global one once at the end.
// With few distinct keys every row of the frame would otherwise hit the same few L2 lines with global
// atomics.
// One 1024-thread CTA per SM, the whole dynamic shared memory is the table; rows are loaded straight from
// global memory (lane == row, every load a coalesced 256-byte warp access; 32 warps x 9 loads in flight
// cover the HBM latency) and lane == row also for the atomics: table rows are padded to vs + 1 doubles so
// that 32 different groups spread over the banks.  64-bit float shared atomics are CAS loops
// (ATOMS.CAST.SPIN.64); per-CTA counts fit 32 bits and use the native ATOMS.ADD.
constexpr int kSmemThreads = 1024;

struct SmemTableLayout {
  unsigned int acc_off, cnt_off, size_off, present_off, total;
  int svs;      // padded row stride of the shared-memory arrays (doubles)
  int nrep;     // table replicas (power of two <= 32): lane l of every warp works on replica l & (nrep - 1)
  int rstride;  // replica stride of acc / cnt in elements, = 1 (mod 16) so replicas sit in different banks
  int zstride;  // replica stride of the size array (odd)
};

// POS: FIRST / LAST tables -- the MIN / MAX code on row positions (FIRST = min, LAST = max), NULL value columns read
// as "no NaN" without a load.
template <bool POS>
__global__ void __launch_bounds__(kSmemThreads, 1) gb_accumulate_smem_kernel(const __grid_constant__ GbParams p,
                                                                             const SmemTableLayout lay) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* s_acc = reinterpret_cast<double*>(smem_raw + lay.acc_off);
  long long* s_acc_i = reinterpret_cast<long long*>(s_acc);
  unsigned int* s_cnt = reinterpret_cast<unsigned int*>(smem_raw + lay.cnt_off);
  unsigned int* s_size = reinterpret_cast<unsigned int*>(smem_raw + lay.size_off);
  unsigned char* s_present = smem_raw + lay.present_off;
  const int tid = threadIdx.x;
  const int nv = p.nvals, vs = p.vstride, svs = lay.svs;
  const int R = (int)p.gcap;
  const int nrep = lay.nrep, rstride = lay.rstride, zstride = lay.zstride;
  const bool f_sum = !POS && (p.flags & MB200_GB_SUM);
  const bool f_min = p.flags & (POS ? MB200_GB_FIRST : MB200_GB_MIN), f_max = p.flags & (POS ? MB200_GB_LAST : MB200_GB_MAX);
  const bool f_cnt = p.flags & MB200_GB_COUNT, f_size = p.flags & MB200_GB_SIZE;
  const bool has_acc = f_sum || f_min || f_max;
  const long long init = f_min ? 0x7fffffffffffffffLL : (f_max ? (long long)0x8000000000000000ULL : 0LL);
  for (int i = tid; i < nrep * rstride; i += kSmemThreads) {
    if (has_acc) s_acc_i[i] = init;
    if (f_cnt) s_cnt[i] = 0u;
  }
  if (f_size)
    for (int i = tid; i < nrep * zstride; i += kSmemThreads) s_size[i] = 0u;
  for (int i = tid; i < R; i += kSmemThreads) s_present[i] = 0;
  __syncthreads();
  const uint64_t pol = l2_policy_evict_first();
  const int rep = tid & (nrep - 1);
  const int rbase = rep * rstride;
  const long long stride = (long long)gridDim.x * kSmemThreads;
  for (long long row = (long long)blockIdx.x * kSmemThreads + tid; row < p.nrows; row += stride) {
    const long long key = ldg_stream_i64(p.keys + row, pol);
    double x[8];
    {
      const int nc = nv < 8 ? nv : 8;
#pragma unroll
      for (int c = 0; c < 8; ++c)
        x[c] = (c < nc && (!POS || p.vals[c])) ? ldg_stream_f64(static_cast<const double*>(p.vals[c]) + row, pol) : 0.0;
    }
    const unsigned long long d = (unsigned long long)key - (unsigned long long)p.kbase;
    if (d >= (unsigned long long)R) {
      p.meta->overflow = 1;  // key outside the declared range
      continue;
    }
    const int gid = (int)d;
    if (!s_present[gid]) s_present[gid] = 1;
    if (f_size) atomicAdd(&s_size[rep * zstride + gid], 1u);
    for (int c0 = 0; c0 < nv; c0 += 8) {
      const int nc = (nv - c0) < 8 ? (nv - c0) : 8;
      if (c0 > 0) {
#pragma unroll
        for (int c = 0; c < 8; ++c)
          x[c] = (c < nc && (!POS || p.vals[c0 + c])) ? ldg_stream_f64(static_cast<const double*>(p.vals[c0 + c]) + row, pol)
                                                      : 0.0;
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        if (c < nc && x[c] == x[c]) {
          const int o = rbase + gid * svs + c0 + c;
          if (f_sum) atomicAdd(&s_acc[o], x[c]);
          else if (f_min) atomicMin(&s_acc_i[o], POS ? p.row0 + row : f64_to_ordered(x[c]));
          else if (f_max) atomicMax(&s_acc_i[o], POS ? p.row0 + row : f64_to_ordered(x[c]));
          if (f_cnt) atomicAdd(&s_cnt[o], 1u);
        }
      }
    }
  }
  __syncthreads();
  // ---- fold the replicas and add this CTA's table to the global one (coalesced over the global [gid][vs] arrays)
  for (int i = tid; i < R * vs; i += kSmemThreads) {
    const int g = i / vs, cc = i - g * vs;
    if (cc >= nv || !s_present[g]) continue;
    const int o = g * svs + cc;
    if (f_sum) {
      double a = s_acc[o];
      for (int r = 1; r < nrep; ++r) a += s_acc[r * rstride + o];
      red_add_f64(p.acc + i, a);
    } else if (f_min || f_max) {
      long long a = s_acc_i[o];
      for (int r = 1; r < nrep; ++r) {
        const long long b = s_acc_i[r * rstride + o];
        a = f_min ? (b < a ? b : a) : (b > a ? b : a);
      }
      if (f_min && a != 0x7fffffffffffffffLL) red_min_s64(reinterpret_cast<long long*>(p.acc) + i, a);
      if (f_max && a != (long long)0x8000000000000000ULL) red_max_s64(reinterpret_cast<long long*>(p.acc) + i, a);
    }
    if (f_cnt) {
      long long n = 0;
      for (int r = 0; r < nrep; ++r) n += s_cnt[r * rstride + o];
      if (n) red_add_u64(p.cnt + i, n);
    }
  }
  for (int g = tid; g < R; g += kSmemThreads) {
    if (!s_present[g]) continue;
    reinterpret_cast<unsigned char*>(p.present)[g] = 1;
    if (f_size) {
      long long n = 0;
      for (int r = 0; r < nrep; ++r) n += s_size[r * zstride + g];
      red_add_u64(p.size + g, n);
    }
  }
}

__global__ void gb_fill_kernel(long long* p, long long n, long long v) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = v;
}

__global__ void gb_init_kernel(Slot* slots, long long cap, GbMeta* meta) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cap) {
    Slot s;
    s.key = 0;
    s.gid = -1;
    s.pad = 0;
    slots[i] = s;
  }
  if (i == 0) {
    meta->ngroups = 0;
    meta->overflow = 0;
    meta->kmin = 0x7fffffffffffffffLL;
    meta->kmax = (long long)0x8000000000000000ULL;
  }
}

// keys_by_gid[gid] = key ; perm[gid] = gid ; key range for the sort (one atomic pair per block)
__global__ void __launch_bounds__(256) gb_collect_kernel(const Slot* __restrict__ slots, long long cap, long long gcap,
                                                         long long* __restrict__ keys_by_gid,
                                                         long long* __restrict__ perm, GbMeta* meta) {
  __shared__ long long s_min[8], s_max[8];
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long lo = 0x7fffffffffffffffLL, hi = (long long)0x8000000000000000ULL;
  if (i < cap) {
    const Slot s = slots[i];
    if (s.gid >= 0 && s.gid < gcap) {
      keys_by_gid[s.gid] = s.key;
      perm[s.gid] = s.gid;
      lo = hi = s.key;
    }
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    const long long a = __shfl_xor_sync(0xffffffffu, lo, m), b = __shfl_xor_sync(0xffffffffu, hi, m);
    lo = a < lo ? a : lo;
    hi = b > hi ? b : hi;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    s_min[warp] = lo;
    s_max[warp] = hi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) {
      lo = s_min[w] < lo ? s_min[w] : lo;
      hi = s_max[w] > hi ? s_max[w] : hi;
    }
    if (lo <= hi) {
      atomicMin(&meta->kmin, lo);
      atomicMax(&meta->kmax, hi);
    }
  }
}

struct EmitParams {
  const int* count_dev;  // when set: the number of valid groups lives on the device (sync-free dense emit)
  const long long* keys_sorted;
  const long long* perm;
  const double* acc;
  const long long* cnt;
  const long long* size;
  int nvals;
  int vstride;
  int flags;
  long long ngroups;
  long long* out_keys;
  void* out_sums[MB200_MAX_COLS];
  void* out_cnts[MB200_MAX_COLS];
  long long* out_sizes;
};

__global__ void gb_emit_kernel(const __grid_constant__ EmitParams p) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.ngroups) return;
  if (p.count_dev && i >= (long long)*p.count_dev) return;
  const long long g = p.perm[i];
  if (p.out_keys) p.out_keys[i] = p.keys_sorted[i];
  if (p.out_sizes && p.size) p.out_sizes[i] = p.size[g];
  for (int v = 0; v < p.nvals; ++v) {
    if (p.out_sums[v] && p.acc) {
      double val = p.acc[(size_t)g * p.vstride + v];
      if (p.flags & (MB200_GB_FIRST | MB200_GB_LAST | MB200_GB_ARGMIN | MB200_GB_ARGMAX)) {
        // int64 position; -1: no non-NaN value in the group (every position table but LAST's starts at INT64_MAX)
        const long long o = __double_as_longlong(val);
        const bool empty = (p.flags & MB200_GB_LAST) ? (o == (long long)0x8000000000000000ULL) : (o == 0x7fffffffffffffffLL);
        val = __longlong_as_double(empty ? -1LL : o);
      } else if (p.flags & (MB200_GB_MIN | MB200_GB_MAX)) {
        const long long o = __double_as_longlong(val);
        const bool empty = (p.flags & MB200_GB_MIN) ? (o == 0x7fffffffffffffffLL) : (o == (long long)0x8000000000000000ULL);
        val = empty ? __longlong_as_double(0x7ff8000000000000LL) : ordered_to_f64(o);
      } else {
        val = val + 0.0;  // dense sums start from -0.0 (the "untouched" mark): an empty sum is +0.0 as in pandas
      }
      static_cast<double*>(p.out_sums[v])[i] = val;
    }
    if (p.out_cnts[v] && p.cnt) static_cast<long long*>(p.out_cnts[v])[i] = p.cnt[(size_t)g * p.vstride + v];
  }
}

// ---------------------------------------------------------------- dense tables: key range, ordered emit
// min / max (+ skew sample) of an int64 key column whose statistics are not known yet (a column that no
// stats-producing kernel of this library wrote): 8 x 128-bit streaming loads in flight per thread, one atomic
// quadruple per block.  The result is cached on the column by the caller (column metadata), so a column pays
// this 8 B/row pass at most once, not once per query.
__global__ void __launch_bounds__(256) key_range_kernel(const long long* __restrict__ keys, long long n,
                                                        long long* minmax) {
  KeyStatsAcc st;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  const long long head = (((uintptr_t)keys & 31u) == 0) ? (n & ~15LL) : 0;  // 16 keys per thread-iteration
  unsigned int iter = 0;
  for (long long i = tid * 4; i + 3 < head; i += nthreads * 16, ++iter) {
    i64x4 v[4];
    bool ok[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long j = i + (long long)u * nthreads * 4;
      ok[u] = j + 3 < head;
      if (ok[u]) v[u] = ldg_stream_i64x4(keys + j);
    }
    // skew statistic (every 4th iteration, whole warps only): how many of 32 sampled keys share their value
    // with another lane's.  Uniform keys over G values: ~ 496 / G of them; a heavy hitter at 10 %: > 80 %.
    if ((iter & 3u) == 0 && __activemask() == 0xffffffffu) st.sample_warp(v[0].x);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (!ok[u]) continue;
      st.add(v[u].x);
      st.add(v[u].y);
      st.add(v[u].z);
      st.add(v[u].w);
    }
  }
  for (long long i = head + tid; i < n; i += nthreads) st.add(keys[i]);
  st.flush(minmax);
}

__global__ void key_range_init_kernel(long long* minmax) {
  minmax[0] = 0x7fffffffffffffffLL;
  minmax[1] = (long long)0x8000000000000000ULL;
  minmax[2] = 0;  // keys sampled for the skew statistic
  minmax[3] = 0;  // ... of which shared their value with another of the 32 keys sampled with them
}

// shared with synth.cu (the generators that produce key columns fill the same quadruple)
int key_stats_init(long long* stats_dev, cudaStream_t st) {
  key_range_init_kernel<<<1, 1, 0, st>>>(stats_dev);
  MB_LAUNCH_CHECK("key_range_init_kernel");
  return 0;
}

// presence of a dense key = its byte was marked (rows that changed nothing) OR its accumulators moved
// away from their initial values.  Run before counting; idempotent.
__global__ void __launch_bounds__(256) dense_presence_kernel(unsigned char* __restrict__ present,
                                                             const long long* __restrict__ acc,
                                                             const long long* __restrict__ cnt,
                                                             const long long* __restrict__ size, long long g0,
                                                             long long g1, int nvals, int vstride, long long acc_init) {
  const long long g = g0 + (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= g1 || present[g]) return;
  bool seen = size && size[g] != 0;
  for (int v = 0; v < nvals && !seen; ++v) {
    if (acc && acc[g * vstride + v] != acc_init) seen = true;
    if (cnt && cnt[g * vstride + v] != 0) seen = true;
  }
  if (seen) present[g] = 1;
}

// block b counts the set bits of presence words [256 b, 256 b + 256)
__global__ void __launch_bounds__(256) dense_count_kernel(const unsigned int* __restrict__ present, long long nwords,
                                                          unsigned int* __restrict__ blockoff) {
  __shared__ unsigned int s[8];
  const long long w = (long long)blockIdx.x * 256 + threadIdx.x;
  unsigned int c = w < nwords ? __popc(present[w]) : 0u;
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) c += __shfl_xor_sync(0xffffffffu, c, m);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int t = 0;
    for (int i = 0; i < 8; ++i) t += s[i];
    blockoff[blockIdx.x] = t;
  }
}

// single block: exclusive scan of blockoff[0..nblocks) in place; total -> meta->ngroups
__global__ void __launch_bounds__(1024) dense_scan_kernel(unsigned int* blockoff, long long nblocks, GbMeta* meta) {
  __shared__ unsigned int s_part[1024];
  const int t = threadIdx.x;
  const long long per = (nblocks + 1023) / 1024;
  const long long lo = (long long)t * per, hi = (lo + per < nblocks) ? lo + per : nblocks;
  unsigned int sum = 0;
  for (long long i = lo; i < hi; ++i) sum += blockoff[i];
  s_part[t] = sum;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {  // Hillis-Steele inclusive scan
    const unsigned int v = (t >= off) ? s_part[t - off] : 0u;
    __syncthreads();
    s_part[t] += v;
    __syncthreads();
  }
  unsigned int run = s_part[t] - sum;
  for (long long i = lo; i < hi; ++i) {
    const unsigned int c = blockoff[i];
    blockoff[i] = run;
    run += c;
  }
  if (t == 1023) meta->ngroups = (int)s_part[1023];
}

// block b writes the keys / gids of its set bits at blockoff[b] + rank, in ascending key order
__global__ void __launch_bounds__(256) dense_fill_kernel(const unsigned int* __restrict__ present, long long nwords,
                                                         const unsigned int* __restrict__ blockoff, long long kbase,
                                                         long long gid0, long long* __restrict__ keys_out,
                                                         long long* __restrict__ perm_out, long long nout) {
  __shared__ unsigned int s[8];
  const long long w = (long long)blockIdx.x * 256 + threadIdx.x;
  unsigned int bits = w < nwords ? present[w] : 0u;
  const unsigned int c = __popc(bits);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned int incl = c;
#pragma unroll
  for (int m = 1; m < 32; m <<= 1) {
    const unsigned int v = __shfl_up_sync(0xffffffffu, incl, m);
    if (lane >= m) incl += v;
  }
  if (lane == 31) s[warp] = incl;
  __syncthreads();
  unsigned int base = blockoff[blockIdx.x];
  for (int i = 0; i < warp; ++i) base += s[i];
  long long o = (long long)base + incl - c;
  while (bits) {
    const int b = __ffs(bits) - 1;
    bits &= bits - 1;
    const long long g = gid0 + w * 4 + (b >> 3);  // presence bytes are 0 / 1: bit 8 j of a word = key 4 w + j
    if (o < nout) {
      keys_out[o] = kbase + g;
      perm_out[o] = g;
    }
    ++o;
  }
}

static long long next_pow2(long long v) {
  long long p = 1;
  while (p < v) p <<= 1;
  return p;
}

// The arrays a table of these flags has, and the int64 word each starts from ("no value yet").
//   acc: float64 sums, min / max as order-preserving images, or FIRST / LAST / ARG row positions.  Dense sums start
//        from -0.0, the one value no sum can end on (x + -0.0 = x, and the emit turns it into +0.0), so that a key whose
//        accumulators moved is present; hashed sums from 0.  Min, FIRST and ARG positions start from INT64_MAX, max and
//        LAST from INT64_MIN.
//   cnt: non-NaN counts from 0, or an ARG table's extreme images: from INT64_MIN for ARGMAX, INT64_MAX for ARGMIN.
//   size: rows per group, from 0.
struct TableArrays {
  bool acc, cnt, size;
  long long acc_init, cnt_init;
};
static TableArrays table_arrays(int flags, bool dense) {
  const long long lo = (long long)0x8000000000000000ULL, hi = 0x7fffffffffffffffLL;
  TableArrays a;
  a.acc = flags & (MB200_GB_SUM | MB200_GB_MIN | MB200_GB_MAX | MB200_GB_FIRST | MB200_GB_LAST | kGbArg);
  a.cnt = flags & (MB200_GB_COUNT | kGbArg);
  a.size = flags & MB200_GB_SIZE;
  a.acc_init = (flags & MB200_GB_SUM) ? (dense ? lo : 0) : (flags & (MB200_GB_MIN | MB200_GB_FIRST | kGbArg)) ? hi : lo;
  a.cnt_init = (flags & MB200_GB_ARGMAX) ? lo : (flags & MB200_GB_ARGMIN) ? hi : 0;
  return a;
}

// kernel parameters of table `t` over `nrows` rows of `keys`; the launchers add the value columns
static GbParams gb_params(const mb200_gb_table* t, const long long* keys, long long nrows) {
  GbParams p;
  memset(&p, 0, sizeof(p));
  p.slots = t->slots;
  p.mask = (unsigned int)(t->cap - 1);
  p.cap = t->cap;
  p.acc = t->acc;
  p.cnt = t->cnt;
  p.size = t->size;
  p.gcap = t->gcap;
  p.nvals = t->nvals;
  p.vstride = t->vstride;
  p.flags = t->flags;
  p.meta = t->meta;
  p.dense = t->dense;
  p.kbase = t->kbase;
  p.present = t->present;
  p.keys = keys;
  p.nrows = nrows;
  return p;
}

// MB200_GB_VARIANT=1 sends every row through the direct-load kernel; it is an on / off switch: unset or any other
// value, full tiles take the TMA-staged kernel wherever it applies.  Read per call so one process can compare the two.
// Measured on an H100 80GB HBM3 (400 W power limit), 2^27 rows, V = 8, fresh table per pass, uniform keys, ms TMA /
// direct: G = 65536 dense 5.3 / 6.1, hashed 6.4 / 7.2; G = 1e6 (64 MB dense, 96 MB hashed: both larger than the 50 MB
// L2) dense 13.6 / 13.4, hashed 21.5 / 21.9.  With skewed keys only the TMA kernel has the hot-group cache (6.1 ms
// against 81 at G = 1e6).  So the TMA kernel is taken at every size.
static bool gb_direct_only() {
  const char* e = getenv("MB200_GB_VARIANT");
  return e && e[0] == '1';
}

// MB200_GB_SMEM=0 keeps dense tables out of shared memory, so that small key ranges reach the global-table kernels
static bool gb_smem_tables() {
  const char* e = getenv("MB200_GB_SMEM");
  return !(e && e[0] == '0');
}

// direct-load kernels (gb_accumulate_kernel, gb_arg_kernel): as many CTAs as fit, but no more than one warp per 32 rows
template <typename... K, typename... A>
static int launch_direct(void (*kern)(GbParams, K...), const char* name, const GbParams& p, const DevProps& dp,
                         cudaStream_t st, A... args) {
  int occ = 0;
  MB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kGbThreads, 0));
  const long long nchunks = (p.nrows + 31) / 32;
  long long grid = (long long)dp.sm_count * (occ < 1 ? 1 : occ);
  const long long need = (nchunks + kGbWarps - 1) / kGbWarps;
  if (grid > need) grid = need;
  kern<<<(unsigned)grid, kGbThreads, 0, st>>>(p, args...);
  MB_LAUNCH_CHECK(name);
  return 0;
}

// shared-memory table kernels: one CTA per SM, but no more than the rows need
static unsigned smem_grid(long long nrows, const DevProps& dp) {
  const long long need = (nrows + kSmemThreads - 1) / kSmemThreads;
  return (unsigned)(dp.sm_count < need ? dp.sm_count : need);
}

// Shared-memory layout of table `t` with `nrep` replicas; returns its bytes.
typedef size_t (*SmemLayoutFn)(const mb200_gb_table* t, int nrep, SmemTableLayout* lay);

// accumulate tables: acc replicas (8 B) | cnt replicas (4 B) | size replicas (4 B) | presence bytes
static size_t smem_layout_accumulate(const mb200_gb_table* t, int nrep, SmemTableLayout* lay) {
  const TableArrays ta = table_arrays(t->flags, true);
  lay->svs = t->vstride + 1;
  lay->rstride = (int)((((size_t)t->gcap * lay->svs + 15) & ~(size_t)15) + 1);
  lay->zstride = (int)(t->gcap | 1);
  lay->nrep = nrep;
  const size_t elems = (size_t)nrep * lay->rstride;
  size_t off = 0;
  lay->acc_off = (unsigned)off;
  if (ta.acc) off += elems * 8;
  lay->cnt_off = (unsigned)off;
  if (ta.cnt) off += (elems * 4 + 15) & ~(size_t)15;
  lay->size_off = (unsigned)off;
  if (ta.size) off += (((size_t)nrep * lay->zstride * 4) + 15) & ~(size_t)15;
  lay->present_off = (unsigned)off;
  off += ((size_t)t->gcap + 15) & ~(size_t)15;
  lay->total = (unsigned)off;
  return off;
}

// ARG tables: image / position replicas (8 B) | the final images of pass 1 (8 B) | presence bytes
static size_t smem_layout_arg(const mb200_gb_table* t, int nrep, SmemTableLayout* lay) {
  memset(lay, 0, sizeof(*lay));
  lay->svs = t->vstride + 1;
  const size_t elems1 = (size_t)t->gcap * lay->svs;
  lay->rstride = (int)(((elems1 + 15) & ~(size_t)15) + 1);
  lay->nrep = nrep;
  size_t off = (((size_t)nrep * lay->rstride * 8) + 15) & ~(size_t)15;
  lay->cnt_off = (unsigned)off;
  off += elems1 * 8;
  lay->present_off = (unsigned)off;
  off += ((size_t)t->gcap + 15) & ~(size_t)15;
  lay->total = (unsigned)off;
  return off;
}

// Bytes of the layout with the most replicas (32, 16, ..., 1) that fits in shared memory; 0 when not even one does.
// Lanes of a warp that hit the same group then work on different copies: G = 16 runs 2.6x faster with 32 replicas
// than with one.
static size_t fit_replicas(SmemLayoutFn layout, const mb200_gb_table* t, const DevProps& dp, SmemTableLayout* lay) {
  for (int nrep = 32; nrep >= 1; nrep >>= 1) {
    const size_t bytes = layout(t, nrep, lay);
    if (bytes <= dp.smem_optin) return bytes;
  }
  return 0;
}

static int gb_launch(mb200_gb_table* t, const long long* keys, const void* const* vals, const void* const* pcnt,
                     const long long* psize, long long nrows, bool partial, cudaStream_t st) {
  if (nrows == 0) return 0;
  DevProps dp;
  if (int rc = dev_props(&dp)) return rc;
  GbParams p = gb_params(t, keys, nrows);
  const bool pos = t->flags & (MB200_GB_FIRST | MB200_GB_LAST);
  if (pos && partial) return fail("groupby", "FIRST / LAST tables do not merge partial tables");
  bool aligned = aligned16(keys);
  for (int c = 0; c < t->nvals; ++c) {
    p.vals[c] = vals ? vals[c] : nullptr;
    p.pcnt[c] = pcnt ? pcnt[c] : nullptr;
    if ((t->flags & (MB200_GB_SUM | MB200_GB_COUNT | MB200_GB_MIN | MB200_GB_MAX)) && !p.vals[c])
      return fail("groupby", "null value column");  // FIRST / LAST: NULL = a column without NaN
    if (partial && (t->flags & MB200_GB_COUNT) && !p.pcnt[c]) return fail("groupby", "null partial count column");
    aligned = aligned && aligned16(p.vals[c]);
  }
  if (pos) p.row0 = t->rows;
  else p.psize = psize;
  if (partial && (t->flags & MB200_GB_SIZE) && !psize) return fail("groupby", "null partial size column");

  // Pin the accumulator rows (the 2-sector RED target of every row) in the persisting L2 carve-out for the
  // kernels launched below (the carve-out size is the device's cudaDevAttrMaxPersistingL2CacheSize).
  //  * DENSE tables (default on for acc >= 8 MiB, MB200_GB_PERSIST=0 disables): the accumulators ARE the whole
  //    table; a table larger than the carve-out is pinned in the fraction that fits (hit ratio = carve-out /
  //    window).  The carve-out is released when the table is destroyed (l2_carveout_release) so later kernels
  //    get the whole L2 back.
  //  * HASH tables (opt-in, MB200_GB_PERSIST=1): the probe slots (32 MB at G = 1e6) do not fit next to the sums.
  struct WindowGuard {
    cudaStream_t st;
    bool on = false;
    ~WindowGuard() {
      if (on) {
        cudaStreamAttrValue v;
        memset(&v, 0, sizeof(v));
        cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &v);
      }
    }
  } guard{st};
  {
    const char* e = getenv("MB200_GB_PERSIST");
    const size_t acc_bytes = (size_t)t->gcap * t->vstride * 8;
    const bool off = e && e[0] == '0';
    // dense: the accumulators are the table.  hashed: the whole arena (slots | acc | cnt | size) -- with more
    // table than carve-out the window's hit ratio pins a random carve/arena share of its lines, which still turns
    // most probe and RED misses into hits (the streamed input is evict-first and cannot displace pinned lines).
    void* win_base = t->dense ? (void*)t->acc : t->arena;
    const size_t win_bytes = t->dense ? acc_bytes : t->arena_bytes;
    const bool want = !off && win_base && win_bytes >= ((size_t)8 << 20);
    if (want) {
      if (!t->persisted) {  // one carve-out reference per table, dropped in mb200_gb_destroy
        size_t mw = 0;
        const size_t mp = l2_carveout_acquire(&mw);
        if (mp) {
          t->persisted = 1;
          t->carve_bytes = mp;
          t->window_bytes = mw;
        }
      }
      if (t->persisted) {
        cudaStreamAttrValue v;
        memset(&v, 0, sizeof(v));
        v.accessPolicyWindow.base_ptr = win_base;
        v.accessPolicyWindow.num_bytes = win_bytes < t->window_bytes ? win_bytes : t->window_bytes;
        const double fit = (double)t->carve_bytes / (double)v.accessPolicyWindow.num_bytes;
        v.accessPolicyWindow.hitRatio = fit >= 1.0 ? 1.0f : (float)fit;
        v.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
        v.accessPolicyWindow.missProp = cudaAccessPropertyNormal;
        if (cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &v) == cudaSuccess) guard.on = true;
        else cudaGetLastError();
      }
    }
  }

  // low-cardinality dense tables: privatise the table in shared memory (MB200_GB_SMEM=0 disables)
  SmemTableLayout lay;
  const size_t table_smem = (t->dense && !partial && gb_smem_tables()) ? fit_replicas(smem_layout_accumulate, t, dp, &lay) : 0;
  if (table_smem) {
    auto kern = pos ? gb_accumulate_smem_kernel<true> : gb_accumulate_smem_kernel<false>;
    MB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)table_smem));
    kern<<<smem_grid(nrows, dp), kSmemThreads, table_smem, st>>>(p, lay);
    MB_LAUNCH_CHECK("gb_accumulate_smem_kernel");
    return 0;
  }
  if (!gb_direct_only() && !partial && aligned && t->nvals <= 8 && nrows >= kTileRows) {
    const long long ntiles = nrows / kTileRows;
    const bool hot = t->skewed && !(t->flags & (MB200_GB_MIN | MB200_GB_MAX | MB200_GB_FIRST | MB200_GB_LAST | MB200_GB_SIZE));
    // hashed tables: a 2-stage ring lets 5 CTAs share an SM instead of 4 (the probe chain wants warps, not staging depth)
    const bool two = !hot && !t->dense;
    const size_t smem = hot   ? (size_t)hot_offset(kHotStages) + ((t->flags & MB200_GB_COUNT) ? kHotBytes : kHotBytesSum)
                        : two ? (size_t)2 * kStageBytes + 2 * 2 * sizeof(uint64_t)
                              : (size_t)kGbStages * kStageBytes + 2 * kGbStages * sizeof(uint64_t);
    auto kern = hot   ? gb_accumulate_tma_kernel<true, kHotStages, false>
                : pos ? (two ? gb_accumulate_tma_kernel<false, 2, true> : gb_accumulate_tma_kernel<false, kGbStages, true>)
                : two ? gb_accumulate_tma_kernel<false, 2, false>
                      : gb_accumulate_tma_kernel<false, kGbStages, false>;
    MB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    MB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kGbTmaThreads, smem));
    long long grid = (long long)dp.sm_count * (occ < 1 ? 1 : occ);
    if (grid > ntiles) grid = ntiles;
    kern<<<(unsigned)grid, kGbTmaThreads, smem, st>>>(p, ntiles);
    MB_LAUNCH_CHECK("gb_accumulate_tma_kernel");
    const long long done = ntiles * kTileRows;
    if (done == nrows) return 0;
    // ragged tail (< 256 rows) goes through the direct-load kernel
    p.keys = keys + done;
    for (int c = 0; c < t->nvals; ++c)
      if (p.vals[c]) p.vals[c] = static_cast<const double*>(p.vals[c]) + done;
    p.row0 += done;
    p.nrows = nrows - done;
  }
  auto kern = pos       ? gb_accumulate_kernel<false, true>
              : partial ? gb_accumulate_kernel<true, false>
                        : gb_accumulate_kernel<false, false>;
  return launch_direct(kern, "gb_accumulate_kernel", p, dp, st);
}


// ---------------------------------------------------------------- ARGMIN / ARGMAX tables (groupby.idxmin / idxmax)
// Two passes over the same raw rows, on one stream.  Pass 1 takes, per (group, column), the min / max of the values'
// order-preserving int64 images into `cnt` (RED.MIN / MAX.S64, as min / max do); pass 2 takes the min of the positions
// of the rows whose image equals that final extreme into `acc`.  The extreme is unique and so is the smallest
// position holding it: the result is exact whatever the order of the atomics.  A float64 image folds -0.0 into +0.0
// (the two zeros tie, as in pandas); an int64 image is the value itself, so a group whose values all equal the
// "no value yet" sentinel (INT64_MIN for ARGMAX) still has rows equal to its extreme and resolves in pass 2.
// New kernels: the gb_accumulate* instantiations are untouched.
__device__ __forceinline__ bool arg_image(double x, bool i64, long long& img) {
  if (i64) {
    img = __double_as_longlong(x);
    return true;
  }
  if (x != x) return false;  // NaN: skipped
  img = (x == 0.0) ? 0LL : f64_to_ordered(x);
  return true;
}
__device__ __forceinline__ long long ld_relaxed_s64(const long long* p) {
  long long v;
  asm volatile("ld.relaxed.gpu.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// direct loads, dense or hashed tables: the mapping of gb_accumulate_kernel (warp = 32 rows, value tile transposed
// through shared memory, 8 lanes per row = 8 columns of one group's 64-byte row of the table)
// (pass 1 at 4 CTAs per SM: at 5 the 48-register budget spills around the insert path, as the accumulate kernel does)
template <int PASS>
__global__ void __launch_bounds__(kGbThreads, PASS == 1 ? 4 : 5) gb_arg_kernel(const __grid_constant__ GbParams p,
                                                                 const unsigned int i64_mask) {
  __shared__ double s_tile[kGbWarps][8 * kColStride];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long nchunks = (p.nrows + 31) >> 5;
  const long long wstride = (long long)gridDim.x * kGbWarps;
  const int gcap = (int)p.gcap;
  const uint64_t pol = l2_policy_evict_first();
  const bool amax = p.flags & MB200_GB_ARGMAX;
  long long* const img_tab = p.cnt;
  long long* const pos_tab = reinterpret_cast<long long*>(p.acc);
  for (long long ch = (long long)blockIdx.x * kGbWarps + warp; ch < nchunks; ch += wstride) {
    const long long base = ch << 5;
    const long long row = base + lane;
    const bool valid = row < p.nrows;
    long long k = valid ? ldg_stream_i64(p.keys + row, pol) : 0;
    double x[8];
    {
      const int nc = p.nvals < 8 ? p.nvals : 8;
#pragma unroll
      for (int c = 0; c < 8; ++c)
        x[c] = (c < nc && valid) ? ldg_stream_f64(static_cast<const double*>(p.vals[c]) + row, pol) : 0.0;
    }
    {
      const long long k0 = __shfl_sync(0xffffffffu, k, 0);  // rows past the end join lane 0's peer group
      k = valid ? k : k0;
    }
    const int gid = resolve_gid(p, k);  // pass 2: every key is in the table already, nothing is inserted
    if (PASS == 1 && p.dense && p.nvals == 0 && valid && gid < gcap) dense_mark(p, gid);
    for (int c0 = 0; c0 < p.nvals; c0 += 8) {
      const int nc = (p.nvals - c0) < 8 ? (p.nvals - c0) : 8;
      if (c0 > 0) {
#pragma unroll
        for (int c = 0; c < 8; ++c)
          x[c] = (c < nc && valid) ? ldg_stream_f64(static_cast<const double*>(p.vals[c0 + c]) + row, pol) : 0.0;
      }
      double* tile = s_tile[warp];
#pragma unroll
      for (int c = 0; c < 8; ++c) tile[c * kColStride + lane] = x[c];
      __syncwarp();
      const int c = lane & 7;
      const bool is_i64 = c < nc && ((i64_mask >> (c0 + c)) & 1u);
      unsigned int seen = 0, rowok = 0;
      int gs[8];
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const int r = 4 * kk + (lane >> 3);
        const int g = __shfl_sync(0xffffffffu, gid, r);
        const double xv = tile[c * kColStride + r];
        const bool rok = (base + r < p.nrows) && g < gcap;
        gs[kk] = g;
        if (rok) rowok |= 1u << kk;
        long long img;
        if (rok && c < nc && arg_image(xv, is_i64, img)) {
          const size_t o = (size_t)g * p.vstride + c0 + c;
          if (PASS == 1) {
            seen |= 1u << kk;
            if (amax) red_max_s64(img_tab + o, img);
            else red_min_s64(img_tab + o, img);
          } else if (img == __ldg(img_tab + o)) {
            // positions only fall: a row at or past the current minimum cannot win, and skipping it keeps a run of
            // equal extremes (bool columns, few distinct int64 values) from serialising on one address
            const long long pos = base + r;
            if (pos < ld_relaxed_s64(pos_tab + o)) red_min_s64(pos_tab + o, pos);
          }
        }
      }
      if (PASS == 1 && p.dense) {  // rows without a value in these columns mark their presence byte
        seen |= __shfl_xor_sync(0xffffffffu, seen, 1);
        seen |= __shfl_xor_sync(0xffffffffu, seen, 2);
        seen |= __shfl_xor_sync(0xffffffffu, seen, 4);
        const unsigned int unseen = ~seen & rowok;
        if (c == 0 && unseen) {
#pragma unroll
          for (int kk = 0; kk < 8; ++kk)
            if ((unseen >> kk) & 1u) dense_mark(p, gs[kk]);
        }
      }
      __syncwarp();
    }
  }
}

// low-cardinality dense tables (the ranges gb_accumulate_smem_kernel serves): per-CTA shared-memory tables.
// Pass 1: shared atomics on the images in `nrep` replicas (lane l of a warp works on replica l & (nrep - 1)), folded
// into the global images once per CTA; every row marks its key present.  Pass 2: each CTA loads the final images of
// the range into shared memory and takes the position minimum in the replicas, folded into the global positions once.
// Layout: acc_off = replicas (images in pass 1, positions in pass 2), cnt_off = the final images (pass 2), present_off.
template <int PASS>
__global__ void __launch_bounds__(kSmemThreads, 1) gb_arg_smem_kernel(const __grid_constant__ GbParams p,
                                                                        const SmemTableLayout lay,
                                                                        const unsigned int i64_mask) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  long long* s_rep = reinterpret_cast<long long*>(smem_raw + lay.acc_off);
  long long* s_img = reinterpret_cast<long long*>(smem_raw + lay.cnt_off);
  unsigned char* s_present = smem_raw + lay.present_off;
  const int tid = threadIdx.x;
  const int nv = p.nvals, vs = p.vstride, svs = lay.svs;
  const int R = (int)p.gcap;
  const int nrep = lay.nrep, rstride = lay.rstride;
  const bool amax = p.flags & MB200_GB_ARGMAX;
  const long long init = (PASS == 1 && amax) ? (long long)0x8000000000000000ULL : 0x7fffffffffffffffLL;
  for (int i = tid; i < nrep * rstride; i += kSmemThreads) s_rep[i] = init;
  if (PASS == 1) {
    for (int i = tid; i < R; i += kSmemThreads) s_present[i] = 0;
  } else {
    for (int i = tid; i < R * vs; i += kSmemThreads) {
      const int g = i / vs, cc = i - g * vs;
      if (cc < nv) s_img[g * svs + cc] = p.cnt[i];
    }
  }
  __syncthreads();
  const uint64_t pol = l2_policy_evict_first();
  const int rbase = (tid & (nrep - 1)) * rstride;
  const long long stride = (long long)gridDim.x * kSmemThreads;
  for (long long row = (long long)blockIdx.x * kSmemThreads + tid; row < p.nrows; row += stride) {
    const long long key = ldg_stream_i64(p.keys + row, pol);
    double x[8];
    {
      const int nc = nv < 8 ? nv : 8;
#pragma unroll
      for (int c = 0; c < 8; ++c) x[c] = (c < nc) ? ldg_stream_f64(static_cast<const double*>(p.vals[c]) + row, pol) : 0.0;
    }
    const unsigned long long d = (unsigned long long)key - (unsigned long long)p.kbase;
    if (d >= (unsigned long long)R) {
      p.meta->overflow = 1;  // key outside the declared range
      continue;
    }
    const int gid = (int)d;
    if (PASS == 1 && !s_present[gid]) s_present[gid] = 1;
    for (int c0 = 0; c0 < nv; c0 += 8) {
      const int nc = (nv - c0) < 8 ? (nv - c0) : 8;
      if (c0 > 0) {
#pragma unroll
        for (int c = 0; c < 8; ++c)
          x[c] = (c < nc) ? ldg_stream_f64(static_cast<const double*>(p.vals[c0 + c]) + row, pol) : 0.0;
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        long long img;
        if (c < nc && arg_image(x[c], (i64_mask >> (c0 + c)) & 1u, img)) {
          const int o = gid * svs + c0 + c;
          if (PASS == 1) {
            if (amax) atomicMax(&s_rep[rbase + o], img);
            else atomicMin(&s_rep[rbase + o], img);
          } else if (img == s_img[o] && row < s_rep[rbase + o]) {
            atomicMin(&s_rep[rbase + o], row);
          }
        }
      }
    }
  }
  __syncthreads();
  for (int i = tid; i < R * vs; i += kSmemThreads) {
    const int g = i / vs, cc = i - g * vs;
    if (cc >= nv || (PASS == 1 && !s_present[g])) continue;
    const int o = g * svs + cc;
    long long a = s_rep[o];
    for (int r = 1; r < nrep; ++r) {
      const long long b = s_rep[r * rstride + o];
      a = (PASS == 1 && amax) ? (b > a ? b : a) : (b < a ? b : a);
    }
    if (a == init) continue;
    if (PASS == 2) red_min_s64(reinterpret_cast<long long*>(p.acc) + i, a);
    else if (amax) red_max_s64(p.cnt + i, a);
    else red_min_s64(p.cnt + i, a);
  }
  if (PASS == 1)
    for (int g = tid; g < R; g += kSmemThreads)
      if (s_present[g]) reinterpret_cast<unsigned char*>(p.present)[g] = 1;
}

static int gb_arg_launch(mb200_gb_table* t, const long long* keys, const void* const* vals, unsigned int i64_mask,
                         long long nrows, cudaStream_t st) {
  if (nrows == 0) return 0;
  DevProps dp;
  if (int rc = dev_props(&dp)) return rc;
  GbParams p = gb_params(t, keys, nrows);
  for (int c = 0; c < t->nvals; ++c) {
    p.vals[c] = vals[c];
    if (!p.vals[c]) return fail("mb200_gb_accumulate_arg", "null value column");
  }
  SmemTableLayout lay;
  const size_t table_smem = (t->dense && gb_smem_tables()) ? fit_replicas(smem_layout_arg, t, dp, &lay) : 0;
  if (table_smem) {
    const unsigned grid = smem_grid(nrows, dp);
    MB_CUDA(cudaFuncSetAttribute(gb_arg_smem_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)table_smem));
    MB_CUDA(cudaFuncSetAttribute(gb_arg_smem_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)table_smem));
    gb_arg_smem_kernel<1><<<grid, kSmemThreads, table_smem, st>>>(p, lay, i64_mask);
    MB_LAUNCH_CHECK("gb_arg_smem_kernel");
    gb_arg_smem_kernel<2><<<grid, kSmemThreads, table_smem, st>>>(p, lay, i64_mask);
    MB_LAUNCH_CHECK("gb_arg_smem_kernel");
    return 0;
  }
  if (int rc = launch_direct(gb_arg_kernel<1>, "gb_arg_kernel", p, dp, st, i64_mask)) return rc;
  return launch_direct(gb_arg_kernel<2>, "gb_arg_kernel", p, dp, st, i64_mask);
}

}  // namespace mb200

using namespace mb200;

struct DenseArrays {  // caller-owned arrays of a dense table (all NULL: the library allocates)
  void* acc;
  void* cnt;
  void* size;
  void* present;
};

static int gb_create_impl(mb200_gb_table** table, int64_t group_capacity, int nvals, int flags, bool dense,
                          int64_t kbase, const DenseArrays& ext, mb200_stream_t stream, bool init_arrays = true);

extern "C" int mb200_gb_create(mb200_gb_table** table, int64_t group_capacity, int nvals, int flags,
                               mb200_stream_t stream) {
  return gb_create_impl(table, group_capacity, nvals, flags, false, 0, DenseArrays{}, stream);
}

// Arguments of a dense table over [key_min, key_max]: a range of at most 2^29 keys (left in *range) and, when the
// caller owns the arrays (`borrowed`), the presence array and every other array the flags need, all 16-byte aligned.
// Arrays given without the presence array are refused.
static int check_dense_args(const char* fn, int64_t key_min, int64_t key_max, int flags, const DenseArrays& ext,
                            bool borrowed, int64_t* range) {
  if (key_max < key_min) return fail(fn, "empty key range");
  const unsigned long long r = (unsigned long long)key_max - (unsigned long long)key_min + 1ULL;
  if (r == 0 || r > (1ULL << 29)) return fail(fn, "key range above 2^29");
  *range = (int64_t)r;
  if (!borrowed) return (ext.acc || ext.cnt || ext.size) ? fail(fn, "caller-owned arrays need the presence array too") : 0;
  const TableArrays ta = table_arrays(flags, true);
  if (!ext.present || (ta.acc && !ext.acc) || (ta.cnt && !ext.cnt) || (ta.size && !ext.size))
    return fail(fn, "caller-owned arrays: every array the flags need must be given");
  if (!aligned16(ext.acc) || !aligned16(ext.cnt) || !aligned16(ext.size) || !aligned16(ext.present))
    return fail(fn, "caller-owned arrays must be 16-byte aligned");
  return 0;
}

extern "C" int mb200_gb_create_dense(mb200_gb_table** table, int64_t key_min, int64_t key_max, int nvals, int flags,
                                     void* acc, void* cnt, void* size, void* present, mb200_stream_t stream) {
  const DenseArrays ext{acc, cnt, size, present};
  int64_t range;
  if (int rc = check_dense_args("mb200_gb_create_dense", key_min, key_max, flags, ext, present != nullptr, &range))
    return rc;
  return gb_create_impl(table, range, nvals, flags, true, key_min, ext, stream);
}

namespace mb200 {
__global__ void gb_inherit_overflow_kernel(GbMeta* child, const GbMeta* parent) {
  if (parent->overflow) child->overflow = 1;
}
}  // namespace mb200

extern "C" int mb200_gb_adopt_dense(mb200_gb_table** table, int64_t key_min, int64_t key_max, int nvals, int flags,
                                    void* acc, void* cnt, void* size, void* present, const mb200_gb_table* parent,
                                    mb200_stream_t stream) {
  const DenseArrays ext{acc, cnt, size, present};
  int64_t range;
  if (int rc = check_dense_args("mb200_gb_adopt_dense", key_min, key_max, flags, ext, true, &range)) return rc;
  if (int rc = gb_create_impl(table, range, nvals, flags, true, key_min, ext, stream, /*init_arrays=*/false))
    return rc;
  if (parent) {
    gb_inherit_overflow_kernel<<<1, 1, 0, (cudaStream_t)stream>>>((*table)->meta, parent->meta);
    MB_LAUNCH_CHECK("gb_inherit_overflow_kernel");
  }
  return 0;
}

extern "C" int mb200_gb_hint_skew(mb200_gb_table* t, int skewed) {
  if (!t) return fail("mb200_gb_hint_skew", "null table");
  t->skewed = skewed ? 1 : 0;
  return 0;
}

extern "C" int mb200_gb_dense_window(mb200_gb_table* t, int64_t gid_lo, int64_t gid_hi) {
  if (!t || !t->dense) return fail("mb200_gb_dense_window", "not a dense table");
  if (gid_lo < 0 || gid_hi < gid_lo || gid_hi > t->gcap || (gid_lo & 3) || ((gid_hi & 3) && gid_hi != t->gcap))
    return fail("mb200_gb_dense_window", "window must be [lo, hi) within the range, lo and hi multiples of 4");
  t->win_lo = gid_lo;
  t->win_hi = gid_hi;
  return 0;
}

extern "C" int mb200_key_range(const int64_t* keys, int64_t nrows, int64_t* minmax_dev, int init,
                               mb200_stream_t stream) {
  if (!minmax_dev) return fail("mb200_key_range", "null output");
  if (nrows < 0) return fail("mb200_key_range", "negative nrows");
  if (nrows > 0 && !keys) return fail("mb200_key_range", "null keys");
  DevProps dp;
  if (int rc = dev_props(&dp)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (init)
    if (int rc = key_stats_init(reinterpret_cast<long long*>(minmax_dev), st)) return rc;
  if (nrows == 0) return 0;
  long long grid = (long long)dp.sm_count * 8;
  const long long need = (nrows + 256 * 16 - 1) / (256 * 16);
  if (grid > need) grid = need;
  key_range_kernel<<<(unsigned)grid, 256, 0, st>>>(reinterpret_cast<const long long*>(keys), nrows,
                                                  reinterpret_cast<long long*>(minmax_dev));
  MB_LAUNCH_CHECK("key_range_kernel");
  return 0;
}

static int gb_create_impl(mb200_gb_table** table, int64_t group_capacity, int nvals, int flags, bool dense,
                          int64_t kbase, const DenseArrays& ext, mb200_stream_t stream, bool init_arrays) {
  if (!table) return fail("mb200_gb_create", "null out pointer");
  if (nvals < 0 || nvals > MB200_MAX_COLS) return fail("mb200_gb_create", "nvals out of range (0..32)");
  if (group_capacity < 1) group_capacity = 1;
  if (group_capacity > (1LL << 29)) return fail("mb200_gb_create", "group capacity above 2^29");
  if ((flags & (MB200_GB_FIRST | MB200_GB_LAST)) &&
      (flags & (MB200_GB_SUM | MB200_GB_COUNT | MB200_GB_MIN | MB200_GB_MAX) ||
       (flags & (MB200_GB_FIRST | MB200_GB_LAST)) == (MB200_GB_FIRST | MB200_GB_LAST)))
    return fail("mb200_gb_create", "FIRST / LAST exclude every other accumulator flag");
  if ((flags & kGbArg) && flags != MB200_GB_ARGMIN && flags != MB200_GB_ARGMAX)
    return fail("mb200_gb_create", "ARGMIN / ARGMAX exclude every other flag");
  DevProps dp;
  if (int rc = dev_props(&dp)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  mb200_gb_table* t = new mb200_gb_table();
  memset(t, 0, sizeof(*t));
  t->gcap = group_capacity;
  t->cap = dense ? 0 : next_pow2(2 * group_capacity < 1024 ? 1024 : 2 * group_capacity);
  t->dense = dense ? 1 : 0;
  t->kbase = kbase;
  t->win_lo = 0;
  t->win_hi = group_capacity;
  t->borrowed = (dense && ext.present) ? 1 : 0;
  t->nwords = dense ? (group_capacity + 3) / 4 : 0;  // one presence byte per key, scanned as 32-bit words
  t->nvals = nvals;
  t->vstride = (nvals + 3) & ~3;  // 32-byte sector aligned rows
  if (t->vstride == 0) t->vstride = 4;
  t->flags = flags;
  cudaError_t e;
  const size_t accb = (size_t)t->gcap * t->vstride * 8;
  const TableArrays ta = table_arrays(flags, dense);
  // allocates a dense array the caller does not own, then sets every word to `init`: a memset for 0, the fill kernel
  // for anything else (INT64_MAX = bytes ff..ff 7f is not a byte pattern)
  auto init_array = [&](void** arr, size_t bytes, long long init) -> cudaError_t {
    if (dense && !t->borrowed)
      if (cudaError_t err = cudaMallocAsync(arr, bytes, st)) return err;
    if (init == 0) return cudaMemsetAsync(*arr, 0, bytes, st);
    gb_fill_kernel<<<(unsigned)dp.sm_count * 4, 256, 0, st>>>(static_cast<long long*>(*arr), (long long)(bytes / 8), init);
    const cudaError_t err = cudaGetLastError();
    if (err == cudaSuccess) g_launches.fetch_add(1);
    return err;
  };
#define MB_TRY(call)                \
  do {                              \
    e = (call);                     \
    if (e != cudaSuccess) goto bad; \
  } while (0)
  if (t->borrowed) {  // arrays live in the caller's allocator (so that it can run collectives on them)
    t->present = static_cast<unsigned int*>(ext.present);
    t->acc = static_cast<double*>(ext.acc);
    t->cnt = static_cast<long long*>(ext.cnt);
    t->size = static_cast<long long*>(ext.size);
  }
  if (dense) {
    if (!t->borrowed) MB_TRY(cudaMallocAsync((void**)&t->present, (size_t)t->nwords * 4, st));
    if (init_arrays) MB_TRY(cudaMemsetAsync(t->present, 0, (size_t)t->nwords * 4, st));
    MB_TRY(cudaMallocAsync((void**)&t->blockoff, (size_t)((t->nwords + 255) / 256 + 1) * 4, st));
  } else {
    const size_t slot_b = ((size_t)t->cap * sizeof(Slot) + 255) & ~(size_t)255;
    const size_t acc_b = (accb + 255) & ~(size_t)255;
    const size_t size_b = (((size_t)t->gcap * 8) + 255) & ~(size_t)255;
    t->arena_bytes = slot_b + (ta.acc ? acc_b : 0) + (ta.cnt ? acc_b : 0) + (ta.size ? size_b : 0);
    MB_TRY(cudaMallocAsync(&t->arena, t->arena_bytes, st));
    char* a = static_cast<char*>(t->arena);
    t->slots = reinterpret_cast<Slot*>(a);
    a += slot_b;
    if (ta.acc) {
      t->acc = reinterpret_cast<double*>(a);
      a += acc_b;
    }
    if (ta.cnt) {
      t->cnt = reinterpret_cast<long long*>(a);
      a += acc_b;
    }
    if (ta.size) t->size = reinterpret_cast<long long*>(a);
  }
  MB_TRY(cudaMallocAsync((void**)&t->meta, sizeof(GbMeta), st));
  // adopted arrays (mb200_gb_adopt_dense) already hold a merged table: nothing to initialise
  if (init_arrays) {
    if (ta.acc) MB_TRY(init_array((void**)&t->acc, accb, ta.acc_init));
    if (ta.cnt) MB_TRY(init_array((void**)&t->cnt, accb, ta.cnt_init));
    if (ta.size) MB_TRY(init_array((void**)&t->size, (size_t)t->gcap * 8, 0));
  }
#undef MB_TRY
  gb_init_kernel<<<(unsigned)(dense ? 1 : (t->cap + 255) / 256), 256, 0, st>>>(t->slots, t->cap, t->meta);
  e = cudaGetLastError();
  if (e != cudaSuccess) goto bad;
  g_launches.fetch_add(1);
  *table = t;
  return 0;
bad:
  mb200_gb_destroy(t, stream);
  return cuda_fail("mb200_gb_create", e);
}

extern "C" int mb200_gb_destroy(mb200_gb_table* t, mb200_stream_t stream) {
  if (!t) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (t->arena) cudaFreeAsync(t->arena, st);
  if (t->meta) cudaFreeAsync(t->meta, st);
  if (!t->borrowed && !t->arena) {
    if (t->acc) cudaFreeAsync(t->acc, st);
    if (t->cnt) cudaFreeAsync(t->cnt, st);
    if (t->size) cudaFreeAsync(t->size, st);
    if (t->present) cudaFreeAsync(t->present, st);
  }
  if (t->blockoff) cudaFreeAsync(t->blockoff, st);
  if (t->persisted) l2_carveout_release();  // the last table hands the carve-out back to normally managed L2
  delete t;
  return 0;
}

/* number of bytes the device can pin in L2 (diagnostics for the persisting-window experiment) */
extern "C" int mb200_l2_persist_info(int* max_persist_bytes, int* max_window_bytes) {
  int dev = 0;
  MB_CUDA(cudaGetDevice(&dev));
  if (max_persist_bytes) MB_CUDA(cudaDeviceGetAttribute(max_persist_bytes, cudaDevAttrMaxPersistingL2CacheSize, dev));
  if (max_window_bytes) MB_CUDA(cudaDeviceGetAttribute(max_window_bytes, cudaDevAttrMaxAccessPolicyWindowSize, dev));
  return 0;
}

extern "C" int mb200_gb_accumulate(mb200_gb_table* t, const int64_t* keys, const void* const* vals,
                                   int64_t nrows, mb200_stream_t stream) {
  if (!t) return fail("mb200_gb_accumulate", "null table");
  if (nrows < 0) return fail("mb200_gb_accumulate", "negative nrows");
  if (nrows > 0 && !keys) return fail("mb200_gb_accumulate", "null keys");
  if (t->flags & kGbArg) return fail("mb200_gb_accumulate", "ARGMIN / ARGMAX tables take mb200_gb_accumulate_arg");
  if (int rc = gb_launch(t, reinterpret_cast<const long long*>(keys), vals, nullptr, nullptr, nrows, false,
                         (cudaStream_t)stream))
    return rc;
  t->rows += nrows;
  return 0;
}

extern "C" int mb200_gb_merge_partial(mb200_gb_table* t, const int64_t* keys, const void* const* sums,
                                      const void* const* cnts, const int64_t* sizes, int64_t npartial,
                                      mb200_stream_t stream) {
  if (!t) return fail("mb200_gb_merge_partial", "null table");
  if (npartial < 0) return fail("mb200_gb_merge_partial", "negative npartial");
  if (npartial > 0 && !keys) return fail("mb200_gb_merge_partial", "null keys");
  if (t->flags & kGbArg) return fail("mb200_gb_merge_partial", "ARGMIN / ARGMAX tables do not merge partial tables");
  return gb_launch(t, reinterpret_cast<const long long*>(keys), sums, cnts, reinterpret_cast<const long long*>(sizes),
                   npartial, true, (cudaStream_t)stream);
}

extern "C" int mb200_gb_accumulate_arg(mb200_gb_table* t, const int64_t* keys, const void* const* vals,
                                       uint32_t i64_mask, int64_t nrows, mb200_stream_t stream) {
  if (!t) return fail("mb200_gb_accumulate_arg", "null table");
  if (!(t->flags & kGbArg)) return fail("mb200_gb_accumulate_arg", "not an ARGMIN / ARGMAX table");
  if (t->arg_filled) return fail("mb200_gb_accumulate_arg", "an ARGMIN / ARGMAX table is filled by one call");
  if (nrows < 0) return fail("mb200_gb_accumulate_arg", "negative nrows");
  if (nrows > 0 && !keys) return fail("mb200_gb_accumulate_arg", "null keys");
  if (nrows > 0 && t->nvals > 0 && !vals) return fail("mb200_gb_accumulate_arg", "null value columns");
  if (int rc = gb_arg_launch(t, reinterpret_cast<const long long*>(keys), vals, i64_mask, nrows, (cudaStream_t)stream))
    return rc;
  t->arg_filled = 1;
  t->rows = nrows;
  return 0;
}

static int dense_finalize_presence(mb200_gb_table* t, cudaStream_t st) {
  const long long n = t->win_hi - t->win_lo;
  if (n <= 0) return 0;
  // ARGMIN / ARGMAX: cnt holds images, not counts; presence is a moved position or a marked byte
  dense_presence_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
      reinterpret_cast<unsigned char*>(t->present), reinterpret_cast<const long long*>(t->acc),
      (t->flags & kGbArg) ? nullptr : t->cnt, t->size,
      t->win_lo, t->win_hi, t->nvals, t->vstride, table_arrays(t->flags, true).acc_init);
  MB_LAUNCH_CHECK("dense_presence_kernel");
  return 0;
}

extern "C" int mb200_gb_ngroups(mb200_gb_table* t, int64_t* ngroups, int* overflow, mb200_stream_t stream) {
  if (!t) return fail("mb200_gb_ngroups", "null table");
  if (t->dense) {  // count the presence bytes of the window
    if (int rc = dense_finalize_presence(t, (cudaStream_t)stream)) return rc;
    const long long w0 = t->win_lo / 4, nw = (t->win_hi - t->win_lo + 3) / 4;
    const long long nblocks = nw > 0 ? (nw + 255) / 256 : 1;
    dense_count_kernel<<<(unsigned)nblocks, 256, 0, (cudaStream_t)stream>>>(t->present + w0, nw, t->blockoff);
    MB_LAUNCH_CHECK("dense_count_kernel");
    dense_scan_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(t->blockoff, nblocks, t->meta);
    MB_LAUNCH_CHECK("dense_scan_kernel");
  }
  GbMeta m;
  MB_CUDA(cudaMemcpyAsync(&m, t->meta, sizeof(m), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  MB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  long long n = m.ngroups;
  if (n > t->gcap) n = t->gcap;
  if (ngroups) *ngroups = n;
  if (overflow) *overflow = m.overflow;
  return 0;
}

extern "C" size_t mb200_gb_emit_scratch_bytes(int64_t ngroups) {
  if (ngroups < 1) ngroups = 1;
  // keys_by_gid + perm (2 * 8 * n) + sort scratch
  return (size_t)ngroups * 16 + 512 + sort_scratch_bytes(ngroups);
}

namespace mb200 {
__global__ void gb_export_meta_kernel(const GbMeta* meta, long long* out2) {
  out2[0] = meta->ngroups;
  out2[1] = meta->overflow;
}
}  // namespace mb200

static int gb_emit_impl(mb200_gb_table* t, int64_t ngroups, int sort, int64_t* out_keys, void* const* out_sums,
                        void* const* out_cnts, int64_t* out_sizes, void* scratch, int64_t* count_overflow_dev,
                        mb200_stream_t stream);

extern "C" int mb200_gb_emit(mb200_gb_table* t, int64_t ngroups, int sort, int64_t* out_keys,
                             void* const* out_sums, void* const* out_cnts, int64_t* out_sizes, void* scratch,
                             mb200_stream_t stream) {
  return gb_emit_impl(t, ngroups, sort, out_keys, out_sums, out_cnts, out_sizes, scratch, nullptr, stream);
}

extern "C" int mb200_gb_emit_dense_async(mb200_gb_table* t, int64_t capacity, int64_t* out_keys, void* const* out_sums,
                                         void* const* out_cnts, int64_t* out_sizes, void* scratch,
                                         int64_t* count_overflow_dev, mb200_stream_t stream) {
  if (!t || !t->dense) return fail("mb200_gb_emit_dense_async", "not a dense table");
  if (!count_overflow_dev) return fail("mb200_gb_emit_dense_async", "null count output");
  if (capacity < t->win_hi - t->win_lo) return fail("mb200_gb_emit_dense_async", "capacity below the window size");
  return gb_emit_impl(t, capacity, 0, out_keys, out_sums, out_cnts, out_sizes, scratch, count_overflow_dev, stream);
}

static int gb_emit_impl(mb200_gb_table* t, int64_t ngroups, int sort, int64_t* out_keys, void* const* out_sums,
                        void* const* out_cnts, int64_t* out_sizes, void* scratch, int64_t* count_overflow_dev,
                        mb200_stream_t stream) {
  if (!t) return fail("mb200_gb_emit", "null table");
  if (ngroups < 0 || ngroups > t->gcap) return fail("mb200_gb_emit", "ngroups out of range");
  if (ngroups == 0) return 0;
  if (!scratch) return fail("mb200_gb_emit", "null scratch");
  cudaStream_t st = (cudaStream_t)stream;
  char* s = static_cast<char*>(scratch);
  long long* keys_by_gid = reinterpret_cast<long long*>(s);
  long long* perm = reinterpret_cast<long long*>(s + (size_t)ngroups * 8);
  size_t off = ((size_t)ngroups * 16 + 255) & ~(size_t)255;
  char* sort_s = s + off;
  GbMeta m;
  memset(&m, 0, sizeof(m));
  if (t->dense) {
    // presence bits -> (key, gid) lists, already in ascending key order: no collect, no sort, and no host
    // round trip (mb200_gb_ngroups reported the overflow flag when the caller sized the outputs)
    if (int rc = dense_finalize_presence(t, st)) return rc;
    const long long w0 = t->win_lo / 4, nw = (t->win_hi - t->win_lo + 3) / 4;
    const long long nblocks = nw > 0 ? (nw + 255) / 256 : 1;
    dense_count_kernel<<<(unsigned)nblocks, 256, 0, st>>>(t->present + w0, nw, t->blockoff);
    MB_LAUNCH_CHECK("dense_count_kernel");
    dense_scan_kernel<<<1, 1024, 0, st>>>(t->blockoff, nblocks, t->meta);
    MB_LAUNCH_CHECK("dense_scan_kernel");
    dense_fill_kernel<<<(unsigned)nblocks, 256, 0, st>>>(t->present + w0, nw, t->blockoff, t->kbase, t->win_lo,
                                                        keys_by_gid, perm, ngroups);
    MB_LAUNCH_CHECK("dense_fill_kernel");
    sort = 0;
  } else {
    gb_collect_kernel<<<(unsigned)((t->cap + 255) / 256), 256, 0, st>>>(t->slots, t->cap, t->gcap, keys_by_gid, perm,
                                                                        t->meta);
    MB_LAUNCH_CHECK("gb_collect_kernel");
    MB_CUDA(cudaMemcpyAsync(&m, t->meta, sizeof(m), cudaMemcpyDeviceToHost, st));
    MB_CUDA(cudaStreamSynchronize(st));
    if (m.overflow) return fail("mb200_gb_emit", "table overflowed: recreate with a larger group capacity");
  }
  if (sort) {
    long long* tk = reinterpret_cast<long long*>(sort_s);
    long long* tp = reinterpret_cast<long long*>(sort_s + (size_t)ngroups * 8);
    size_t coff = ((size_t)ngroups * 16 + 255) & ~(size_t)255;
    unsigned int* counts = reinterpret_cast<unsigned int*>(sort_s + coff);
    const unsigned long long range = (unsigned long long)m.kmax - (unsigned long long)m.kmin;
    int nbits = 0;
    while (nbits < 64 && (range >> nbits) != 0) ++nbits;
    if (int rc = sort_pairs_device(keys_by_gid, perm, tk, tp, counts, ngroups, (unsigned long long)m.kmin, nbits, st))
      return rc;
  }
  EmitParams p;
  memset(&p, 0, sizeof(p));
  if (count_overflow_dev) {
    // the group count stays on the device: dense_scan_kernel left it in meta->ngroups; export {count, overflow}
    // for the caller (the table may be destroyed before anybody reads them) and bound the emit by it
    gb_export_meta_kernel<<<1, 1, 0, st>>>(t->meta, reinterpret_cast<long long*>(count_overflow_dev));
    MB_LAUNCH_CHECK("gb_export_meta_kernel");
    p.count_dev = &t->meta->ngroups;
  }
  p.keys_sorted = keys_by_gid;
  p.perm = perm;
  p.acc = t->acc;
  p.cnt = t->cnt;
  p.size = t->size;
  p.nvals = t->nvals;
  p.vstride = t->vstride;
  p.flags = t->flags;
  p.ngroups = ngroups;
  p.out_keys = reinterpret_cast<long long*>(out_keys);
  for (int v = 0; v < t->nvals; ++v) {
    p.out_sums[v] = out_sums ? out_sums[v] : nullptr;
    p.out_cnts[v] = out_cnts ? out_cnts[v] : nullptr;
  }
  p.out_sizes = reinterpret_cast<long long*>(out_sizes);
  gb_emit_kernel<<<(unsigned)((ngroups + 255) / 256), 256, 0, st>>>(p);
  MB_LAUNCH_CHECK("gb_emit_kernel");
  return 0;
}
