// join.cu — broadcast hash join: build once over the (broadcast) dim key column, probe with
// every fact row block, gather the dim payload.
//
// Reference path: MergeImpl.row_axis_merge (modin/core/storage_formats/pandas/merge.py:104-252)
// collapses the right frame into one partition (`right._modin_frame.combine()`, merge.py:178),
// broadcasts it to every left row partition (broadcast_apply_full_axis, df.py:3483-3676) and
// calls pandas.merge(left_block, right, how, on, sort=False) per block (merge.py:166-168);
// pandas factorizes both key columns, builds hash-join indexers and `take`s the payload.
//
// Here: slots[cap] {int64 key, int32 row} (cap = pow2 >= 2 * ndim).  For the many-to-one case
// (distinct dim keys; star-schema fact x dim) a fact row needs one probe and the output keeps
// the fact's row order, so `how="left"` only has to materialise the dim payload columns; the
// fact columns are shared by reference with the input frame (blocks are immutable values).
// Algorithmic traffic for the fused probe+gather: 8 B key read + 8 B per payload column written
// per fact row; the slot / payload reads hit the L2-resident dim table.
//
// Dim keys that span a narrow range (max - min + 1 <= 4 * ndim: surrogate keys, ids) get a DENSE table
// instead: rows[key - kmin] = dim row, built with one atomicCAS per dim row (which also detects
// duplicates); a probe is one bounds check + one 4-byte read, four fact rows in flight per thread, output
// written with streaming stores.
#include "common.cuh"

namespace mb200 {

struct __align__(16) JSlot {
  long long key;
  int row;  // -1 empty, -2 being inserted, >= 0 dim row index
  int pad;
};
struct JMeta {
  int duplicate;  // some dim key occurs twice
  int pad;
};

}  // namespace mb200

struct mb200_join_table {
  mb200::JSlot* slots;
  long long cap;
  long long ndim;
  mb200::JMeta* meta;
  // dense (direct-addressed) form, chosen at build time when the dim keys span a narrow range:
  // rows[key - kmin] = dim row (-1 = no such key); no hashing, one 4-byte read per probe
  int dense;
  long long kmin;
  unsigned long long range;
  int* rows;
  int persisted;  // holds a reference on the persisting L2 carve-out
  size_t carve_bytes, window_bytes;
  // key-ordered copies of float64 payload columns (dense tables; see join_order_payload_kernel), one per source
  // column and kept until the table is destroyed: a payload wider than one launch is probed in several launches,
  // each of which finds its own columns' copies (malloc'd arrays of ordered_cap entries).  Nothing is evicted: every
  // distinct source column costs range * 8 bytes of device memory until the table is destroyed.  A merge's table lives
  // with its dim frame and is probed with that frame's payload columns only, so this is one copy per dim column.
  int nordered, ordered_cap;
  const void** ordered_src;
  double** ordered;
};

namespace mb200 {

__device__ __forceinline__ void ld_jslot(const JSlot* s, long long& key, int& row) {
  unsigned long long a, b;
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(s) : "memory");
  key = (long long)a;
  row = (int)(unsigned int)(b & 0xffffffffULL);
}

__global__ void join_init_kernel(JSlot* slots, long long cap, JMeta* meta) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cap) {
    JSlot s;
    s.key = 0;
    s.row = -1;
    s.pad = 0;
    slots[i] = s;
  }
  if (i == 0) {
    meta->duplicate = 0;
    meta->pad = 0;
  }
}

__global__ void join_build_kernel(JSlot* slots, unsigned int mask, const long long* __restrict__ keys, long long n,
                                  JMeta* meta) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const long long k = keys[i];
    unsigned int slot = hash_key(k) & mask;
    for (;;) {
      long long sk;
      int r;
      ld_jslot(&slots[slot], sk, r);
      if (r >= 0) {
        if (sk == k) {  // duplicate dim key: keep the first row seen, flag it
          meta->duplicate = 1;
          break;
        }
        slot = (slot + 1) & mask;
        continue;
      }
      if (r == -1) {
        const int old = atomicCAS(&slots[slot].row, -1, -2);
        if (old == -1) {
          *reinterpret_cast<volatile long long*>(&slots[slot].key) = k;
          __threadfence();
          *reinterpret_cast<volatile int*>(&slots[slot].row) = (int)i;
          break;
        }
      }
      // slot is being published by another thread: look again
    }
  }
}

// Warp-wide lookup with a vote-controlled (warp-uniform) probe loop: every lane leaves together, so the
// stores that follow run converged (a per-lane `return` inside the loop lets nvcc run the rest of the
// iteration in diverged groups -- measured on the groupby kernel, see groupby.cu).  Must be called by
// all 32 lanes; lanes without a row pass valid = false.
__device__ __forceinline__ int join_lookup(const JSlot* slots, unsigned int mask, long long k, bool valid) {
  unsigned int slot = hash_key(k) & mask;
  int res = -1;
  bool active = valid;
  while (__any_sync(0xffffffffu, active)) {
    if (active) {
      long long sk;
      int r;
      ld_jslot(&slots[slot], sk, r);
      if (r < 0) {
        active = false;  // table is read-only during probing: an empty slot terminates the chain
      } else if (sk == k) {
        res = r;
        active = false;
      } else {
        slot = (slot + 1) & mask;
      }
    }
  }
  return res;
}

__global__ void __launch_bounds__(256) join_probe_kernel(const JSlot* __restrict__ slots, unsigned int mask,
                                                         const long long* __restrict__ fact_keys, long long n,
                                                         long long* __restrict__ out_idx,
                                                         unsigned long long* nmatch) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const uint64_t pol = l2_policy_evict_first();
  const int lane = threadIdx.x & 31;
  unsigned long long hits = 0;
  // warp-uniform outer loop: `base` is the row of lane 0
  for (long long base = (long long)blockIdx.x * blockDim.x + (threadIdx.x - lane); base < n; base += stride) {
    const long long i = base + lane;
    const bool valid = i < n;
    const long long k = valid ? ldg_stream_i64(fact_keys + i, pol) : 0;
    const int r = join_lookup(slots, mask, k, valid);
    if (valid) out_idx[i] = (long long)r;
    hits += (valid && r >= 0);
  }
  // one atomic per warp
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) hits += __shfl_xor_sync(0xffffffffu, hits, m);
  if (lane == 0 && hits && nmatch) atomicAdd(nmatch, hits);
}

struct GatherParams {
  const void* dim_cols[MB200_MAX_COLS];
  void* out_cols[MB200_MAX_COLS];
  int ncols;
};

template <typename T>
__global__ void __launch_bounds__(256) join_probe_gather_kernel(const JSlot* __restrict__ slots, unsigned int mask,
                                                                const long long* __restrict__ fact_keys, long long n,
                                                                const __grid_constant__ GatherParams g,
                                                                unsigned long long* nmatch, T null_value) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const uint64_t pol = l2_policy_evict_first();
  const int lane = threadIdx.x & 31;
  unsigned long long hits = 0;
  for (long long base = (long long)blockIdx.x * blockDim.x + (threadIdx.x - lane); base < n; base += stride) {
    const long long i = base + lane;
    const bool valid = i < n;
    const long long k = valid ? ldg_stream_i64(fact_keys + i, pol) : 0;
    const int r = join_lookup(slots, mask, k, valid);
    hits += (valid && r >= 0);
    if (valid) {
      for (int c = 0; c < g.ncols; ++c) {
        const T v = r >= 0 ? static_cast<const T*>(g.dim_cols[c])[r] : null_value;
        static_cast<T*>(g.out_cols[c])[i] = v;
      }
    }
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) hits += __shfl_xor_sync(0xffffffffu, hits, m);
  if (lane == 0 && hits && nmatch) atomicAdd(nmatch, hits);
}

template <typename T>
__global__ void __launch_bounds__(256) take_kernel(const __grid_constant__ GatherParams g,
                                                   const long long* __restrict__ idx, long long n, T null_value) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const long long r = idx[i];
    for (int c = 0; c < g.ncols; ++c)
      static_cast<T*>(g.out_cols[c])[i] = r >= 0 ? static_cast<const T*>(g.dim_cols[c])[r] : null_value;
  }
}

// ---------------------------------------------------------------- dense (direct-addressed) dim table
__global__ void join_dense_build_kernel(int* rows, long long kmin, const long long* __restrict__ keys, long long n,
                                        JMeta* meta) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const long long d = keys[i] - kmin;
    if (atomicCAS(&rows[d], -1, (int)i) != -1) meta->duplicate = 1;  // duplicate dim key
  }
}

// Four fact rows per thread and iteration: the dependent chain of a row is key -> rows[] -> payload, so the
// loads of four independent rows are issued together (the probe is latency-, not bandwidth-bound per row).
template <typename T, bool GATHER>
__global__ void __launch_bounds__(256) join_dense_probe_kernel(const int* __restrict__ rows, long long kmin,
                                                               unsigned long long range,
                                                               const long long* __restrict__ fact_keys, long long n,
                                                               const __grid_constant__ GatherParams g,
                                                               long long* __restrict__ out_idx,
                                                               unsigned long long* nmatch, T null_value) {
  constexpr int U = 4;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  const uint64_t pol = l2_policy_evict_first();
  const int lane = threadIdx.x & 31;
  unsigned long long hits = 0;
  for (long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; i0 < n; i0 += nthreads * U) {
    long long k[U];
    int r[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + u * nthreads;
      k[u] = i < n ? ldg_stream_i64(fact_keys + i, pol) : kmin - 1;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned long long d = (unsigned long long)k[u] - (unsigned long long)kmin;
      const bool in = (i0 + u * nthreads < n) && d < range;
      r[u] = in ? __ldg(rows + d) : -1;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + u * nthreads;
      if (i >= n) continue;
      hits += r[u] >= 0;
      if (GATHER) {
        for (int c = 0; c < g.ncols; ++c)  // streaming store: the output must not push the dim table out of L2
          __stcs(static_cast<T*>(g.out_cols[c]) + i,
                 r[u] >= 0 ? __ldg(static_cast<const T*>(g.dim_cols[c]) + r[u]) : null_value);
      } else {
        __stcs(out_idx + i, (long long)r[u]);
      }
    }
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) hits += __shfl_xor_sync(0xffffffffu, hits, m);
  if (lane == 0 && hits && nmatch) atomicAdd(nmatch, hits);
}

// Key-ordered payload of a dense table: ord[g] = rows[g] >= 0 ? col[rows[g]] : NaN.  Built once per (table, payload
// column) on the first left-join probe that does not need the match count; the probe then makes ONE random
// read per fact row and payload column (ord[key - kmin]) instead of two (rows[], then col[row]).
__global__ void join_order_payload_kernel(const int* __restrict__ rows, unsigned long long range,
                                          const double* __restrict__ col, double* __restrict__ ord) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < (long long)range; g += stride) {
    const int r = rows[g];
    ord[g] = r >= 0 ? col[r] : __longlong_as_double(0x7ff8000000000000LL);
  }
}

struct OrderedParams {
  const double* ord[MB200_MAX_COLS];
  double* out[MB200_MAX_COLS];
  int ncols;
};

__global__ void __launch_bounds__(256) join_dense_ordered_probe_kernel(long long kmin, unsigned long long range,
                                                                       const long long* __restrict__ fact_keys,
                                                                       long long n,
                                                                       const __grid_constant__ OrderedParams g) {
  constexpr int U = 4;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  const uint64_t pol = l2_policy_evict_first();
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  for (long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; i0 < n; i0 += nthreads * U) {
    unsigned long long d[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + u * nthreads;
      const long long k = i < n ? ldg_stream_i64(fact_keys + i, pol) : kmin - 1;
      d[u] = (unsigned long long)k - (unsigned long long)kmin;
    }
    for (int c = 0; c < g.ncols; ++c) {
      double v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = (i0 + u * nthreads < n && d[u] < range) ? __ldg(g.ord[c] + d[u]) : nan;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long i = i0 + u * nthreads;
        if (i < n) __stcs(g.out[c] + i, v[u]);
      }
    }
  }
}

// ---- compaction of hit positions: block counts -> scan -> ranked scatter
constexpr int kCompBlock = 256;
constexpr int kCompItems = 2048;  // per block

__global__ void __launch_bounds__(kCompBlock) compact_count_kernel(const long long* __restrict__ idx, long long n,
                                                                   unsigned int* __restrict__ counts) {
  __shared__ unsigned int s;
  if (threadIdx.x == 0) s = 0;
  __syncthreads();
  const long long base = (long long)blockIdx.x * kCompItems;
  unsigned int c = 0;
  for (int j = threadIdx.x; j < kCompItems; j += kCompBlock) {
    const long long i = base + j;
    c += (i < n && idx[i] >= 0);
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) c += __shfl_xor_sync(0xffffffffu, c, m);
  if ((threadIdx.x & 31) == 0) atomicAdd(&s, c);
  __syncthreads();
  if (threadIdx.x == 0) counts[blockIdx.x] = s;
}

// exclusive scan of counts[nblocks] into 64-bit offsets; single block; also writes the total.
__global__ void __launch_bounds__(1024) compact_scan_kernel(const unsigned int* __restrict__ counts, long long nblocks,
                                                            long long* __restrict__ offsets, long long* total) {
  __shared__ long long part[1024];
  const int t = threadIdx.x;
  const long long per = (nblocks + 1023) / 1024;
  const long long lo = (long long)t * per;
  long long hi = lo + per;
  if (hi > nblocks) hi = nblocks;
  long long s = 0;
  for (long long i = lo; i < hi; ++i) s += counts[i];
  part[t] = s;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    long long v = t >= off ? part[t - off] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  long long run = t ? part[t - 1] : 0;
  for (long long i = lo; i < hi; ++i) {
    offsets[i] = run;
    run += counts[i];
  }
  if (t == 1023 && total) *total = part[1023];
}

__global__ void __launch_bounds__(kCompBlock) compact_scatter_kernel(const long long* __restrict__ idx, long long n,
                                                                     const long long* __restrict__ offsets,
                                                                     long long* __restrict__ out_pos) {
  __shared__ unsigned int warp_base[kCompBlock / 32];
  __shared__ unsigned int running;
  if (threadIdx.x == 0) running = 0;
  __syncthreads();
  const long long base = (long long)blockIdx.x * kCompItems;
  const long long off = offsets[blockIdx.x];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int j0 = 0; j0 < kCompItems; j0 += kCompBlock) {
    const long long i = base + j0 + threadIdx.x;
    const bool hit = (i < n) && idx[i] >= 0;
    const unsigned int bal = __ballot_sync(0xffffffffu, hit);
    const unsigned int rank = __popc(bal & ((1u << lane) - 1u));
    if (lane == 0) warp_base[warp] = __popc(bal);
    __syncthreads();
    if (threadIdx.x == 0) {  // serial prefix over 8 warps keeps row order
      unsigned int run = running;
      for (int w = 0; w < kCompBlock / 32; ++w) {
        const unsigned int c = warp_base[w];
        warp_base[w] = run;
        run += c;
      }
      running = run;
    }
    __syncthreads();
    if (hit) out_pos[off + warp_base[warp] + rank] = i;
    __syncthreads();
  }
}

static long long jnext_pow2(long long v) {
  long long p = 1;
  while (p < v) p <<= 1;
  return p;
}

static int launch_grid(long long n, int threads, int per_sm, int* grid) {
  DevProps dp;
  if (int rc = dev_props(&dp)) return rc;
  long long g = (n + threads - 1) / threads;
  const long long cap = (long long)dp.sm_count * per_sm;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  *grid = (int)g;
  return 0;
}

}  // namespace mb200

using namespace mb200;

extern "C" int mb200_join_build(mb200_join_table** table, const int64_t* dim_keys, int64_t ndim,
                                mb200_stream_t stream) {
  if (!table) return fail("mb200_join_build", "null out pointer");
  l2_carveout_drop_idle();  // a carve-out left behind by group tables: the dim table wants the whole L2
  if (ndim < 0 || ndim > 0x7fffffffLL) return fail("mb200_join_build", "dim rows must be in [0, 2^31)");
  if (ndim > 0 && !dim_keys) return fail("mb200_join_build", "null keys");
  DevProps dp;
  if (int rc = dev_props(&dp)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  mb200_join_table* t = new mb200_join_table();
  memset(t, 0, sizeof(*t));
  t->ndim = ndim;
  cudaError_t e = cudaMallocAsync((void**)&t->meta, sizeof(JMeta), st);
  if (e != cudaSuccess) {
    delete t;
    return cuda_fail("mb200_join_build", e);
  }
  // dense form when the dim keys span a narrow range (one min/max pass over the dim keys + a 16-byte D2H;
  // MB200_JOIN_DENSE=0 forces the hash table)
  {
    const char* env = getenv("MB200_JOIN_DENSE");
    if (ndim > 0 && !(env && env[0] == '0')) {
      long long* mmbuf = nullptr;
      e = cudaMallocAsync((void**)&mmbuf, 32, st);  // {min, max, sampled, duplicates}
      if (e != cudaSuccess) {
        mb200_join_destroy(t, stream);
        return cuda_fail("mb200_join_build", e);
      }
      long long host_mm[2];
      int rc = mb200_key_range(dim_keys, ndim, reinterpret_cast<int64_t*>(mmbuf), 1, stream);
      if (!rc) {
        e = cudaMemcpyAsync(host_mm, mmbuf, 16, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
      }
      cudaFreeAsync(mmbuf, st);
      if (rc || e != cudaSuccess) {
        mb200_join_destroy(t, stream);
        return rc ? rc : cuda_fail("mb200_join_build", e);
      }
      const unsigned long long range = (unsigned long long)host_mm[1] - (unsigned long long)host_mm[0] + 1ULL;
      const unsigned long long limit = (unsigned long long)(4 * ndim > 65536 ? 4 * ndim : 65536);
      if (range != 0 && range <= limit && range <= 0x7fffffffULL) {
        t->dense = 1;
        t->kmin = host_mm[0];
        t->range = range;
      }
    }
  }
  if (t->dense) {
    e = cudaMallocAsync((void**)&t->rows, (size_t)t->range * sizeof(int), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(t->rows, 0xff, (size_t)t->range * sizeof(int), st);  // -1
    if (e == cudaSuccess) e = cudaMemsetAsync(t->meta, 0, sizeof(JMeta), st);
    if (e != cudaSuccess) {
      mb200_join_destroy(t, stream);
      return cuda_fail("mb200_join_build", e);
    }
    int grid;
    if (int rc = launch_grid(ndim, 256, 8, &grid)) return rc;
    join_dense_build_kernel<<<grid, 256, 0, st>>>(t->rows, t->kmin, reinterpret_cast<const long long*>(dim_keys), ndim,
                                                 t->meta);
    MB_LAUNCH_CHECK("join_dense_build_kernel");
    *table = t;
    return 0;
  }
  t->cap = jnext_pow2(2 * ndim < 1024 ? 1024 : 2 * ndim);
  e = cudaMallocAsync((void**)&t->slots, (size_t)t->cap * sizeof(JSlot), st);
  if (e != cudaSuccess) {
    mb200_join_destroy(t, stream);
    return cuda_fail("mb200_join_build", e);
  }
  join_init_kernel<<<(unsigned)((t->cap + 255) / 256), 256, 0, st>>>(t->slots, t->cap, t->meta);
  MB_LAUNCH_CHECK("join_init_kernel");
  if (ndim > 0) {
    int grid;
    if (int rc = launch_grid(ndim, 256, 8, &grid)) return rc;
    join_build_kernel<<<grid, 256, 0, st>>>(t->slots, (unsigned int)(t->cap - 1),
                                            reinterpret_cast<const long long*>(dim_keys), ndim, t->meta);
    MB_LAUNCH_CHECK("join_build_kernel");
  }
  *table = t;
  return 0;
}

extern "C" int mb200_join_destroy(mb200_join_table* t, mb200_stream_t stream) {
  if (!t) return 0;
  if (t->slots) cudaFreeAsync(t->slots, (cudaStream_t)stream);
  if (t->rows) cudaFreeAsync(t->rows, (cudaStream_t)stream);
  for (int c = 0; c < t->nordered; ++c)
    if (t->ordered[c]) cudaFreeAsync(t->ordered[c], (cudaStream_t)stream);
  free(t->ordered_src);
  free(t->ordered);
  if (t->meta) cudaFreeAsync(t->meta, (cudaStream_t)stream);
  if (t->persisted) l2_carveout_release();
  delete t;
  return 0;
}

extern "C" int mb200_join_is_unique(mb200_join_table* t, int* unique, mb200_stream_t stream) {
  if (!t || !unique) return fail("mb200_join_is_unique", "null argument");
  JMeta m;
  MB_CUDA(cudaMemcpyAsync(&m, t->meta, sizeof(m), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  MB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  *unique = m.duplicate ? 0 : 1;
  return 0;
}

// EXPERIMENT, off by default (MB200_JOIN_PERSIST=rows | payload): pin one array of the dense dim table in the
// persisting L2 carve-out while a probe kernel runs.  The probe makes one random 4-byte read of rows[] and
// one random read per payload column for every fact row (1e7 dim rows = 40 MB of rows[] + 80 MB per float64
// payload column).  Whichever array is pinned, the other one works with a shrunken normal L2.
struct JoinWindow {
  cudaStream_t st;
  bool on = false;
  JoinWindow(cudaStream_t s, mb200_join_table* t, const void* base, size_t bytes) : st(s) {
    const char* e = getenv("MB200_JOIN_PERSIST");
    if (!(e && (e[0] == 'r' || e[0] == 'p')) || !base || bytes < ((size_t)8 << 20)) return;
    if (!t->persisted) {  // one carve-out reference per table, dropped in mb200_join_destroy
      size_t mw = 0;
      const size_t mp = l2_carveout_acquire(&mw);
      if (!mp) return;
      t->persisted = 1;
      t->carve_bytes = mp;
      t->window_bytes = mw;
    }
    cudaStreamAttrValue v;
    memset(&v, 0, sizeof(v));
    v.accessPolicyWindow.base_ptr = const_cast<void*>(base);
    v.accessPolicyWindow.num_bytes = bytes < t->window_bytes ? bytes : t->window_bytes;
    const double fit = (double)t->carve_bytes / (double)v.accessPolicyWindow.num_bytes;
    v.accessPolicyWindow.hitRatio = fit >= 1.0 ? 1.0f : (float)fit;
    v.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    v.accessPolicyWindow.missProp = cudaAccessPropertyNormal;
    if (cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &v) == cudaSuccess) on = true;
    else cudaGetLastError();
  }
  ~JoinWindow() {
    if (on) {
      cudaStreamAttrValue v;
      memset(&v, 0, sizeof(v));
      cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &v);
    }
  }
};

extern "C" int mb200_join_probe(mb200_join_table* t, const int64_t* fact_keys, int64_t nfact, int64_t* out_idx,
                                int64_t* out_nmatch_dev, mb200_stream_t stream) {
  l2_carveout_drop_idle();
  if (!t) return fail("mb200_join_probe", "null table");
  if (nfact < 0) return fail("mb200_join_probe", "negative nfact");
  if (nfact == 0) return 0;
  if (!fact_keys || !out_idx) return fail("mb200_join_probe", "null argument");
  int grid;
  if (int rc = launch_grid(nfact, 256, 8, &grid)) return rc;
  if (t->dense) {
    GatherParams g0;
    memset(&g0, 0, sizeof(g0));
    join_dense_probe_kernel<long long, false><<<grid, 256, 0, (cudaStream_t)stream>>>(
        t->rows, t->kmin, t->range, reinterpret_cast<const long long*>(fact_keys), nfact, g0,
        reinterpret_cast<long long*>(out_idx), reinterpret_cast<unsigned long long*>(out_nmatch_dev), 0LL);
    MB_LAUNCH_CHECK("join_dense_probe_kernel");
    return 0;
  }
  join_probe_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      t->slots, (unsigned int)(t->cap - 1), reinterpret_cast<const long long*>(fact_keys), nfact,
      reinterpret_cast<long long*>(out_idx), reinterpret_cast<unsigned long long*>(out_nmatch_dev));
  MB_LAUNCH_CHECK("join_probe_kernel");
  return 0;
}

// The key-ordered copy of one float64 payload column of a dense table: found by source pointer, or built and kept.
static int ordered_payload(mb200_join_table* t, const void* src, cudaStream_t st, const double** out) {
  for (int i = 0; i < t->nordered; ++i)
    if (t->ordered_src[i] == src) {
      *out = t->ordered[i];
      return 0;
    }
  if (t->nordered == t->ordered_cap) {
    const int cap = t->ordered_cap ? 2 * t->ordered_cap : MB200_MAX_COLS;
    const void** s = static_cast<const void**>(realloc(t->ordered_src, cap * sizeof(*s)));
    if (!s) return fail("mb200_join_probe_gather", "out of host memory");
    t->ordered_src = s;
    double** o = static_cast<double**>(realloc(t->ordered, cap * sizeof(*o)));
    if (!o) return fail("mb200_join_probe_gather", "out of host memory");
    t->ordered = o;
    t->ordered_cap = cap;
  }
  int grid;
  if (int rc = launch_grid((long long)t->range, 256, 8, &grid)) return rc;
  double* ord = nullptr;
  MB_CUDA(cudaMallocAsync((void**)&ord, (size_t)t->range * 8, st));
  t->ordered_src[t->nordered] = src;
  t->ordered[t->nordered++] = ord;
  join_order_payload_kernel<<<grid, 256, 0, st>>>(t->rows, t->range, static_cast<const double*>(src), ord);
  MB_LAUNCH_CHECK("join_order_payload_kernel");
  *out = ord;
  return 0;
}

extern "C" int mb200_join_probe_gather(mb200_join_table* t, const int64_t* fact_keys, int64_t nfact, int ncols,
                                       const void* const* dim_cols, int dim_dtype, void* const* out_cols,
                                       int64_t* out_nmatch_dev, mb200_stream_t stream) {
  l2_carveout_drop_idle();
  if (!t) return fail("mb200_join_probe_gather", "null table");
  if (ncols < 0 || ncols > MB200_MAX_COLS) return fail("mb200_join_probe_gather", "ncols out of range (0..32)");
  if (nfact < 0) return fail("mb200_join_probe_gather", "negative nfact");
  if (nfact == 0) return 0;
  if (!fact_keys || (ncols > 0 && (!dim_cols || !out_cols))) return fail("mb200_join_probe_gather", "null argument");
  GatherParams g;
  memset(&g, 0, sizeof(g));
  g.ncols = ncols;
  for (int c = 0; c < ncols; ++c) {
    g.dim_cols[c] = dim_cols[c];
    g.out_cols[c] = out_cols[c];
    if (!out_cols[c] || (!dim_cols[c] && t->ndim > 0)) return fail("mb200_join_probe_gather", "null column pointer");
  }
  int grid;
  if (int rc = launch_grid(nfact, 256, 8, &grid)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned int mask = (unsigned int)(t->cap - 1);
  unsigned long long* nm = reinterpret_cast<unsigned long long*>(out_nmatch_dev);
  const long long* fk = reinterpret_cast<const long long*>(fact_keys);
  if (t->dense && dim_dtype == MB200_F64 && !out_nmatch_dev && ncols > 0) {
    // left join, float64 payload, nobody asks for the match count: probe the key-ordered payload copies
    // (MB200_JOIN_ORDERED=0 keeps the two-read probe)
    const char* oe = getenv("MB200_JOIN_ORDERED");
    if (!(oe && oe[0] == '0')) {
      OrderedParams op;
      memset(&op, 0, sizeof(op));
      op.ncols = ncols;
      for (int c = 0; c < ncols; ++c) {
        if (int rc = ordered_payload(t, dim_cols[c], st, &op.ord[c])) return rc;
        op.out[c] = static_cast<double*>(out_cols[c]);
      }
      join_dense_ordered_probe_kernel<<<grid, 256, 0, st>>>(t->kmin, t->range, fk, nfact, op);
      MB_LAUNCH_CHECK("join_dense_ordered_probe_kernel");
      return 0;
    }
  }
  if (t->dense) {
    const char* pe = getenv("MB200_JOIN_PERSIST");
    const bool pin_payload = pe && pe[0] == 'p' && ncols > 0;
    JoinWindow window(st, t, pin_payload ? dim_cols[0] : (const void*)t->rows,
                      pin_payload ? (size_t)t->ndim * 8 : (size_t)t->range * sizeof(int));
    if (dim_dtype == MB200_F64)
      join_dense_probe_kernel<double, true><<<grid, 256, 0, st>>>(t->rows, t->kmin, t->range, fk, nfact, g, nullptr, nm,
                                                                  (double)__builtin_nan(""));
    else if (dim_dtype == MB200_I64)
      join_dense_probe_kernel<long long, true><<<grid, 256, 0, st>>>(t->rows, t->kmin, t->range, fk, nfact, g, nullptr,
                                                                     nm, 0LL);
    else
      return fail("mb200_join_probe_gather", "unsupported payload dtype");
    MB_LAUNCH_CHECK("join_dense_probe_kernel");
    return 0;
  }
  if (dim_dtype == MB200_F64) {
    join_probe_gather_kernel<double><<<grid, 256, 0, st>>>(t->slots, mask, fk, nfact, g, nm,
                                                           (double)__builtin_nan(""));
  } else if (dim_dtype == MB200_I64) {
    join_probe_gather_kernel<long long><<<grid, 256, 0, st>>>(t->slots, mask, fk, nfact, g, nm, 0LL);
  } else {
    return fail("mb200_join_probe_gather", "unsupported payload dtype");
  }
  MB_LAUNCH_CHECK("join_probe_gather_kernel");
  return 0;
}

extern "C" int mb200_take(int dtype, int ncols, const void* const* src, const int64_t* idx, int64_t nidx,
                          void* const* out, mb200_stream_t stream) {
  if (ncols < 0 || ncols > MB200_MAX_COLS) return fail("mb200_take", "ncols out of range (0..32)");
  if (nidx < 0) return fail("mb200_take", "negative nidx");
  if (nidx == 0 || ncols == 0) return 0;
  if (!src || !idx || !out) return fail("mb200_take", "null argument");
  GatherParams g;
  memset(&g, 0, sizeof(g));
  g.ncols = ncols;
  for (int c = 0; c < ncols; ++c) {
    g.dim_cols[c] = src[c];
    g.out_cols[c] = out[c];
    if (!out[c]) return fail("mb200_take", "null column pointer");
  }
  int grid;
  if (int rc = launch_grid(nidx, 256, 8, &grid)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const long long* ix = reinterpret_cast<const long long*>(idx);
  if (dtype == MB200_F64)
    take_kernel<double><<<grid, 256, 0, st>>>(g, ix, nidx, (double)__builtin_nan(""));
  else if (dtype == MB200_I64)
    take_kernel<long long><<<grid, 256, 0, st>>>(g, ix, nidx, 0LL);
  else if (dtype == MB200_U8)
    take_kernel<unsigned char><<<grid, 256, 0, st>>>(g, ix, nidx, (unsigned char)0);
  else
    return fail("mb200_take", "unsupported dtype");
  MB_LAUNCH_CHECK("take_kernel");
  return 0;
}

extern "C" int mb200_compact_hits(const int64_t* idx, int64_t n, int64_t* out_pos, int64_t* out_count_dev,
                                  void* scratch, size_t scratch_bytes, mb200_stream_t stream) {
  if (n < 0) return fail("mb200_compact_hits", "negative n");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) {
    if (out_count_dev) MB_CUDA(cudaMemsetAsync(out_count_dev, 0, 8, st));
    return 0;
  }
  if (!idx || !out_pos || !scratch) return fail("mb200_compact_hits", "null argument");
  const long long nblocks = (n + kCompItems - 1) / kCompItems;
  const size_t need = (size_t)nblocks * 12 + 256;
  if (scratch_bytes < need) return fail("mb200_compact_hits", "scratch too small (need 12 B per 2048 rows + 256)");
  long long* offsets = static_cast<long long*>(scratch);
  unsigned int* counts = reinterpret_cast<unsigned int*>(static_cast<char*>(scratch) + (size_t)nblocks * 8);
  const long long* ix = reinterpret_cast<const long long*>(idx);
  compact_count_kernel<<<(unsigned)nblocks, kCompBlock, 0, st>>>(ix, n, counts);
  MB_LAUNCH_CHECK("compact_count_kernel");
  compact_scan_kernel<<<1, 1024, 0, st>>>(counts, nblocks, offsets, reinterpret_cast<long long*>(out_count_dev));
  MB_LAUNCH_CHECK("compact_scan_kernel");
  compact_scatter_kernel<<<(unsigned)nblocks, kCompBlock, 0, st>>>(ix, n, offsets, reinterpret_cast<long long*>(out_pos));
  MB_LAUNCH_CHECK("compact_scatter_kernel");
  return 0;
}
