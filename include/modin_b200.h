/*
 * modin_b200.h — C ABI of libmodin_b200.so: the sm_90a kernels behind Modin's
 * partition-execution hot path (Map / Binary / TreeReduce / GroupByReduce /
 * broadcast-merge operator templates).
 *
 * The reference (modin-project/modin) is pure Python and has NO native/FFI
 * boundary on this path: the per-partition arithmetic is a Python closure
 * around a pandas method, invoked by
 *   PandasDataframePartition.apply(func)            modin/core/dataframe/pandas/partitioning/partition.py:77-140
 *   PandasOnPythonDataframePartition.apply          modin/core/execution/python/implementations/pandas_on_python/partitioning/partition.py:76-123
 *   PandasDataframeAxisPartition.deploy_axis_func   modin/core/dataframe/pandas/partitioning/axis_partition.py:396-499
 * Each entry point below therefore names the *pandas call site in the
 * reference* whose per-block work it replaces.  INTEGRATION.md shows the
 * ctypes binding (modin_b200/_lib.py) a Modin maintainer would add.
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on failure; the message is
 *     available from mb200_last_error() (thread-local, valid until the next
 *     failing call on the same thread);
 *   - all column pointers are DEVICE pointers (one contiguous buffer per column,
 *     Arrow fixed-width layout: float64 / int64 / uint8-bool; float64 nulls are
 *     NaN as in pandas, so no validity bitmap is carried on this path);
 *   - pointer *arrays* (`const void* const* cols`) and scalar arrays are HOST
 *     arrays of length ncols; they are copied into kernel parameters;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *     calls are asynchronous with respect to the host unless stated;
 *   - no global state besides the CUDA context; no CPU fallback: on a machine
 *     without a usable sm_90 device every compute call fails with an error.
 */
#ifndef MODIN_B200_H
#define MODIN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 2: round 2 (key statistics, async dense emit, expand / concat / comm entry points); 3: + the Fold template's
 * cumulative scans (mb200_cum_*); 4: + MB200_GB_FIRST / MB200_GB_LAST group tables (row positions, NULL value
 * columns); 5: + MB200_GB_ARGMIN / MB200_GB_ARGMAX group tables and mb200_gb_accumulate_arg; 6: + MB200_GB_VAR group
 * tables and mb200_gb_accumulate_m2; 7: + MB200_GB_NUNIQUE group tables, their distinct set and
 * mb200_gb_reserve_distinct / mb200_gb_accumulate_distinct / mb200_gb_emit_distinct.  Checked by the binding at load
 * time (modin_b200/_lib.py). */
#define MB200_ABI_VERSION 7
#define MB200_MAX_COLS 32 /* max columns per launch == Modin's MinColumnPartitionSize (envvars.py:1149-1190) */

typedef void* mb200_stream_t;

/* ---- column element types ------------------------------------------------ */
enum mb200_dtype {
  MB200_F64 = 0, /* pandas float64 (NaN == null) */
  MB200_I64 = 1, /* pandas int64 */
  MB200_U8 = 2   /* pandas bool (0/1 bytes) */
};

/* ---- Map / Binary elementwise opcodes ------------------------------------
 * Replaces the per-block pandas call of
 *   Map.register(pandas.DataFrame.abs)          qc.py:2036      (MB200_OP_ABS)
 *   Map.register(pandas.DataFrame.isna/notna)   qc.py:2063-2106 (ISNA/NOTNA)
 *   qc.fillna scalar branch                      qc.py:2710-2813 (FILLNA)
 *   Binary.register(pandas.DataFrame.<op>)       qc.py:535-624   (ADD..GE, scalar and frame forms)
 * `*_S` forms take the right operand from the per-column scalar s0[col];
 * R* forms are the reflected versions (scalar OP x).
 * AFFINE  : out = (x * s0[col]) + s1[col]   -- two IEEE roundings, like pandas `df * b + c`
 * FMA3    : out = (a * b) + c  on three frames -- two roundings, NOT a fused multiply-add
 * Comparison ops write uint8 0/1.
 */
enum mb200_map_op {
  MB200_OP_ABS = 0,
  MB200_OP_NEG = 1,
  MB200_OP_ISNA = 2,
  MB200_OP_NOTNA = 3,
  MB200_OP_FILLNA_S = 4,
  MB200_OP_AFFINE = 5,
  MB200_OP_ADD_S = 6,
  MB200_OP_SUB_S = 7,
  MB200_OP_RSUB_S = 8,
  MB200_OP_MUL_S = 9,
  MB200_OP_DIV_S = 10,
  MB200_OP_RDIV_S = 11,
  MB200_OP_EQ_S = 12,
  MB200_OP_NE_S = 13,
  MB200_OP_LT_S = 14,
  MB200_OP_LE_S = 15,
  MB200_OP_GT_S = 16,
  MB200_OP_GE_S = 17,
  MB200_OP_CLIP_S = 18, /* x < s0 ? s0 : (x > s1 ? s1 : x); NaN preserved; absent bounds = -inf / +inf (pandas clip) */
  MB200_OP_COPY = 19,
  MB200_OP_ROUND_S = 20, /* numpy.round(x, d): s0 = 10^|d|, s1 = sign of d; rint(x * s0) / s0 (DataFrame.round) */
  MB200_OP_ORDERED_S = 21, /* sort key: int64 image whose signed order = sort_values order (float64 or int64 in,
                              int64 out; NaN last; s0 != 0 = descending).  Feeds mb200_sort_pairs_i64. */
  MB200_OP_NOT = 22, /* bool (uint8) in, bool out: ~x (qc.py:541-571 logical ops; DataFrame.__invert__) */
  /* two-frame ops (in0 OP in1) */
  MB200_OP_ADD = 32,
  MB200_OP_SUB = 33,
  MB200_OP_MUL = 34,
  MB200_OP_DIV = 35,
  MB200_OP_EQ = 36,
  MB200_OP_NE = 37,
  MB200_OP_LT = 38,
  MB200_OP_LE = 39,
  MB200_OP_GT = 40,
  MB200_OP_GE = 41,
  MB200_OP_FILLNA = 42, /* isnan(in0) ? in1 : in0 */
  MB200_OP_AND = 43, /* bool columns: in0 & in1, | and ^ (Binary.register(pandas.DataFrame.__and__ ...) qc.py:541-571) */
  MB200_OP_OR = 44,
  MB200_OP_XOR = 45,
  /* three-frame op */
  MB200_OP_FMA3 = 64
};

/* ---- TreeReduce opcodes ---------------------------------------------------
 * Replaces the map-phase pandas call of TreeReduce.register(pandas.DataFrame.sum / count /
 * max / min / mean) qc.py:976-1096 (per block: nanops.nansum etc.).
 */
enum mb200_reduce_op {
  MB200_RED_SUM = 0,  /* out_val = sum (NaN skipped iff skipna), out_cnt = #non-NaN */
  MB200_RED_MIN = 1,  /* out_val = min over non-NaN, out_cnt = #non-NaN             */
  MB200_RED_MAX = 2,
  MB200_RED_COUNT = 3, /* out_cnt only */
  MB200_RED_PROD = 4,  /* out_val = product (NaN skipped iff skipna), out_cnt = #non-NaN */
  MB200_RED_SSD = 5,   /* out_val = sum of (centre - x)^2 (NaN skipped iff skipna), out_cnt = #non-NaN:
                          the second pass of pandas' two-pass var / std (nanops.nanvar), float64 only,
                          through mb200_reduce_columns_centered */
  MB200_RED_ARGMIN = 6, /* out_val = min over non-NaN, out_pos = first row holding it, out_cnt = #non-NaN:  */
  MB200_RED_ARGMAX = 7  /* through mb200_reduce_arg_columns only                                           */
};

/* ---- groupby aggregate selection (bit flags) ------------------------------ */
enum mb200_gb_flags {
  MB200_GB_SUM = 1,   /* acc[g][v]  += x   (NaN skipped, pandas min_count=0)       */
  MB200_GB_COUNT = 2, /* cnt[g][v]  += !isnan(x)                                     */
  MB200_GB_SIZE = 4,  /* size[g]    += 1                                             */
  MB200_GB_MIN = 8,   /* acc[g][v]   = min(acc, x)  (NaN skipped; exclusive with SUM / MAX) */
  MB200_GB_MAX = 16,  /* acc[g][v]   = max(acc, x)                                          */
  /* row positions (int64) instead of values; each excludes SUM / COUNT / MIN / MAX and the other (SIZE may be set):
   * see mb200_gb_accumulate and mb200_gb_emit */
  MB200_GB_FIRST = 32, /* acc[g][v]   = min(position) over the rows whose value in column v is not NaN */
  MB200_GB_LAST = 64,  /* acc[g][v]   = max(position) over the same rows                               */
  /* the first row holding the group's extreme value; each excludes every other flag (see mb200_gb_accumulate_arg):
   * cnt[g][v] = min / max of the value's order-preserving int64 image, acc[g][v] = min(position) of the rows holding it */
  MB200_GB_ARGMIN = 128,
  MB200_GB_ARGMAX = 256,
  /* groupby.var / std: a VAR table is exactly SUM | COUNT | VAR.  It has one more float64 array, m2[g][v], which the
   * library allocates for dense tables too (it is not among the caller-owned arrays of mb200_gb_create_dense) and
   * which starts at 0.  Pass 1 fills acc / cnt (mb200_gb_accumulate, mb200_gb_merge_partial); pass 2 fills m2
   * (mb200_gb_accumulate_m2) */
  MB200_GB_VAR = 512,
  /* groupby.nunique: a NUNIQUE table is exactly SIZE | NUNIQUE.  cnt[g][v] holds the number of distinct values of
   * column v in group g, from 0.  Pass 1 (mb200_gb_accumulate / mb200_gb_merge_partial) is the SIZE launch: it inserts
   * the groups and reads no value column.  Pass 2 (mb200_gb_accumulate_distinct) inserts (group, column, value image)
   * entries into the table's distinct set (mb200_gb_reserve_distinct) and counts the new ones into cnt */
  MB200_GB_NUNIQUE = 1024
};

/* ======================= runtime / memory ================================== */
int mb200_abi_version(void);
const char* mb200_last_error(void);
/* Fails unless a CUDA device of compute capability 10.x is present. */
int mb200_device_check(int device);
int mb200_device_info(int device, int* sm_count, size_t* l2_bytes, size_t* total_mem,
                      int* cc_major, int* cc_minor);
int mb200_set_device(int device);
int mb200_alloc(void** ptr, size_t bytes, mb200_stream_t stream);
int mb200_free(void* ptr, mb200_stream_t stream);
int mb200_alloc_host(void** ptr, size_t bytes); /* pinned */
int mb200_free_host(void* ptr);
int mb200_h2d(void* dst, const void* src, size_t bytes, mb200_stream_t stream);
int mb200_d2h(void* dst, const void* src, size_t bytes, mb200_stream_t stream);
int mb200_d2d(void* dst, const void* src, size_t bytes, mb200_stream_t stream);
int mb200_memset(void* dst, int byte, size_t bytes, mb200_stream_t stream);
int mb200_stream_sync(mb200_stream_t stream);
/* number of kernels launched by this library in this process (bench `gpu_launches`) */
int64_t mb200_launch_count(void);

/* ======================= Map / Binary ====================================== */
/* One launch sweeps all `ncols` columns of a block (partition).
 * in1/in2 may be NULL for unary ops; s0/s1 are per-column scalar bit patterns
 * (double or int64 according to `dtype`), may be NULL when the op takes none.
 * `out_dtype` must be MB200_U8 for predicates, else equal `dtype`
 * (MB200_OP_DIV on int64 inputs writes float64).
 * Reference: pm.map_partitions pm.py:708-769, pm.n_ary_operation pm.py:1725-1788.
 */
int mb200_map(int op, int dtype, int ncols, const void* const* in0, const void* const* in1,
              const void* const* in2, void* const* out, int64_t nrows, const uint64_t* s0,
              const uint64_t* s1, mb200_stream_t stream);

/* Streaming form of mb200_map for HOST-resident blocks: chunks of rows are staged through
 * pinned buffers, H2D / kernel / D2H overlapped on three streams.  Host pointers in, host
 * pointers out.  Synchronous.  Used by the e2e measurement and by from_pandas->op->to_pandas. */
int mb200_map_host(int op, int dtype, int ncols, const void* const* in0_host,
                   const void* const* in1_host, const void* const* in2_host, void* const* out_host,
                   int64_t nrows, const uint64_t* s0, const uint64_t* s1, int64_t chunk_rows);

/* ======================= TreeReduce ======================================== */
/* Scratch size (bytes) needed by mb200_reduce_columns for `ncols` columns. */
size_t mb200_reduce_scratch_bytes(int ncols);
/* Column-wise reduction of one block: out_val[ncols] (double or int64 by dtype) and
 * out_cnt[ncols] (int64) are DEVICE arrays.  Deterministic (fixed tile->CTA map, fixed
 * combine order).  Float sums are Kahan-compensated per thread.
 * variant: 0 = TMA (cp.async.bulk) staged shared-memory tiles, 1 = direct 128-bit loads.
 * Reference: PandasDataframe.tree_reduce map phase df.py:2208-2250.
 */
int mb200_reduce_columns(int op, int dtype, int ncols, const void* const* in, int64_t nrows,
                         int skipna, void* out_val, int64_t* out_cnt, void* scratch,
                         int variant, mb200_stream_t stream);
/* MB200_RED_SSD: out_val[c] = sum over rows of (centers_dev[c] - x)^2, centers_dev[ncols] a DEVICE array
 * (the column means from a previous sum / count pass, so no host round trip sits between the passes).
 * Replaces the per-column work of Reduce.register(pandas.DataFrame.var / std) qc.py:1152-1153. */
int mb200_reduce_columns_centered(int op, int dtype, int ncols, const void* const* in, int64_t nrows,
                                  int skipna, const double* centers_dev, void* out_val,
                                  int64_t* out_cnt, void* scratch, int variant,
                                  mb200_stream_t stream);
/* MB200_RED_ARGMIN / MB200_RED_ARGMAX over float64 or int64 columns, one read of every element: out_val[c] = the
 * extreme value (column dtype), out_pos[c] = the first row holding it (-1 when no value is valid; out_val is then the
 * identity, +-inf or the int64 limit), out_cnt[c] = #non-NaN.  NaN is skipped; -0.0 and 0.0 tie; a tie goes to the
 * smaller row, so the result does not depend on tiles or CTAs.  Scratch and variants as for mb200_reduce_columns.
 * Replaces the per-column work of Reduce.register(pandas.DataFrame.idxmax / idxmin) qc.py:1101-1102. */
int mb200_reduce_arg_columns(int op, int dtype, int ncols, const void* const* in, int64_t nrows,
                             void* out_val, int64_t* out_pos, int64_t* out_cnt, void* scratch,
                             int variant, mb200_stream_t stream);

/* ======================= GroupByReduce ===================================== */
typedef struct mb200_gb_table mb200_gb_table; /* opaque, device resident */

/* Create an empty open-addressed table with room for `group_capacity` distinct keys and
 * `nvals` float64 accumulator columns.  flags = mb200_gb_flags. */
int mb200_gb_create(mb200_gb_table** table, int64_t group_capacity, int nvals, int flags,
                    mb200_stream_t stream);
/* Key statistics of an int64 key column into stats_dev[4] (device): {min, max, sampled, duplicated}.
 * init != 0 resets them to {INT64_MAX, INT64_MIN, 0, 0} first; several row partitions accumulate into one
 * quadruple with init = 0.  `duplicated` of the `sampled` keys shared their value with another of the 32
 * keys sampled with them: ~496/G of them for uniform keys over G values, most of them under a heavy hitter.
 * The pre-pass (8 B/row) that lets the caller choose a DENSE table when the key range is narrow and the
 * hot-key cache (mb200_gb_hint_skew) when the keys are skewed. */
int mb200_key_range(const int64_t* keys, int64_t nrows, int64_t* stats_dev, int init,
                    mb200_stream_t stream);
/* Tell the table that its keys are skewed (a few keys take a large share of the rows): accumulate calls
 * then keep a small per-CTA cache of hot groups in shared memory and add it to the table once per CTA,
 * instead of serialising every row of a hot key on one L2 line.  Supported for SUM / COUNT tables. */
int mb200_gb_hint_skew(mb200_gb_table* table, int skewed);
/* Create a DENSE (direct-addressed) table for keys known to lie in [key_min, key_max]
 * (R = key_max - key_min + 1 <= 2^29): group id = key - key_min, no hashing, no probe; one presence byte
 * per key.  Same accumulate / merge_partial / ngroups / emit / destroy calls as a hashed table; emit is
 * always key-ascending and needs no sort.  A key outside the range sets the overflow flag.
 * acc / cnt / size / present: all NULL = the library allocates; otherwise CALLER-OWNED device arrays
 * (16-byte aligned; the library initialises them and never frees them) laid out as
 *   acc[R][vs] float64 (int64 ordered images for MIN / MAX), cnt[R][vs] int64, size[R] int64,
 *   present[4 * ceil(R / 4)] uint8,      vs = max(4, nvals rounded up to a multiple of 4),
 * so that the host can run collectives on them (NCCL SUM / MIN / MAX on acc, SUM on cnt and size, MAX on
 * present merge the tables of several GPUs: the multi-GPU GroupByReduce.reduce for dense keys). */
int mb200_gb_create_dense(mb200_gb_table** table, int64_t key_min, int64_t key_max, int nvals,
                          int flags, void* acc, void* cnt, void* size, void* present,
                          mb200_stream_t stream);
/* A dense table over caller-owned arrays that ALREADY hold accumulated state in the layout above -- the slice of
 * the job-wide table this rank received from a reduce-scatter over the GPUs (NCCL SUM / MIN / MAX on acc, SUM on cnt
 * and size, MAX on present).  Nothing is initialised; mb200_gb_ngroups / mb200_gb_emit then report the slice.  This
 * is the reduce phase of GroupByReduce (alg/groupby.py:211-300) for dense keys across GPUs: each rank receives and
 * emits only its own key range. */
int mb200_gb_adopt_dense(mb200_gb_table** table, int64_t key_min, int64_t key_max, int nvals,
                         int flags, void* acc, void* cnt, void* size, void* present,
                         const mb200_gb_table* parent, mb200_stream_t stream);
/* `parent` (may be NULL): the table whose arrays were scattered; its overflow flag (a key outside the declared range
 * during accumulate) is inherited, so mb200_gb_ngroups on the slice reports it without a second host round trip. */
/* Restrict what mb200_gb_ngroups / mb200_gb_emit report to group ids [gid_lo, gid_hi) (multiples of 4,
 * or gid_hi = R): after a cross-GPU merge each rank emits its own slice of the key range. */
int mb200_gb_dense_window(mb200_gb_table* table, int64_t gid_lo, int64_t gid_hi);
int mb200_gb_destroy(mb200_gb_table* table, mb200_stream_t stream);
/* Hash-aggregate one block: keys[nrows] int64, vals[nvals][nrows] float64 (device).
 * May be called repeatedly (one call per row partition resident on this GPU);
 * replaces GroupByReduce.map alg/groupby.py:124-208 (df.groupby(by).sum() per block).
 * If the table overflows, the call succeeds but mb200_gb_ngroups reports overflow.
 * FIRST / LAST tables aggregate row POSITIONS: a position counts rows across every mb200_gb_accumulate call on the
 * table, in call order (the first row of the second call of n1 rows is position n1).  vals[v] may be NULL for them:
 * the column has no NaN (int64 / bool columns, or any column under skipna=False), every row counts and no value
 * byte is read.  min / max of positions do not depend on the order of the atomics, so the result is deterministic. */
int mb200_gb_accumulate(mb200_gb_table* table, const int64_t* keys, const void* const* vals,
                        int64_t nrows, mb200_stream_t stream);
/* Merge partial tables (keys + partial sums/counts/sizes as produced by mb200_gb_emit) into
 * `table`: replaces GroupByReduce.reduce alg/groupby.py:211-300 (groupby(level=0).sum()).
 * Refused for FIRST / LAST and ARGMIN / ARGMAX tables: positions of one table mean nothing in another; their reduce
 * re-accumulates the concatenated partial VALUES as raw rows.  mb200_gb_accumulate refuses ARGMIN / ARGMAX tables. */
int mb200_gb_merge_partial(mb200_gb_table* table, const int64_t* keys,
                           const void* const* sums, const void* const* cnts,
                           const int64_t* sizes, int64_t npartial, mb200_stream_t stream);
/* groupby.idxmin / idxmax of an ARGMIN / ARGMAX table: keys[nrows] int64, vals[nvals][nrows] float64 or int64 (bit
 * v of i64_mask set: column v is int64), row positions 0 .. nrows-1.  Two passes on `stream`: every non-NaN value
 * takes the min / max of its image into cnt (float64: f64_to_ordered with -0.0 folded into +0.0, so the two zeros
 * tie; int64: the value itself), then every row whose image equals its group's extreme takes the min of its position
 * into acc.  The maximum is unique and so is the smallest position holding it, so the result does not depend on the
 * order of the atomics.  Called once per table: a second call is refused (positions would not run on). */
int mb200_gb_accumulate_arg(mb200_gb_table* table, const int64_t* keys, const void* const* vals, uint32_t i64_mask,
                            int64_t nrows, mb200_stream_t stream);
/* Pass 2 of a VAR table (groupby.var / std): m2[g][v] += the squared deviations of the inputs from the group's mean
 * m = acc[g][v] / cnt[g][v], as pass 1 left it.  Raw form (cnts == NULL): vals[nvals][nrows] float64 values, each
 * non-NaN x adds (x - m)^2.  Partial form: the rows of other VAR tables' emits, vals = their sums S_p, cnts = their
 * counts n_p (int64), m2s = their M2_p; each row with n_p > 0 adds M2_p + n_p (S_p / n_p - m)^2 (Chan et al.'s
 * pairwise update).  Keys that are not in the table, and (group, column) pairs that pass 1 gave no value, add nothing.
 * May be called any number of times, in either form; after the first call mb200_gb_accumulate and
 * mb200_gb_merge_partial refuse the table (its means must not move).  Float atomics: the summation order is
 * run-dependent, the result is within the bound stated in README.md, not bit for bit. */
int mb200_gb_accumulate_m2(mb200_gb_table* table, const int64_t* keys, const void* const* vals,
                           const void* const* cnts, const void* const* m2s, int64_t nrows, mb200_stream_t stream);
/* The distinct set of a NUNIQUE table: open addressing over `capacity` (a power of two, at most 2^32) 16-byte slots
 * {int64 entry = gid * vstride + column, int64 image}, empty = {-1, 0}, in library-owned memory.  Allocates the set,
 * or clears it for reuse when it is already at least that large.  Must be called before mb200_gb_accumulate_distinct. */
int mb200_gb_reserve_distinct(mb200_gb_table* table, int64_t capacity, mb200_stream_t stream);
/* Pass 2 of a NUNIQUE table (groupby.nunique), after every pass-1 call.  Each (group, column, image) entry that is not
 * in the set yet is inserted and adds 1 to cnt[gid][column]; keys that are not in the table add nothing.  Images: a
 * float64 value's order-preserving int64 image with -0.0 folded into +0.0 and every NaN mapped to one image; an int64
 * value itself (bool columns are widened to int64 by the caller).
 * Raw form (col_ids == NULL): vals[nvals][nrows], column v int64 iff bit v of i64_mask is set; NaN is skipped iff
 * dropna.  Partial form (col_ids != NULL): the rows of other NUNIQUE tables' mb200_gb_emit_distinct, col_ids[nrows] and
 * images[nrows] (int64); a row with column id -1 carries its group only.  A full set raises the table's overflow flag
 * (mb200_gb_ngroups reports it).  The counts are exact whatever the order of the atomics. */
int mb200_gb_accumulate_distinct(mb200_gb_table* table, const int64_t* keys, const void* const* vals, uint32_t i64_mask,
                                 int dropna, const int64_t* col_ids, const int64_t* images, int64_t nrows,
                                 mb200_stream_t stream);
/* The distinct set of a NUNIQUE table as rows for another table's partial pass 2: out_keys / out_cols / out_images
 * [capacity] (int64) take one (key, -1, 0) row per group of the table, then one (key, column, image) row per entry, in
 * no particular order.  `ngroups` as reported by mb200_gb_ngroups.  The number of rows is decided on the device and
 * left, with an overflow flag (rows beyond `capacity`), in count_overflow_dev[2] (device int64).  Scratch as for
 * mb200_gb_emit(ngroups). */
int mb200_gb_emit_distinct(mb200_gb_table* table, int64_t ngroups, int64_t capacity, int64_t* out_keys,
                           int64_t* out_cols, int64_t* out_images, void* scratch, int64_t* count_overflow_dev,
                           mb200_stream_t stream);
/* Synchronises `stream`; returns number of groups and whether capacity was exceeded. */
int mb200_gb_ngroups(mb200_gb_table* table, int64_t* ngroups, int* overflow,
                     mb200_stream_t stream);
/* Scratch bytes needed by mb200_gb_emit for `ngroups` groups. */
size_t mb200_gb_emit_scratch_bytes(int64_t ngroups);
/* Write the result block: out_keys[ngroups] (ascending iff sort), out_sums[nvals][ngroups],
 * out_cnts[nvals][ngroups] (int64, may be NULL), out_sizes[ngroups] (may be NULL).
 * FIRST / LAST and ARGMIN / ARGMAX tables write int64 positions into out_sums, -1 where the group has no non-NaN
 * value in the column (mb200_take turns -1 into NaN).  A VAR table's out_sums holds 2 * nvals pointers: the sums
 * out_sums[0 .. nvals), then the M2s out_sums[nvals .. 2 nvals) (float64; an entry may be NULL).  A NUNIQUE table
 * writes its distinct counts into out_cnts. */
int mb200_gb_emit(mb200_gb_table* table, int64_t ngroups, int sort, int64_t* out_keys,
                  void* const* out_sums, void* const* out_cnts, int64_t* out_sizes,
                  void* scratch, mb200_stream_t stream);

/* Sync-free emit of a DENSE table: the outputs have room for `capacity` groups (>= the table's window), the number of
 * groups actually written (ascending keys, first entries of every output) is decided on the device and left, with the
 * table's overflow flag, in count_overflow_dev[2] (device int64) -- no host round trip sits between the accumulate
 * and the emit, so a stream of groupby queries keeps the GPU busy while the host prepares the next one.  Scratch as
 * for mb200_gb_emit(capacity). */
int mb200_gb_emit_dense_async(mb200_gb_table* table, int64_t capacity, int64_t* out_keys,
                              void* const* out_sums, void* const* out_cnts, int64_t* out_sizes,
                              void* scratch, int64_t* count_overflow_dev, mb200_stream_t stream);

/* ======================= broadcast hash join =============================== */
typedef struct mb200_join_table mb200_join_table;
/* Build a hash table over the (broadcast) right/dim key column.
 * Replaces the right side of pandas.merge in MergeImpl.row_axis_merge merge.py:104-252. */
int mb200_join_build(mb200_join_table** table, const int64_t* dim_keys, int64_t ndim,
                     mb200_stream_t stream);
int mb200_join_destroy(mb200_join_table* table, mb200_stream_t stream);
/* 1 if every dim key is distinct (many-to-one probe is valid), else 0. Synchronises. */
int mb200_join_is_unique(mb200_join_table* table, int* unique, mb200_stream_t stream);
/* many-to-one probe: out_idx[i] = row of fact_keys[i] in dim, or -1. Also counts matches. */
int mb200_join_probe(mb200_join_table* table, const int64_t* fact_keys, int64_t nfact,
                     int64_t* out_idx, int64_t* out_nmatch_dev, mb200_stream_t stream);
/* fused left-join payload gather for unique dim keys:
 * out[c][i] = hit ? dim_cols[c][idx] : NaN  (float64 payload; int64 payload promoted by caller).
 * out_nmatch_dev may be NULL.  A dense table probed with float64 payload and no match count keeps key-ordered
 * copies of the payload columns (range x 8 B each, cached by source pointer until the table is destroyed or other
 * columns are passed: the caller must keep the payload buffers alive that long) and reads one value per row. */
int mb200_join_probe_gather(mb200_join_table* table, const int64_t* fact_keys, int64_t nfact,
                            int ncols, const void* const* dim_cols, int dim_dtype,
                            void* const* out_cols, int64_t* out_nmatch_dev,
                            mb200_stream_t stream);
/* take: out[c][i] = idx[i] >= 0 ? src[c][idx[i]] : null_value (gather rows). */
int mb200_take(int dtype, int ncols, const void* const* src, const int64_t* idx, int64_t nidx,
               void* const* out, mb200_stream_t stream);
/* stream compaction of rows where idx >= 0: writes positions; returns count via device ptr. */
int mb200_compact_hits(const int64_t* idx, int64_t n, int64_t* out_pos, int64_t* out_count_dev,
                       void* scratch, size_t scratch_bytes, mb200_stream_t stream);

/* ---- many-to-many merge (duplicate keys on the broadcast side; merge.py:139-168 is plain pandas.merge per block) ----
 * The right keys are sorted with their row ids (mb200_sort_pairs_i64); mb200_run_heads marks the first row of every
 * run of equal keys (idx_out[i] = i at a run head, else -1; feed it to mb200_compact_hits to get starts[U]); the U
 * distinct keys go into a join table, so the probe stays many-to-one and returns u[i] = run of fact row i or -1. */
int mb200_run_heads(const int64_t* sorted_keys, int64_t n, int64_t* idx_out, mb200_stream_t stream);
/* Per left row: cnt[i] = rows it produces (length of run u[i]; 1 for a miss when keep_misses, the LEFT join; else 0),
 * first[i] = start of its run in the sorted right rows (or -1). */
int mb200_expand_counts(const int64_t* u, int64_t n, const int64_t* starts, int64_t nuniq, int64_t nright,
                        int keep_misses, int64_t* cnt, int64_t* first, mb200_stream_t stream);
/* Exclusive prefix sum of int64 values: out_offsets[i] = values[0] + ... + values[i - 1]; *out_total_dev = the sum
 * (device).  scratch_bytes >= mb200_scan_scratch_bytes(n). */
size_t mb200_scan_scratch_bytes(int64_t n);
int mb200_scan_i64(const int64_t* values, int64_t n, int64_t* out_offsets, int64_t* out_total_dev, void* scratch,
                   size_t scratch_bytes, mb200_stream_t stream);
/* Left row i writes its cnt[i] output pairs at offsets[i]: out_left = i, out_right = order[first[i] + j] (the right
 * row ids in key-sorted order) or -1 for a miss.  The result columns are mb200_take gathers of the two. */
int mb200_expand_rows(const int64_t* offsets, const int64_t* cnt, const int64_t* first, const int64_t* order,
                      int64_t n, int64_t* out_left, int64_t* out_right, mb200_stream_t stream);

/* ---- Fold template: cumulative functions down the rows (alg/fold.py:32-95 -> PandasDataframe.fold, df.py:2357-2400;
 * registrations qc.py:2429-2431 cummax / cummin / cumsum, and fillna(method="ffill"), qc.py:2809-2810).  pandas skips
 * NaN: the running value ignores them, the output keeps NaN where the input has it (FFILL: the running value goes
 * everywhere).  Two phases so that a frame sharded over ranks (or cut into several row partitions) needs one pass:
 *   mb200_cum_partials  per 4096-row tile aggregates, scanned per column into `scratch`; totals_dev[j] (may be NULL)
 *                       = the aggregate of the whole column j -- what the ranks exchange;
 *   mb200_cum_carry     carry_dev[j] = totals of ranks 0 .. rank-1 combined in rank order, from the all-gathered
 *                       totals [nranks][ncols];
 *   mb200_cum_apply     out[j][i] = carry (+) rows 0 .. i of column j  (carry_dev may be NULL; out may alias in).
 * in / out: HOST arrays of ncols device column pointers (8-byte aligned; any ncols, 32 per launch); dtype MB200_F64
 * or MB200_I64 (FFILL: float64 only); scratch_bytes >= mb200_cum_scratch_bytes(ncols, nrows); the same scratch goes
 * from partials to apply.  Sums re-associate (tile tree instead of pandas' sequential loop); max / min / ffill and
 * int64 results are exact. */
enum mb200_cum_op { MB200_CUM_SUM = 0, MB200_CUM_MAX = 1, MB200_CUM_MIN = 2, MB200_CUM_FFILL = 3 };
size_t mb200_cum_scratch_bytes(int ncols, int64_t nrows);
int mb200_cum_partials(int op, int dtype, int ncols, const void* const* in, int64_t nrows, void* scratch,
                       size_t scratch_bytes, void* totals_dev, mb200_stream_t stream);
int mb200_cum_carry(int op, int dtype, int ncols, const void* gathered_totals_dev, int rank, void* carry_dev,
                    mb200_stream_t stream);
int mb200_cum_apply(int op, int dtype, int ncols, const void* const* in, void* const* out, int64_t nrows,
                    const void* scratch, const void* carry_dev, mb200_stream_t stream);

/* Range-partitioning shuffle, split step (ShuffleSortFunctions.split_partitions, dfutils.py:355-475: np.digitize of
 * the key column against the sampled pivots): out_bins[i] = number of pivots <= values[i]; pivots_dev ascending,
 * npivots <= 1023.  Keys go in as their order-preserving int64 image (MB200_OP_ORDERED_S). */
int mb200_digitize_i64(const int64_t* values, int64_t n, const int64_t* pivots_dev, int npivots,
                       int64_t* out_bins, mb200_stream_t stream);

/* ======================= synthetic data (from_map-style generators) ======== */
/* Counter-based generators, reproducible for any row range; the numpy twin lives in
 * modin_b200/synth.py.  value(row, col) depends only on (seed, col, row_offset + i).
 * gen_f64: approx N(0,1) (Irwin-Hall of 4 exact uniforms); nan_per_64k of every 65536
 * values are NaN.  gen_i64: uniform integer in [0, modulus). */
int mb200_gen_f64(double* out, int64_t nrows, uint64_t seed, uint64_t col, int64_t row_offset,
                  int nan_per_64k, mb200_stream_t stream);
/* stats_dev (may be NULL): DEVICE int64[4] that receives the generated column's key statistics {min, max, sampled,
 * duplicated} (same quadruple as mb200_key_range) -- the producing kernel leaves them behind as column metadata,
 * so a groupby on the column needs no 8 B/row pre-pass. */
int mb200_gen_i64(int64_t* out, int64_t nrows, uint64_t seed, uint64_t col, int64_t row_offset,
                  uint64_t modulus, int64_t* stats_dev, mb200_stream_t stream);
/* Skewed keys in [0, modulus) (the Zipf-like variant of the groupby workload): mass per octave of the key
 * space grows towards small keys like k^-1.1 -- for modulus = 1e6 key 0 takes ~11 % of the rows. */
int mb200_gen_i64_skew(int64_t* out, int64_t nrows, uint64_t seed, uint64_t col, int64_t row_offset,
                       uint64_t modulus, int64_t* stats_dev, mb200_stream_t stream);

/* Row labels of a RangeIndex block as a device column: out[i] = start + i.  The labels a block needs on the device
 * when it is re-indexed against another frame's labels (PandasDataframe._copartition, df.py:3799-3840). */
int mb200_iota_i64(int64_t* out, int64_t nrows, int64_t start, mb200_stream_t stream);
/* Constant column of 8-byte elements: out[i] = bits (a float64 / int64 bit pattern; NaN columns for labels that
 * re-indexing adds). */
int mb200_fill_u64(void* out, int64_t n, uint64_t bits, mb200_stream_t stream);

/* Row-wise concatenation of column pieces: dst = src[0] | src[1] | ... (src_bytes[i] bytes each; HOST arrays of
 * device pointers / sizes), one launch per 64 sources.  Replaces the pandas.concat of the gathered blocks of an axis
 * partition (PandasDataframeAxisPartition.deploy_axis_func, axpart.py:445-452) and pm.combine (pm.py:1328-1373). */
int mb200_concat(int nsrc, const void* const* src, const int64_t* src_bytes, void* dst, mb200_stream_t stream);

/* ======================= collectives (NCCL over NVLink 5 / NVSwitch) ======= */
/* The reference issues no collective: it gathers all blocks of an axis into one task (axis_partition.py:445-452),
 * hands one object to many tasks (pm.py:443-494) or shuffles rows between partitions (pm.py:1937-2052).  With one
 * process per GPU those steps are the calls below, issued on the caller's stream on device buffers.  NCCL is resolved
 * at run time: mb200_comm_load(path or NULL) once per process; rank 0 calls mb200_comm_unique_id and the host side
 * carries the 128 bytes to every rank (any control channel), then every rank calls mb200_comm_init_rank. */
typedef struct mb200_comm mb200_comm;
enum mb200_comm_op { MB200_COMM_SUM = 0, MB200_COMM_MIN = 1, MB200_COMM_MAX = 2 };
int mb200_comm_load(const char* libnccl_path);
int mb200_comm_unique_id(void* out128);
int mb200_comm_init_rank(mb200_comm** comm, int nranks, const void* id128, int rank);
int mb200_comm_destroy(mb200_comm* comm);
/* TreeReduce combine (W-vector) and the element-wise merge of dense group tables. */
int mb200_comm_allreduce(mb200_comm* comm, const void* send, void* recv, int64_t count, int dtype, int op,
                         mb200_stream_t stream);
/* Reduce phase of GroupByReduce for dense keys: rank r receives elements [r * recvcount, (r + 1) * recvcount). */
int mb200_comm_reduce_scatter(mb200_comm* comm, const void* send, void* recv, int64_t recvcount, int dtype,
                              int op, mb200_stream_t stream);
/* Broadcast merge: every rank's (equal-length, padded) shard of a dim column -> the whole column everywhere. */
int mb200_comm_allgather(mb200_comm* comm, const void* send, void* recv, int64_t sendcount, int dtype,
                         mb200_stream_t stream);
int mb200_comm_broadcast(mb200_comm* comm, void* buf, int64_t count, int dtype, int root, mb200_stream_t stream);
/* Range-partitioning shuffle / exchange of partial group tables: counts and displacements in ELEMENTS of elem_bytes
 * (HOST arrays of length nranks); grouped ncclSend / ncclRecv. */
int mb200_comm_alltoallv(mb200_comm* comm, const void* send, const int64_t* sendcounts, const int64_t* sdispls,
                         void* recv, const int64_t* recvcounts, const int64_t* rdispls, int elem_bytes,
                         mb200_stream_t stream);

/* ======================= utilities ========================================= */
/* Stable LSD radix sort of (key, payload) pairs by key ascending (signed), in place.
 * scratch_bytes >= mb200_sort_scratch_bytes(n). */
size_t mb200_sort_scratch_bytes(int64_t n);
int mb200_sort_pairs_i64(int64_t* keys, int64_t* payload, int64_t n, void* scratch,
                         size_t scratch_bytes, mb200_stream_t stream);
/* Bytes of L2 the device can pin (persisting carve-out) and the largest access-policy window; the
 * groupby kernels pin the accumulator rows of tables larger than L2/2. */
int mb200_l2_persist_info(int* max_persist_bytes, int* max_window_bytes);
/* Write >= L2-sized buffer to evict L2 between timed iterations. */
int mb200_flush_l2(void* buf, size_t bytes, mb200_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* MODIN_B200_H */
