"""ctypes binding of libmodin_b200.so (the C ABI declared in include/modin_b200.h).

This is the binding a Modin maintainer would add next to the partition classes
(INTEGRATION.md): every per-block pandas call on the hot path goes through one of these
entry points instead.  There is no CPU fallback: if the library is missing or no sm_90
device is present, calls raise ``B200Error``.
"""

from __future__ import annotations

import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_native", "libmodin_b200.so")


class B200Error(RuntimeError):
    """Raised when a libmodin_b200 call fails (message from mb200_last_error)."""


ABI_VERSION = 7

# enums (keep in sync with include/modin_b200.h)
F64, I64, U8 = 0, 1, 2
MAX_COLS = 32  # MB200_MAX_COLS: columns of one dtype per launch / value columns per group table

OP = {
    "abs": 0, "neg": 1, "isna": 2, "notna": 3, "fillna_s": 4, "affine": 5,
    "add_s": 6, "sub_s": 7, "rsub_s": 8, "mul_s": 9, "div_s": 10, "rdiv_s": 11,
    "eq_s": 12, "ne_s": 13, "lt_s": 14, "le_s": 15, "gt_s": 16, "ge_s": 17,
    "clip_s": 18, "copy": 19, "round_s": 20, "ordered_s": 21, "not": 22,
    "and": 43, "or": 44, "xor": 45,
    "add": 32, "sub": 33, "mul": 34, "div": 35, "eq": 36, "ne": 37, "lt": 38, "le": 39,
    "gt": 40, "ge": 41, "fillna": 42,
    "fma3": 64,
}  # fmt: skip
PREDICATES = {"isna", "notna", "eq_s", "ne_s", "lt_s", "le_s", "gt_s", "ge_s", "eq", "ne", "lt", "le", "gt", "ge"}
RED = {"sum": 0, "min": 1, "max": 2, "count": 3, "prod": 4, "ssd": 5, "argmin": 6, "argmax": 7}
CUM = {"sum": 0, "max": 1, "min": 2, "ffill": 3}
GB_SUM, GB_COUNT, GB_SIZE, GB_MIN, GB_MAX = 1, 2, 4, 8, 16
GB_FIRST, GB_LAST = 32, 64  # int64 row positions instead of values (include/modin_b200.h)
GB_ARGMIN, GB_ARGMAX = 128, 256  # the first row holding each group's extreme (mb200_gb_accumulate_arg)
GB_VAR = 512  # SUM | COUNT | VAR: sums of squared deviations from the group means (mb200_gb_accumulate_m2)
GB_NUNIQUE = 1024  # SIZE | NUNIQUE: distinct counts through the table's distinct set (mb200_gb_accumulate_distinct)

_vp = C.c_void_p
_vpp = C.POINTER(C.c_void_p)
_i64 = C.c_int64
_u64p = C.POINTER(C.c_uint64)

_SIGNATURES = {
    "mb200_abi_version": (C.c_int, []),
    "mb200_last_error": (C.c_char_p, []),
    "mb200_device_check": (C.c_int, [C.c_int]),
    "mb200_device_info": (C.c_int, [C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t),
                                     C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "mb200_set_device": (C.c_int, [C.c_int]),
    "mb200_alloc": (C.c_int, [_vpp, C.c_size_t, _vp]),
    "mb200_free": (C.c_int, [_vp, _vp]),
    "mb200_alloc_host": (C.c_int, [_vpp, C.c_size_t]),
    "mb200_free_host": (C.c_int, [_vp]),
    "mb200_h2d": (C.c_int, [_vp, _vp, C.c_size_t, _vp]),
    "mb200_d2h": (C.c_int, [_vp, _vp, C.c_size_t, _vp]),
    "mb200_d2d": (C.c_int, [_vp, _vp, C.c_size_t, _vp]),
    "mb200_memset": (C.c_int, [_vp, C.c_int, C.c_size_t, _vp]),
    "mb200_stream_sync": (C.c_int, [_vp]),
    "mb200_launch_count": (_i64, []),
    "mb200_map": (C.c_int, [C.c_int, C.c_int, C.c_int, _vpp, _vpp, _vpp, _vpp, _i64, _u64p, _u64p, _vp]),
    "mb200_map_host": (C.c_int, [C.c_int, C.c_int, C.c_int, _vpp, _vpp, _vpp, _vpp, _i64, _u64p, _u64p, _i64]),
    "mb200_reduce_scratch_bytes": (C.c_size_t, [C.c_int]),
    "mb200_reduce_columns": (C.c_int, [C.c_int, C.c_int, C.c_int, _vpp, _i64, C.c_int, _vp, _vp, _vp, C.c_int, _vp]),
    "mb200_reduce_columns_centered": (C.c_int, [C.c_int, C.c_int, C.c_int, _vpp, _i64, C.c_int, _vp, _vp, _vp, _vp,
                                                C.c_int, _vp]),
    "mb200_reduce_arg_columns": (C.c_int, [C.c_int, C.c_int, C.c_int, _vpp, _i64, _vp, _vp, _vp, _vp, C.c_int, _vp]),
    "mb200_gb_create": (C.c_int, [_vpp, _i64, C.c_int, C.c_int, _vp]),
    "mb200_key_range": (C.c_int, [_vp, _i64, _vp, C.c_int, _vp]),
    "mb200_gb_create_dense": (C.c_int, [_vpp, _i64, _i64, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp]),
    "mb200_gb_adopt_dense": (C.c_int, [_vpp, _i64, _i64, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mb200_gb_dense_window": (C.c_int, [_vp, _i64, _i64]),
    "mb200_gb_hint_skew": (C.c_int, [_vp, C.c_int]),
    "mb200_gb_destroy": (C.c_int, [_vp, _vp]),
    "mb200_gb_accumulate": (C.c_int, [_vp, _vp, _vpp, _i64, _vp]),
    "mb200_gb_accumulate_arg": (C.c_int, [_vp, _vp, _vpp, C.c_uint32, _i64, _vp]),
    "mb200_gb_merge_partial": (C.c_int, [_vp, _vp, _vpp, _vpp, _vp, _i64, _vp]),
    "mb200_gb_accumulate_m2": (C.c_int, [_vp, _vp, _vpp, _vpp, _vpp, _i64, _vp]),
    "mb200_gb_reserve_distinct": (C.c_int, [_vp, _i64, _vp]),
    "mb200_gb_accumulate_distinct": (C.c_int, [_vp, _vp, _vpp, C.c_uint32, C.c_int, _vp, _vp, _i64, _vp]),
    "mb200_gb_emit_distinct": (C.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mb200_gb_ngroups": (C.c_int, [_vp, C.POINTER(_i64), C.POINTER(C.c_int), _vp]),
    "mb200_gb_emit_scratch_bytes": (C.c_size_t, [_i64]),
    "mb200_gb_emit": (C.c_int, [_vp, _i64, C.c_int, _vp, _vpp, _vpp, _vp, _vp, _vp]),
    "mb200_gb_emit_dense_async": (C.c_int, [_vp, _i64, _vp, _vpp, _vpp, _vp, _vp, _vp, _vp]),
    "mb200_join_build": (C.c_int, [_vpp, _vp, _i64, _vp]),
    "mb200_join_destroy": (C.c_int, [_vp, _vp]),
    "mb200_join_is_unique": (C.c_int, [_vp, C.POINTER(C.c_int), _vp]),
    "mb200_join_probe": (C.c_int, [_vp, _vp, _i64, _vp, _vp, _vp]),
    "mb200_join_probe_gather": (C.c_int, [_vp, _vp, _i64, C.c_int, _vpp, C.c_int, _vpp, _vp, _vp]),
    "mb200_take": (C.c_int, [C.c_int, C.c_int, _vpp, _vp, _i64, _vpp, _vp]),
    "mb200_compact_hits": (C.c_int, [_vp, _i64, _vp, _vp, _vp, C.c_size_t, _vp]),
    "mb200_run_heads": (C.c_int, [_vp, _i64, _vp, _vp]),
    "mb200_expand_counts": (C.c_int, [_vp, _i64, _vp, _i64, _i64, C.c_int, _vp, _vp, _vp]),
    "mb200_scan_scratch_bytes": (C.c_size_t, [_i64]),
    "mb200_scan_i64": (C.c_int, [_vp, _i64, _vp, _vp, _vp, C.c_size_t, _vp]),
    "mb200_expand_rows": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp]),
    "mb200_digitize_i64": (C.c_int, [_vp, _i64, _vp, C.c_int, _vp, _vp]),
    "mb200_gen_f64": (C.c_int, [_vp, _i64, C.c_uint64, C.c_uint64, _i64, C.c_int, _vp]),
    "mb200_gen_i64": (C.c_int, [_vp, _i64, C.c_uint64, C.c_uint64, _i64, C.c_uint64, _vp, _vp]),
    "mb200_gen_i64_skew": (C.c_int, [_vp, _i64, C.c_uint64, C.c_uint64, _i64, C.c_uint64, _vp, _vp]),
    "mb200_comm_load": (C.c_int, [C.c_char_p]),
    "mb200_comm_unique_id": (C.c_int, [_vp]),
    "mb200_comm_init_rank": (C.c_int, [_vpp, C.c_int, _vp, C.c_int]),
    "mb200_comm_destroy": (C.c_int, [_vp]),
    "mb200_comm_allreduce": (C.c_int, [_vp, _vp, _vp, _i64, C.c_int, C.c_int, _vp]),
    "mb200_comm_reduce_scatter": (C.c_int, [_vp, _vp, _vp, _i64, C.c_int, C.c_int, _vp]),
    "mb200_comm_allgather": (C.c_int, [_vp, _vp, _vp, _i64, C.c_int, _vp]),
    "mb200_comm_broadcast": (C.c_int, [_vp, _vp, _i64, C.c_int, C.c_int, _vp]),
    "mb200_comm_alltoallv": (C.c_int, [_vp, _vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64), _vp, C.POINTER(C.c_int64),
                                       C.POINTER(C.c_int64), C.c_int, _vp]),
    "mb200_concat": (C.c_int, [C.c_int, _vpp, C.POINTER(C.c_int64), _vp, _vp]),
    "mb200_cum_scratch_bytes": (C.c_size_t, [C.c_int, _i64]),
    "mb200_cum_partials": (C.c_int, [C.c_int, C.c_int, C.c_int, _vpp, _i64, _vp, C.c_size_t, _vp, _vp]),
    "mb200_cum_carry": (C.c_int, [C.c_int, C.c_int, C.c_int, _vp, C.c_int, _vp, _vp]),
    "mb200_cum_apply": (C.c_int, [C.c_int, C.c_int, C.c_int, _vpp, _vpp, _i64, _vp, _vp, _vp]),
    "mb200_iota_i64": (C.c_int, [_vp, _i64, _i64, _vp]),
    "mb200_fill_u64": (C.c_int, [_vp, _i64, C.c_uint64, _vp]),
    "mb200_sort_scratch_bytes": (C.c_size_t, [_i64]),
    "mb200_sort_pairs_i64": (C.c_int, [_vp, _vp, _i64, _vp, C.c_size_t, _vp]),
    "mb200_l2_persist_info": (C.c_int, [C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "mb200_flush_l2": (C.c_int, [_vp, C.c_size_t, _vp]),
}  # fmt: skip

EXPORTED_SYMBOLS = tuple(_SIGNATURES)

_lib = None
_lock = threading.Lock()


def load() -> C.CDLL:
    """Load the shared library (once) and attach signatures.  Raises B200Error if missing."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise B200Error(
                f"{LIB_PATH} is missing: build it with `python -m modin_b200.build` "
                "(modin_b200 has no CPU fallback on the partition-execution path)"
            )
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        if lib.mb200_abi_version() != ABI_VERSION:
            raise B200Error("libmodin_b200 ABI version mismatch")
        _lib = lib
        return lib


def check(rc: int) -> None:
    if rc != 0:
        msg = load().mb200_last_error()
        raise B200Error(msg.decode() if msg else f"libmodin_b200 call failed with status {rc}")


def ptr_array(ptrs) -> C.Array:
    """Host array of device pointers for the `const void* const*` parameters."""
    arr = (C.c_void_p * max(len(ptrs), 1))()
    for i, p in enumerate(ptrs):
        arr[i] = p
    return arr


def u64_array(vals) -> C.Array:
    arr = (C.c_uint64 * max(len(vals), 1))()
    for i, v in enumerate(vals):
        arr[i] = v
    return arr
