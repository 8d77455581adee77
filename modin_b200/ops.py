"""Block-level operations: DeviceBlock in, DeviceBlock out, every one a libmodin_b200 call.

These are the bodies that replace the per-block pandas calls of the reference
(``func(self._data.copy())`` in pandas_on_python/partitioning/partition.py:76-123).
No function here touches a host copy of the data, and none has a CPU branch.
"""

from __future__ import annotations

import ctypes as C
import os
from typing import List, NamedTuple, Optional, Sequence

import numpy as np

from . import _lib
from .block import DeviceColumn, KeyStats, current_device, current_stream, torch_mod

_scratch_cache = {}


class KernelTimer:
    """Measurement hook (bench.py): while installed, the wrappers of the dominant kernels bracket their C call with
    CUDA events on the launching stream, so that a kernel's own duration can be read apart from the step around it.
    ``with KernelTimer() as kt: ...; kt.mean_ms("gb_accumulate")`` (synchronises when read)."""

    active = None

    def __init__(self):
        self.events = {}

    def __enter__(self):
        KernelTimer.active = self
        return self

    def __exit__(self, *exc):
        KernelTimer.active = None
        return False

    def mean_ms(self, tag):
        torch_mod().cuda.synchronize()
        ev = self.events.get(tag, [])
        return sum(a.elapsed_time(b) for a, b in ev) / len(ev) if ev else None

    def total_ms(self, tag):
        torch_mod().cuda.synchronize()
        ev = self.events.get(tag, [])
        return sum(a.elapsed_time(b) for a, b in ev) if ev else None

    def launches(self, tag):
        return len(self.events.get(tag, []))


class _timed:
    """Bracket one C call with events when a KernelTimer is installed (no-op otherwise)."""

    def __init__(self, tag):
        self.tag, self.kt = tag, KernelTimer.active

    def __enter__(self):
        if self.kt is not None:
            t = torch_mod()
            self.a, self.b = t.cuda.Event(enable_timing=True), t.cuda.Event(enable_timing=True)
            self.a.record()

    def __exit__(self, *exc):
        if self.kt is not None:
            self.b.record()
            self.kt.events.setdefault(self.tag, []).append((self.a, self.b))
        return False


def _scratch(nbytes: int, tag: str = "default"):
    """Per-device reusable scratch buffer (grown geometrically)."""
    t = torch_mod()
    key = (t.cuda.current_device(), tag)
    buf = _scratch_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = t.empty(max(int(nbytes), 1 << 20), dtype=t.uint8, device=current_device())
        _scratch_cache[key] = buf
    return buf


def f64_bits(x: float) -> int:
    return int(np.float64(x).view(np.uint64))


def i64_bits(x: int) -> int:
    return int(np.int64(x).view(np.uint64))


def _scalar_bits(vals, code):
    if vals is None:
        return None
    conv = f64_bits if code == _lib.F64 else i64_bits
    return _lib.u64_array([conv(v) for v in vals])


# ------------------------------------------------------------------ Map / Binary
def map_columns(
    op: str,
    in0: Sequence[DeviceColumn],
    in1: Optional[Sequence[DeviceColumn]] = None,
    in2: Optional[Sequence[DeviceColumn]] = None,
    s0: Optional[Sequence] = None,
    s1: Optional[Sequence] = None,
) -> List[DeviceColumn]:
    """Elementwise op over W columns of equal dtype with ONE kernel launch per dtype group."""
    lib = _lib.load()
    n = len(in0[0]) if in0 else 0
    out: List[Optional[DeviceColumn]] = [None] * len(in0)
    groups = {}
    for j, c in enumerate(in0):
        groups.setdefault(c.code, []).append(j)
    for code, idxs in groups.items():
        if code == _lib.U8:
            if op not in ("copy", "not", "and", "or", "xor"):
                raise TypeError(f"elementwise {op!r} on bool columns is not on the B200 path")
            odt = np.dtype("int64") if op == "copy" else np.dtype("bool")  # copy widens bool -> int64
        elif op in _lib.PREDICATES:
            odt = np.dtype("bool")
        elif op in ("div", "div_s", "rdiv_s"):
            odt = np.dtype("float64")
        elif op == "ordered_s":
            odt = np.dtype("int64")
        else:
            odt = in0[idxs[0]].dtype
        for k in range(0, len(idxs), _lib.MAX_COLS):
            sel = idxs[k : k + _lib.MAX_COLS]
            outs = [DeviceColumn.empty(n, odt) for _ in sel]
            a = _lib.ptr_array([in0[j].ptr for j in sel])
            b = _lib.ptr_array([in1[j].ptr for j in sel]) if in1 is not None else None
            c = _lib.ptr_array([in2[j].ptr for j in sel]) if in2 is not None else None
            if in1 is not None and any(in1[j].code != code for j in sel):
                raise TypeError("mixed dtypes between operands of a device binary op")
            if in2 is not None and any(in2[j].code != code for j in sel):
                raise TypeError("mixed dtypes between operands of a device ternary op")
            o = _lib.ptr_array([x.ptr for x in outs])
            s0a = _scalar_bits([s0[j] for j in sel], code) if s0 is not None else None
            s1a = _scalar_bits([s1[j] for j in sel], code) if s1 is not None else None
            with _timed("map_" + op):
                _lib.check(lib.mb200_map(_lib.OP[op], code, len(sel), a, b, c, o, n, s0a, s1a, current_stream()))
            for j, x in zip(sel, outs):
                out[j] = x
    return out  # type: ignore[return-value]


def cast_columns_i64(cols: Sequence[DeviceColumn]) -> List[DeviceColumn]:
    """bool -> int64 widening (what pandas does before it sums / averages booleans); others unchanged."""
    return [map_columns("copy", [c])[0] if c.dtype == np.bool_ else c for c in cols]


def cast_columns_f64(cols: Sequence[DeviceColumn]) -> List[DeviceColumn]:
    """int64 -> float64 promotion (x / 1.0 through the division kernel); bool goes through int64."""
    res = []
    for c in cols:
        if c.dtype == np.float64:
            res.append(c)
        elif c.dtype == np.bool_:
            res.extend(map_columns("div_s", cast_columns_i64([c]), s0=[1]))
        elif c.dtype == np.int64:
            res.extend(map_columns("div_s", [c], s0=[1]))
        else:
            raise TypeError(f"cannot promote {c.dtype} to float64 on device")
    return res


# ------------------------------------------------------------------ TreeReduce
def reduce_columns(op: str, cols: Sequence[DeviceColumn], skipna: bool = True, variant: int = 0, centers=None):
    """Column-wise reduction.  Returns (values DeviceColumn-per-dtype-group arrays, counts).

    ``op="ssd"`` (sum of squared deviations, float64 only) takes ``centers``: a float64 device tensor with one
    centre per column.

    Output: list of (value_tensor_1elem_view, count_tensor_1elem_view) is avoided; instead two
    device tensors of length W are returned per dtype group, mapped back to column order:
    ``vals[j]`` is a 0-d device view (float64 or int64), ``cnts[j]`` a 0-d int64 view.
    """
    lib = _lib.load()
    t = torch_mod()
    n = len(cols[0]) if cols else 0
    vals: list = [None] * len(cols)
    cnts: list = [None] * len(cols)
    groups = {}
    for j, c in enumerate(cols):
        groups.setdefault(c.code, []).append(j)
    for code, idxs in groups.items():
        if code == _lib.U8:
            raise TypeError("reductions over bool columns are not on the B200 path")
        # 8 columns per launch: the TMA ring and the tile -> CTA map are sized for 8 streams per CTA
        per = int(os.environ.get("MB200_REDUCE_COLS_PER_LAUNCH", "8"))
        for k in range(0, len(idxs), per):
            sel = idxs[k : k + per]
            odt = t.float64 if code == _lib.F64 else t.int64
            oval = t.empty(len(sel), dtype=odt, device=current_device())
            ocnt = t.empty(len(sel), dtype=t.int64, device=current_device())
            scratch = _scratch(lib.mb200_reduce_scratch_bytes(len(sel)), "reduce")
            ptrs = _lib.ptr_array([cols[j].ptr for j in sel])
            if op == "ssd":
                if code != _lib.F64 or centers is None:
                    raise TypeError("ssd reduces float64 columns around given centres")
                cen = centers[t.tensor(sel, device=centers.device)].contiguous() if len(sel) != len(cols) else centers
                _lib.check(
                    lib.mb200_reduce_columns_centered(
                        _lib.RED[op], code, len(sel), ptrs, n, 1 if skipna else 0, cen.data_ptr(), oval.data_ptr(),
                        ocnt.data_ptr(), scratch.data_ptr(), variant, current_stream(),
                    )
                )  # fmt: skip
            else:
                with _timed("reduce_" + op):
                    _lib.check(
                        lib.mb200_reduce_columns(
                            _lib.RED[op], code, len(sel), ptrs, n, 1 if skipna else 0, oval.data_ptr(), ocnt.data_ptr(),
                            scratch.data_ptr(), variant, current_stream(),
                        )
                    )  # fmt: skip
            for pos, j in enumerate(sel):
                vals[j] = oval[pos : pos + 1]
                cnts[j] = ocnt[pos : pos + 1]
    return vals, cnts


def arg_reduce_columns(op: str, cols: Sequence[DeviceColumn], variant: int = 0):
    """Column-wise extreme value and the first row holding it (``op`` "max" / "min"; idxmax / idxmin) in one pass.

    Returns ``(vals, poss, cnts)``, 1-element device views per column in column order: the extreme value in the
    column's dtype, its row position (-1 when the column holds no valid value) and the number of non-NaN values.
    float64 / int64 columns; 8 columns per launch, like ``reduce_columns``."""
    lib = _lib.load()
    t = torch_mod()
    code_op = _lib.RED["arg" + op]
    n = len(cols[0]) if cols else 0
    vals: list = [None] * len(cols)
    poss: list = [None] * len(cols)
    cnts: list = [None] * len(cols)
    groups = {}
    for j, c in enumerate(cols):
        groups.setdefault(c.code, []).append(j)
    for code, idxs in groups.items():
        if code == _lib.U8:
            raise TypeError("arg-reductions over bool columns are not on the B200 path (widen them to int64)")
        for k in range(0, len(idxs), 8):
            sel = idxs[k : k + 8]
            oval = t.empty(len(sel), dtype=t.float64 if code == _lib.F64 else t.int64, device=current_device())
            opos = t.empty(len(sel), dtype=t.int64, device=current_device())
            ocnt = t.empty(len(sel), dtype=t.int64, device=current_device())
            scratch = _scratch(lib.mb200_reduce_scratch_bytes(len(sel)), "reduce")
            with _timed("reduce_arg" + op):
                _lib.check(lib.mb200_reduce_arg_columns(code_op, code, len(sel), _lib.ptr_array([cols[j].ptr for j in sel]),
                                                        n, oval.data_ptr(), opos.data_ptr(), ocnt.data_ptr(),
                                                        scratch.data_ptr(), variant, current_stream()))  # fmt: skip
            for pos, j in enumerate(sel):
                vals[j], poss[j], cnts[j] = oval[pos : pos + 1], opos[pos : pos + 1], ocnt[pos : pos + 1]
    return vals, poss, cnts


# ------------------------------------------------------------------ GroupByReduce
_GB_ARG = _lib.GB_ARGMIN | _lib.GB_ARGMAX  # idxmin / idxmax: extreme images in ``cnt``, row positions in ``acc``
_GB_POS = _lib.GB_FIRST | _lib.GB_LAST | _GB_ARG  # tables of int64 row positions (first / last / idxmin / idxmax)
_GB_ACC = _lib.GB_SUM | _lib.GB_MIN | _lib.GB_MAX | _GB_POS
_GB_CNT = _lib.GB_COUNT | _GB_ARG | _lib.GB_NUNIQUE  # tables with a ``cnt`` array (a NUNIQUE table's distinct counts)
_DENSE_ARRAYS = ("acc", "cnt", "size", "present")


def value_stride(nvals: int) -> int:
    """Accumulator slots per key of a dense table (include/modin_b200.h): ``nvals`` rounded up to 4, at least 4."""
    return max(4, (nvals + 3) & ~3)


def refuse_dense_overflow(count_overflow) -> None:
    """Raise when a dense table reports ``[groups, overflow]`` with the overflow flag set: a key fell outside the
    range the table was sized for, so some rows were not aggregated."""
    if count_overflow[1]:
        raise _lib.B200Error("dense group table saw a key outside its measured range")


class GroupTable:
    """Owner of one device group table (mb200_gb_table): hashed (``GroupTable(capacity, nvals, flags)``) or dense
    (``GroupTable.dense``; ``kbase`` is its first key, None for a hashed table)."""

    kbase = None

    def __init__(self, group_capacity: int, nvals: int, flags: int):
        self.lib = _lib.load()
        self.handle = C.c_void_p()
        self.capacity = int(group_capacity)
        self.nvals = int(nvals)
        self.flags = int(flags)
        _lib.check(self.lib.mb200_gb_create(C.byref(self.handle), self.capacity, self.nvals, self.flags,
                                            current_stream()))  # fmt: skip

    @classmethod
    def dense(cls, key_min: int, key_max: int, nvals: int, flags: int):
        """Direct-addressed table for keys in [key_min, key_max] (mb200_gb_create_dense)."""
        # the arrays live in torch's allocator (layout: include/modin_b200.h) so that the multi-GPU
        # reduce can run NCCL collectives on them in place
        t = torch_mod()
        dev = current_device()
        R, vs = int(key_max) - int(key_min) + 1, value_stride(nvals)
        arrays = {}
        if flags & _GB_ACC:
            arrays["acc"] = t.empty(R * vs, dtype=t.float64 if flags & _lib.GB_SUM else t.int64, device=dev)
        if flags & _GB_CNT:
            arrays["cnt"] = t.empty(R * vs, dtype=t.int64, device=dev)
        if flags & _lib.GB_SIZE:
            arrays["size"] = t.empty(R, dtype=t.int64, device=dev)
        arrays["present"] = t.empty(4 * ((R + 3) // 4), dtype=t.uint8, device=dev)
        return cls._dense_table(int(key_min), R, nvals, flags, arrays)

    @classmethod
    def _dense_table(cls, kbase: int, nkeys: int, nvals: int, flags: int, arrays: dict, parent=None):
        """A dense table over keys ``[kbase, kbase + nkeys)`` on the given arrays: a fresh one
        (mb200_gb_create_dense) or, with ``parent``, a slice of it that inherits its overflow flag
        (mb200_gb_adopt_dense)."""
        self = cls.__new__(cls)
        self.lib, self.handle = _lib.load(), C.c_void_p()
        self.kbase, self.capacity, self.nvals, self.flags = kbase, nkeys, int(nvals), int(flags)
        self.acc, self.cnt, self.size, self.present = (arrays.get(n) for n in _DENSE_ARRAYS)
        ptrs = [x.data_ptr() if x is not None else None for x in (self.acc, self.cnt, self.size, self.present)]
        args = (C.byref(self.handle), kbase, kbase + nkeys - 1, self.nvals, self.flags, *ptrs)
        if parent is None:
            _lib.check(self.lib.mb200_gb_create_dense(*args, current_stream()))
        else:
            _lib.check(self.lib.mb200_gb_adopt_dense(*args, parent.handle, current_stream()))
        return self

    def collective_arrays(self):
        """(tensor, reduce-op, elements per key) triples whose element-wise reduction over ranks merges dense tables."""
        acc_op = "sum" if self.flags & _lib.GB_SUM else ("min" if self.flags & (_lib.GB_MIN | _lib.GB_FIRST) else "max")
        vs = value_stride(self.nvals)
        out = [(self.acc, acc_op, vs), (self.cnt, "sum", vs), (self.size, "sum", 1), (self.present, "max", 1)]
        return [(x, op, per) for x, op, per in out if x is not None]

    def reduce_scatter(self, chunk: int, reduce_scatter_fn, r: int):
        """Cross-GPU reduce phase for dense keys: every array of this table (job-wide key range, padded to
        ``ws * chunk`` keys) is reduce-scattered over the ranks -- rank ``r`` receives keys
        ``[r * chunk, (r + 1) * chunk)`` fully merged -- and a table over just that slice is returned
        (``mb200_gb_adopt_dense``; it inherits this table's overflow flag).  Half the traffic of an all_reduce,
        and each rank counts and emits only what it owns."""
        t = torch_mod()
        if self.capacity % chunk or chunk % 4:
            raise ValueError("dense table is not padded to equal, 4-key-aligned chunks")
        names = [n for n in _DENSE_ARRAYS if getattr(self, n) is not None]
        arrays = {}
        for name, (x, op, per) in zip(names, self.collective_arrays()):
            arrays[name] = t.empty(chunk * per, dtype=x.dtype, device=x.device)
            reduce_scatter_fn(arrays[name], x[: self.capacity * per], op)
        return self._dense_table(self.kbase + r * chunk, int(chunk), self.nvals, self.flags, arrays, parent=self)

    def window(self, gid_lo: int, gid_hi: int):
        _lib.check(self.lib.mb200_gb_dense_window(self.handle, int(gid_lo), int(gid_hi)))

    def hint_skew(self, skewed: bool):
        """Skewed keys: accumulate with the per-CTA hot-group cache (mb200_gb_hint_skew)."""
        _lib.check(self.lib.mb200_gb_hint_skew(self.handle, 1 if skewed else 0))

    def accumulate(self, keys: DeviceColumn, vals: Sequence[Optional[DeviceColumn]]):
        """Aggregate rows ``keys`` / ``vals`` (float64 columns).  A first / last table also takes None for a column
        without NaN: every row of it counts.  Positions run on across calls, in call order.  An idxmin / idxmax table
        takes float64 and int64 columns, in ONE call (mb200_gb_accumulate_arg): its positions are that call's rows."""
        if keys.dtype != np.int64:
            raise TypeError("device groupby needs an int64 key column")
        if self.flags & _GB_ARG:
            if any(v is None or v.dtype not in (np.float64, np.int64) for v in vals):
                raise TypeError("device groupby.idxmax / idxmin take float64 and int64 value columns")
            mask = sum(1 << j for j, v in enumerate(vals) if v.dtype == np.int64)
            ptrs = _lib.ptr_array([v.ptr for v in vals])
            with _timed("gb_accumulate_arg"):
                _lib.check(self.lib.mb200_gb_accumulate_arg(self.handle, keys.ptr, ptrs, mask, len(keys),
                                                            current_stream()))  # fmt: skip
            return
        for v in vals:
            if v is None and self.flags & _GB_POS:
                continue
            if v is None or v.dtype != np.float64:
                raise TypeError("device groupby aggregates float64 value columns")
        ptrs = _lib.ptr_array([v.ptr if v is not None else None for v in vals])
        with _timed("gb_accumulate"):
            _lib.check(self.lib.mb200_gb_accumulate(self.handle, keys.ptr, ptrs, len(keys), current_stream()))

    def accumulate_m2(self, keys: DeviceColumn, vals: Sequence[DeviceColumn], cnts=None, m2s=None):
        """Pass 2 of a var / std table (mb200_gb_accumulate_m2), after every pass-1 call: add each value's squared
        deviation from its group's mean into the table's M2s.  Raw float64 rows ``vals``, or with ``cnts`` / ``m2s`` the
        emitted sums, counts and M2s of other var / std tables.  The table takes no pass-1 rows afterwards."""
        if any(v.dtype != np.float64 for v in vals):
            raise TypeError("device groupby.var / std aggregate float64 value columns")
        ptrs = lambda cols: _lib.ptr_array([c.ptr for c in cols]) if cols is not None else None  # noqa: E731
        with _timed("gb_accumulate_m2"):
            _lib.check(self.lib.mb200_gb_accumulate_m2(self.handle, keys.ptr, ptrs(vals), ptrs(cnts), ptrs(m2s), len(keys),
                                                       current_stream()))  # fmt: skip

    def reserve_distinct(self, capacity: int):
        """Give a nunique table a distinct set of ``capacity`` (a power of two) 16-byte slots, or clear the one it has
        (mb200_gb_reserve_distinct)."""
        _lib.check(self.lib.mb200_gb_reserve_distinct(self.handle, int(capacity), current_stream()))

    def accumulate_distinct(self, keys: DeviceColumn, vals=None, dropna: bool = True, col_ids=None, images=None):
        """Pass 2 of a nunique table (mb200_gb_accumulate_distinct), after every pass-1 call: raw float64 / int64 rows
        ``vals`` (NaN skipped under ``dropna``), or the ``(col_ids, images)`` rows of other tables' ``emit_distinct``.
        Every (group, column, value) not in the set yet adds 1 to the group's count of that column."""
        if col_ids is None:
            if any(v.dtype not in (np.float64, np.int64) for v in vals):
                raise TypeError("device groupby.nunique takes float64 and int64 value columns (bool widened to int64)")
            mask = sum(1 << j for j, v in enumerate(vals) if v.dtype == np.int64)
            ptrs = _lib.ptr_array([v.ptr for v in vals]) if vals else None
            args = (ptrs, mask, 1 if dropna else 0, None, None)
        else:
            args = (None, 0, 1 if dropna else 0, col_ids.ptr, images.ptr)
        with _timed("gb_accumulate_distinct"):
            _lib.check(self.lib.mb200_gb_accumulate_distinct(self.handle, keys.ptr, *args, len(keys), current_stream()))

    def emit_distinct(self, ngroups: int, capacity: int):
        """The distinct set as ``(keys, col_ids, images, count_dev)`` rows for another nunique table's partial pass 2:
        one ``(key, -1, 0)`` row per group, then one row per entry, valid up to ``count_dev[0]`` (device int64[2]
        ``{rows, overflow}``; mb200_gb_emit_distinct)."""
        t = torch_mod()
        keys, cols, imgs = (DeviceColumn.empty(capacity, np.int64) for _ in range(3))
        count = t.empty(2, dtype=t.int64, device=current_device())
        scratch = _scratch(self.lib.mb200_gb_emit_scratch_bytes(ngroups), "gb_emit")
        _lib.check(self.lib.mb200_gb_emit_distinct(self.handle, int(ngroups), int(capacity), keys.ptr, cols.ptr, imgs.ptr,
                                                   scratch.data_ptr(), count.data_ptr(), current_stream()))  # fmt: skip
        return keys, cols, imgs, count

    def merge_partial(self, keys: DeviceColumn, sums, cnts=None, sizes: Optional[DeviceColumn] = None):
        ps = _lib.ptr_array([v.ptr for v in sums]) if sums else None
        pc = _lib.ptr_array([v.ptr for v in cnts]) if cnts else None
        _lib.check(
            self.lib.mb200_gb_merge_partial(self.handle, keys.ptr, ps, pc, sizes.ptr if sizes is not None else None,
                                            len(keys), current_stream())
        )  # fmt: skip

    def ngroups(self):
        ng = C.c_int64()
        ov = C.c_int()
        _lib.check(self.lib.mb200_gb_ngroups(self.handle, C.byref(ng), C.byref(ov), current_stream()))
        return int(ng.value), bool(ov.value)

    def _outputs(self, rows: int):
        """Empty (keys, sums, cnts, sizes) columns of ``rows`` rows for what this table emits."""
        acc_dtype = np.int64 if self.flags & _GB_POS else np.float64  # first / last / idxmin / idxmax emit row positions
        nsums = 2 * self.nvals if self.flags & _lib.GB_VAR else self.nvals  # var / std: the sums, then the M2s
        sums = [DeviceColumn.empty(rows, acc_dtype) for _ in range(nsums)] if self.flags & _GB_ACC else None
        cnts = [DeviceColumn.empty(rows, np.int64) for _ in range(self.nvals)] if self.flags & _GB_CNT & ~_GB_ARG else None
        sizes = DeviceColumn.empty(rows, np.int64) if self.flags & _lib.GB_SIZE else None
        return DeviceColumn.empty(rows, np.int64), sums, cnts, sizes

    def emit(self, ngroups: int, sort: bool = True):
        keys, sums, cnts, sizes = self._outputs(ngroups)
        scratch = _scratch(self.lib.mb200_gb_emit_scratch_bytes(ngroups), "gb_emit")
        _lib.check(
            self.lib.mb200_gb_emit(
                self.handle, ngroups, 1 if sort else 0, keys.ptr,
                _lib.ptr_array([c.ptr for c in sums]) if sums else None,
                _lib.ptr_array([c.ptr for c in cnts]) if cnts else None,
                sizes.ptr if sizes is not None else None, scratch.data_ptr(), current_stream(),
            )
        )  # fmt: skip
        return keys, sums, cnts, sizes

    def emit_async(self):
        """Dense tables: emit WITHOUT asking the device how many groups there are -- the outputs have room for every
        key of the table's range, the count is left in a device int64[2] ``{groups, overflow}``
        (``mb200_gb_emit_dense_async``; ``refuse_dense_overflow`` checks it once read).  Returns
        ``(keys, sums, cnts, sizes, count_dev)``; the columns are valid up to ``count_dev[0]``."""
        t = torch_mod()
        cap = self.capacity
        keys, sums, cnts, sizes = self._outputs(cap)
        count = t.empty(2, dtype=t.int64, device=current_device())
        scratch = _scratch(self.lib.mb200_gb_emit_scratch_bytes(cap), "gb_emit")
        _lib.check(
            self.lib.mb200_gb_emit_dense_async(
                self.handle, cap, keys.ptr,
                _lib.ptr_array([c.ptr for c in sums]) if sums else None,
                _lib.ptr_array([c.ptr for c in cnts]) if cnts else None,
                sizes.ptr if sizes is not None else None, scratch.data_ptr(), count.data_ptr(), current_stream(),
            )
        )  # fmt: skip
        return keys, sums, cnts, sizes, count

    def close(self):
        if self.handle:
            self.lib.mb200_gb_destroy(self.handle, current_stream())
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# The table driver works through the table's library calls only (accumulate / merge_partial / accumulate_m2 / ngroups /
# emit), so that whatever stands in for a table needs nothing else.
def fill_table(table, items, partial: bool = False):
    """Aggregate every input into ``table``: raw ``(keys, vals)`` rows (``accumulate``), or with ``partial`` the
    emitted ``(keys, sums, cnts, sizes)`` of other tables (``merge_partial``).  A var / std table's partial ``sums``
    hold the sums, then the M2s, as its emit does; once every input has set the group means (pass 1), every input
    goes through ``accumulate_m2`` (pass 2).  Returns the table."""
    var = table.flags & _lib.GB_VAR
    for item in items:
        if partial and var:
            W = len(item[2])
            table.merge_partial(item[0], item[1][:W], item[2], *item[3:])
        elif partial:
            table.merge_partial(*item)
        else:
            table.accumulate(item[0], item[1])
    if var:
        for item in items:
            if partial:
                W = len(item[2])
                table.accumulate_m2(item[0], item[1][:W], item[2], item[1][W:])
            else:
                table.accumulate_m2(item[0], item[1])
    return table


def emit_counted(table, sort: bool = True):
    """Count the groups of ``table`` (one host round trip) and emit them: ``(keys, sums, cnts, sizes)``, or None when
    a hashed table overflowed (recreate it larger).  A dense table that saw a key outside its range is refused."""
    ng, overflow = table.ngroups()
    if overflow and table.kbase is None:
        return None
    refuse_dense_overflow((ng, overflow))
    return table.emit(ng, sort=sort)


DENSE_TABLE_MAX_BYTES = 8 << 30


SKEW_THRESHOLD = 0.05  # share of sampled keys that met their own value among 32 keys (uniform over G keys: ~31/G)


def keys_are_skewed(sampled: int, duplicated: int) -> bool:
    """A heavy hitter (a key with >= ~5 % of the rows) shows up as most sampled keys being duplicates; uniform
    keys over G values give ~496/G (the shared-memory table takes the small-G cases before this matters)."""
    return sampled >= 1024 and duplicated > SKEW_THRESHOLD * sampled


def key_range_device(key_cols: Sequence[DeviceColumn]):
    """Device tensor [min, max, sampled, duplicated] over int64 key columns (mb200_key_range;
    {INT64_MAX, INT64_MIN, 0, 0} when there are no rows)."""
    lib = _lib.load()
    t = torch_mod()
    mm = t.empty(4, dtype=t.int64, device=current_device())
    if not key_cols:
        _lib.check(lib.mb200_key_range(None, 0, mm.data_ptr(), 1, current_stream()))
    for i, k in enumerate(key_cols):
        if k.dtype != np.int64:
            raise TypeError("device groupby needs an int64 key column")
        _lib.check(lib.mb200_key_range(k.ptr, len(k), mm.data_ptr(), 1 if i == 0 else 0, current_stream()))
    return mm


_I64_MAX, _I64_MIN = (1 << 63) - 1, -(1 << 63)
key_stats_passes = 0  # how many columns had to be scanned because nothing had left their statistics behind


def key_stats(key_cols: Sequence[DeviceColumn]):
    """Host ``(min, max, sampled, duplicated)`` over int64 key columns, from the columns' cached ``KeyStats``.
    Columns without statistics are scanned once (``mb200_key_range``) and remember the result; all pending device
    quadruples are read back in ONE D2H.  Steady state (statistics already on the host): no launch, no sync."""
    global key_stats_passes
    t = torch_mod()
    for k in key_cols:
        if k.dtype != np.int64:
            raise TypeError("device groupby needs an int64 key column")
        if k.stats is None:
            if len(k):
                key_stats_passes += 1
                k.stats = KeyStats(dev=key_range_device([k]))
            else:
                k.stats = KeyStats(host=(_I64_MAX, _I64_MIN, 0, 0))
    pending = [k.stats for k in key_cols if k.stats.pending() is not None]
    if pending:
        for st, vals in zip(pending, t.stack([st.pending() for st in pending]).tolist()):
            st.resolve(vals)
    lo, hi, sampled, dup = _I64_MAX, _I64_MIN, 0, 0
    for k in key_cols:
        a, b, s_, d_ = k.stats.host()
        lo, hi, sampled, dup = min(lo, a), max(hi, b), sampled + s_, dup + d_
    return lo, hi, sampled, dup


def key_range(key_cols: Sequence[DeviceColumn]):
    """(min, max) over int64 key columns -- one streaming pass, one 16-byte D2H.  None when empty."""
    lo, hi = key_stats(key_cols)[:2]
    return None if lo > hi else (lo, hi)


def dense_range_ok(lo: int, hi: int, cap: int, total_rows: int, nvals: int, flags: int) -> bool:
    """Dense tables pay range-proportional zero-fill and emit scan; their random footprint is only the
    touched groups.  Take them when the range is within 4x the expected group count (or half the
    rows) and the arrays stay under DENSE_TABLE_MAX_BYTES."""
    rng = hi - lo + 1
    if rng > (1 << 29) or rng > max(4 * cap, total_rows // 2, 1 << 16):
        return False
    arrays = (1 if flags & _GB_ACC else 0) + (1 if flags & _GB_CNT else 0) + (1 if flags & _lib.GB_VAR else 0)
    return rng * (value_stride(nvals) * 8 * arrays + 9) <= DENSE_TABLE_MAX_BYTES


def _job_key_range(key_cols: Sequence[DeviceColumn], lo: int, hi: int, rows: int):
    """Job-wide ``(min, max, rows)`` of key columns whose rows are sharded over the ranks, from this rank's.  Every
    rank must size its table alike, so the ranks agree ONCE per set of key columns (one small all_gather + one D2H)
    and the answer is remembered on the first of them -- columns are immutable and so is the job."""
    from . import dist

    if not dist.is_distributed():
        return lo, hi, rows
    sig = (dist.world_size(), tuple(id(k.data) for k in key_cols))
    anchor = key_cols[0].stats
    if anchor.job is None or anchor.job[0] != sig:
        t = torch_mod()
        trip = dist.all_gather_small(t.tensor([lo, hi, rows], dtype=t.int64, device=current_device()))
        anchor.job = (sig, (min(r[0] for r in trip), max(r[1] for r in trip), sum(r[2] for r in trip)))
    return anchor.job[1]


class TablePlan(NamedTuple):
    """The group table a groupby fills (``plan_table``)."""

    nvals: int
    flags: int
    dense: Optional[tuple]  # (first key, last key) of a dense table; None: a hash table
    capacity: int  # groups a hash table starts with
    rows: int  # rows to aggregate: a hash table never needs more groups than that
    skewed: bool  # accumulate with the hot-group cache
    chunk: int = 0  # job-wide dense table over several ranks: keys per rank (the range is padded to ranks * chunk)

    def create(self, capacity: Optional[int] = None) -> GroupTable:
        if self.dense is not None:
            table = GroupTable.dense(self.dense[0], self.dense[1], self.nvals, self.flags)
        else:
            table = GroupTable(self.capacity if capacity is None else capacity, self.nvals, self.flags)
        table.hint_skew(self.skewed)
        return table


def plan_table(key_cols: Sequence[DeviceColumn], nvals: int, flags: int, capacity_hint: int, partial: bool = False,
               job_wide: bool = False) -> Optional[TablePlan]:
    """Dense or hashed: a dense (direct-addressed) table over the keys' range when ``GroupbyDenseKeys`` is on and
    ``dense_range_ok`` accepts the range for ``max(1024, min(capacity_hint, rows))`` expected groups, else a hash
    table of that many groups.  The hot-group cache is hinted from the keys' sample, except for partial tables.

    ``job_wide``: the key columns are this rank's part of a job that fills ONE dense table per rank and merges them
    across ranks.  Range and row count are then the job's (``_job_key_range``), the table spans the range padded to
    one equal chunk per rank, and the answer is None when no dense table fits."""
    from .config import GroupbyDenseKeys

    dense_keys = GroupbyDenseKeys.get()
    if job_wide and not dense_keys:
        return None
    lo, hi, sampled, dup = key_stats(key_cols)  # column metadata: no pass over the keys, no sync, once known
    rows = sum(len(k) for k in key_cols)
    if job_wide:
        lo, hi, rows = _job_key_range(key_cols, lo, hi, rows)  # `sampled` / `dup` stay local, like the cache
    cap = max(1024, min(int(capacity_hint), rows))
    dense = (lo, hi) if dense_keys and lo <= hi and dense_range_ok(lo, hi, cap, rows, nvals, flags) else None
    chunk = 0
    if job_wide:
        from . import dist

        if dense is None:
            return None
        if dist.is_distributed() and dist.world_size() > 1:
            chunk = dist.dense_chunk(hi - lo + 1, dist.world_size())
            dense = (lo, lo + dist.world_size() * chunk - 1)
    return TablePlan(nvals, flags, dense, cap, rows, not partial and keys_are_skewed(sampled, dup), chunk)


def hash_aggregate(key_cols_vals, flags: int, capacity_hint: int, partial: bool = False, sort: bool = True):
    """Aggregate a list of (keys, vals[, cnts, sizes]) inputs into one table and emit it: a dense
    (direct-addressed) table when the key range allows, else the hash table, grown when it
    overflows.  Returns (keys, sums, cnts, sizes) device columns.  A var / std table's sums are the sums, then the M2s
    (2 x nvals columns), in its partial inputs and in its result alike."""
    halves = 2 if partial and flags & _lib.GB_VAR else 1
    nvals = (len(key_cols_vals[0][1]) if key_cols_vals[0][1] else 0) // halves
    if nvals > _lib.MAX_COLS:
        # a table holds at most MAX_COLS value columns: aggregate them MAX_COLS at a time.  Every pass sees the same
        # keys, so every table holds the same groups; emitted in ascending key order, their rows line up.  Lists of
        # several nvals-long runs (a var / std table's sums, then M2s) are cut and joined run by run.
        def cut(cols, k):
            if not cols:
                return cols
            return [c for h in range(0, len(cols), nvals) for c in cols[h + k : h + min(k + _lib.MAX_COLS, nvals)]]

        def join(lists):
            if lists[0] is None:
                return None
            runs = len(lists[0]) // min(_lib.MAX_COLS, nvals)
            return [c for r in range(runs) for cs in lists for c in cs[r * (len(cs) // runs) : (r + 1) * (len(cs) // runs)]]

        parts = []
        for k in range(0, nvals, _lib.MAX_COLS):
            items = [(it[0], cut(it[1], k)) + ((cut(it[2], k),) + tuple(it[3:]) if len(it) > 2 else ()) for it in key_cols_vals]
            parts.append(hash_aggregate(items, flags, capacity_hint, partial=partial, sort=True))
        return parts[0][0], join([p[1] for p in parts]), join([p[2] for p in parts]), parts[0][3]
    plan = plan_table([item[0] for item in key_cols_vals], nvals, flags, capacity_hint, partial=partial)
    cap = plan.capacity
    while True:
        table = plan.create(cap)
        try:
            out = emit_counted(fill_table(table, key_cols_vals, partial), sort=sort)
        finally:
            table.close()
        if out is not None:
            return out
        if cap >= max(plan.rows, 1024):
            raise _lib.B200Error("group table overflow even with capacity == number of rows")
        cap = min(max(cap * 4, 1024), max(plan.rows, 1024))


# ------------------------------------------------------------------ broadcast hash join
class JoinTable:
    def __init__(self, dim_keys: DeviceColumn):
        if dim_keys.dtype != np.int64:
            raise TypeError("device merge needs an int64 key column")
        self.lib = _lib.load()
        self.handle = C.c_void_p()
        self.keys = dim_keys
        _lib.check(self.lib.mb200_join_build(C.byref(self.handle), dim_keys.ptr, len(dim_keys), current_stream()))

    def is_unique(self) -> bool:
        u = C.c_int()
        _lib.check(self.lib.mb200_join_is_unique(self.handle, C.byref(u), current_stream()))
        return bool(u.value)

    def probe(self, fact_keys: DeviceColumn):
        t = torch_mod()
        idx = DeviceColumn.empty(len(fact_keys), np.int64)
        nm = t.zeros(1, dtype=t.int64, device=current_device())
        _lib.check(self.lib.mb200_join_probe(self.handle, fact_keys.ptr, len(fact_keys), idx.ptr, nm.data_ptr(),
                                             current_stream()))  # fmt: skip
        return idx, nm

    def probe_gather(self, fact_keys: DeviceColumn, dim_cols: Sequence[DeviceColumn]):
        """Left-join payload: float64 out (NaN on miss); int64 payload is promoted like pandas does
        when a left join has misses -- decided by the caller from the returned match count."""
        t = torch_mod()
        n = len(fact_keys)
        nm = t.zeros(1, dtype=t.int64, device=current_device())
        outs: list = [None] * len(dim_cols)
        groups = {}
        for j, c in enumerate(dim_cols):
            groups.setdefault(c.code, []).append(j)
        # the match count is only needed to decide whether int64 payload has to be promoted (misses -> NaN), so
        # only the first int64 launch counts; float64-only payload lets the library probe its key-ordered payload
        # copies (one random read per row).  The table caches those copies per source column, by pointer: keep
        # every source column alive as long as the table is.  Neither side evicts: a table is meant to be probed with
        # the payload columns of its own dim frame.
        if any(code == _lib.U8 for code in groups):
            raise TypeError("bool payload columns are not on the device merge path")
        counted = _lib.I64 not in groups
        refs = self.__dict__.setdefault("_payload_refs", {})
        for code, idxs in groups.items():
            for k in range(0, len(idxs), _lib.MAX_COLS):
                sel = idxs[k : k + _lib.MAX_COLS]
                refs.update((dim_cols[j].ptr, dim_cols[j]) for j in sel)
                sel_out = [DeviceColumn.empty(n, dim_cols[j].dtype) for j in sel]
                count = not counted and code == _lib.I64
                counted = counted or count
                with _timed("join_probe_gather"):
                    _lib.check(
                        self.lib.mb200_join_probe_gather(
                            self.handle, fact_keys.ptr, n, len(sel), _lib.ptr_array([dim_cols[j].ptr for j in sel]),
                            code, _lib.ptr_array([c.ptr for c in sel_out]), nm.data_ptr() if count else None,
                            current_stream(),
                        )
                    )  # fmt: skip
                for j, c in zip(sel, sel_out):
                    outs[j] = c
        return outs, nm

    def close(self):
        if self.handle:
            self.lib.mb200_join_destroy(self.handle, current_stream())
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def expand_matches(fact_keys: DeviceColumn, dim_keys: DeviceColumn, keep_misses: bool):
    """Row pairs of a merge whose broadcast side has DUPLICATE keys (many-to-many): ``(left_rows, right_rows,
    misses)`` -- int64 device columns of equal length, left order preserved, a left row's matches in their order of
    appearance on the right, ``right_rows`` = -1 where a left row found nothing (kept only when ``keep_misses``, the
    left join); ``misses`` = number of such left rows (host int).  Sort + run heads + a many-to-one probe of the
    distinct keys + prefix sum + expansion, all on the device (csrc/expand.cu)."""
    lib = _lib.load()
    t = torch_mod()
    st = current_stream()
    nd, nf = len(dim_keys), len(fact_keys)
    ks = map_columns("copy", [dim_keys])[0] if nd else dim_keys
    order = iota(0, nd)
    if nd:
        sort_pairs(ks, order)
    heads = DeviceColumn.empty(nd, np.int64)
    _lib.check(lib.mb200_run_heads(ks.ptr, nd, heads.ptr, st))
    starts, nuniq = compact_hits(heads)
    uniq = take_columns([ks], starts)[0] if nuniq else DeviceColumn.empty(0, np.int64)
    table = JoinTable(uniq)
    try:
        u, nmatch = table.probe(fact_keys)
    finally:
        table.close()
    cnt, first, offsets = (DeviceColumn.empty(nf, np.int64) for _ in range(3))
    _lib.check(lib.mb200_expand_counts(u.ptr, nf, starts.ptr, nuniq, nd, 1 if keep_misses else 0, cnt.ptr, first.ptr, st))
    total = t.zeros(1, dtype=t.int64, device=current_device())
    sb = lib.mb200_scan_scratch_bytes(nf)
    scratch = _scratch(sb, "scan")
    _lib.check(lib.mb200_scan_i64(cnt.ptr, nf, offsets.ptr, total.data_ptr(), scratch.data_ptr(), sb, st))
    n_out, n_hit = (int(v) for v in t.cat([total, nmatch.reshape(1)]).tolist())  # one D2H sizes the result
    left_rows, right_rows = DeviceColumn.empty(n_out, np.int64), DeviceColumn.empty(n_out, np.int64)
    _lib.check(lib.mb200_expand_rows(offsets.ptr, cnt.ptr, first.ptr, order.ptr, nf, left_rows.ptr, right_rows.ptr, st))
    return left_rows, right_rows, nf - n_hit


def take_columns(cols: Sequence[DeviceColumn], idx: DeviceColumn) -> List[DeviceColumn]:
    lib = _lib.load()
    n = len(idx)
    outs: list = [None] * len(cols)
    groups = {}
    for j, c in enumerate(cols):
        groups.setdefault(c.code, []).append(j)
    for code, idxs in groups.items():
        for k in range(0, len(idxs), _lib.MAX_COLS):
            sel = idxs[k : k + _lib.MAX_COLS]
            o = [DeviceColumn.empty(n, cols[j].dtype) for j in sel]
            _lib.check(lib.mb200_take(code, len(sel), _lib.ptr_array([cols[j].ptr for j in sel]), idx.ptr, n,
                                      _lib.ptr_array([c.ptr for c in o]), current_stream()))  # fmt: skip
            for j, c in zip(sel, o):
                outs[j] = c
    return outs


def compact_hits(idx: DeviceColumn):
    """Positions (ascending) of idx >= 0 and their count (host int; synchronises)."""
    lib = _lib.load()
    t = torch_mod()
    n = len(idx)
    pos = DeviceColumn.empty(n, np.int64)
    cnt = t.zeros(1, dtype=t.int64, device=current_device())
    nb = (n + 2047) // 2048
    sb = nb * 12 + 256
    scratch = _scratch(sb, "compact")
    _lib.check(lib.mb200_compact_hits(idx.ptr, n, pos.ptr, cnt.data_ptr(), scratch.data_ptr(), sb, current_stream()))
    k = int(cnt.item())
    return pos.slice(0, k), k


# ------------------------------------------------------------------ synthetic columns
def gen_f64(nrows: int, seed: int, col: int, row_offset: int = 0, nan_per_64k: int = 0) -> DeviceColumn:
    lib = _lib.load()
    c = DeviceColumn.empty(nrows, np.float64)
    _lib.check(lib.mb200_gen_f64(c.ptr, nrows, seed, col, row_offset, nan_per_64k, current_stream()))
    return c


def gen_i64(nrows: int, seed: int, col: int, modulus: int, row_offset: int = 0, skew: bool = False) -> DeviceColumn:
    """Synthetic int64 column; the generator kernel also leaves the column's key statistics behind (KeyStats)."""
    lib = _lib.load()
    t = torch_mod()
    c = DeviceColumn.empty(nrows, np.int64)
    stats = t.empty(4, dtype=t.int64, device=current_device())
    fn = lib.mb200_gen_i64_skew if skew else lib.mb200_gen_i64
    _lib.check(fn(c.ptr, nrows, seed, col, row_offset, modulus, stats.data_ptr(), current_stream()))
    c.stats = KeyStats(dev=stats)
    return c


def concat_columns(pieces: Sequence[DeviceColumn]) -> DeviceColumn:
    """Row-wise concatenation of column pieces of one dtype into a fresh buffer: ONE ``mb200_concat`` launch (per 64
    pieces) instead of a framework concatenation."""
    pieces = [p for p in pieces]
    if len(pieces) == 1:
        return pieces[0]
    lib = _lib.load()
    dtype = pieces[0].dtype
    if any(p.dtype != dtype for p in pieces):
        raise TypeError("concat_columns needs pieces of one dtype")
    out = DeviceColumn.empty(sum(len(p) for p in pieces), dtype)
    pieces = [p for p in pieces if len(p)]  # empty pieces have no buffer (and nothing to copy)
    if not pieces:
        return out
    item = 1 if dtype == np.bool_ else 8
    sizes = (C.c_int64 * len(pieces))(*[len(p) * item for p in pieces])
    _lib.check(lib.mb200_concat(len(pieces), _lib.ptr_array([p.ptr for p in pieces]), sizes, out.ptr, current_stream()))
    return out


class CumState:
    """What ``cum_partials`` leaves for ``cum_apply``: per dtype group the scanned tile aggregates (scratch) and the
    column totals (device, one per column of the group)."""

    __slots__ = ("op", "n", "groups")

    def __init__(self, op, n):
        self.op, self.n, self.groups = op, n, []  # (code, column positions, scratch tensor, totals tensor)


def cum_partials(op: str, cols: Sequence[DeviceColumn]) -> CumState:
    """Phase 1 of a cumulative function (``mb200_cum_partials``): per-tile aggregates of every column, scanned per
    column; ``state.groups[k][3]`` holds the column totals -- what ranks / row partitions exchange."""
    lib = _lib.load()
    t = torch_mod()
    n = len(cols[0]) if cols else 0
    st = CumState(op, n)
    by_code = {}
    for j, c in enumerate(cols):
        if c.code == _lib.U8 or (op == "ffill" and c.code != _lib.F64):
            raise TypeError(f"cumulative {op} over {c.dtype} columns is not on the B200 path")
        by_code.setdefault(c.code, []).append(j)
    for code, idxs in by_code.items():
        nbytes = lib.mb200_cum_scratch_bytes(len(idxs), n)
        scratch = t.empty(nbytes, dtype=t.uint8, device=current_device())
        totals = t.empty(len(idxs), dtype=t.float64 if code == _lib.F64 else t.int64, device=current_device())
        with _timed("cum_partials"):
            _lib.check(lib.mb200_cum_partials(_lib.CUM[op], code, len(idxs), _lib.ptr_array([cols[j].ptr for j in idxs]), n,
                                              scratch.data_ptr(), nbytes, totals.data_ptr(), current_stream()))  # fmt: skip
        st.groups.append((code, idxs, scratch, totals))
    return st


def cum_carry(state: CumState, gathered: Sequence, rank: int) -> list:
    """Carry of this rank per dtype group from the all-gathered totals (``[nranks * ncols]`` device vectors, rank-major):
    the totals of ranks ``0 .. rank-1`` combined in rank order (``mb200_cum_carry``)."""
    lib = _lib.load()
    t = torch_mod()
    out = []
    for (code, idxs, _s, totals), g in zip(state.groups, gathered):
        carry = t.empty_like(totals)
        _lib.check(lib.mb200_cum_carry(_lib.CUM[state.op], code, len(idxs), g.data_ptr(), int(rank), carry.data_ptr(),
                                       current_stream()))  # fmt: skip
        out.append(carry)
    return out


def cum_apply(state: CumState, cols: Sequence[DeviceColumn], carries=None) -> list:
    """Phase 2 (``mb200_cum_apply``): ``out[j][i] = carry (+) rows 0 .. i`` of column j, into fresh columns."""
    lib = _lib.load()
    outs: list = [None] * len(cols)
    for k, (code, idxs, scratch, _totals) in enumerate(state.groups):
        fresh = [DeviceColumn.empty(state.n, cols[j].dtype) for j in idxs]
        carry = carries[k] if carries is not None else None
        with _timed("cum_apply"):
            _lib.check(lib.mb200_cum_apply(_lib.CUM[state.op], code, len(idxs), _lib.ptr_array([cols[j].ptr for j in idxs]),
                                           _lib.ptr_array([c.ptr for c in fresh]), state.n, scratch.data_ptr(),
                                           carry.data_ptr() if carry is not None else None, current_stream()))  # fmt: skip
        for j, c in zip(idxs, fresh):
            outs[j] = c
    return outs


def run_starts(sorted_keys: DeviceColumn):
    """Runs of equal values in a SORTED int64 column: ``(start positions, value of each run)`` as small host arrays
    (``mb200_run_heads`` + compaction + gather; meant for few runs -- bin ids, not row keys)."""
    lib = _lib.load()
    n = len(sorted_keys)
    if n == 0:
        return np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64)
    heads = DeviceColumn.empty(n, np.int64)
    _lib.check(lib.mb200_run_heads(sorted_keys.ptr, n, heads.ptr, current_stream()))
    starts, nruns = compact_hits(heads)
    vals = take_columns([sorted_keys], starts)[0]
    return starts.to_numpy(), vals.to_numpy()


def digitize(values: DeviceColumn, pivots) -> DeviceColumn:
    """``np.digitize(values, pivots)`` on the device: bin id = number of (ascending int64) pivots <= value."""
    lib = _lib.load()
    t = torch_mod()
    out = DeviceColumn.empty(len(values), np.int64)
    piv = t.as_tensor(list(pivots), dtype=t.int64).to(current_device()) if len(pivots) else None
    _lib.check(lib.mb200_digitize_i64(values.ptr, len(values), piv.data_ptr() if piv is not None else None, len(pivots),
                                      out.ptr, current_stream()))  # fmt: skip
    return out


def iota(start: int, nrows: int) -> DeviceColumn:
    """int64 column ``start, start + 1, ...``: the labels of a RangeIndex block as device data."""
    lib = _lib.load()
    c = DeviceColumn.empty(nrows, np.int64)
    _lib.check(lib.mb200_iota_i64(c.ptr, nrows, int(start), current_stream()))
    return c


def full_column(nrows: int, dtype, value) -> DeviceColumn:
    """Constant float64 / int64 column (NaN columns that re-indexing adds)."""
    lib = _lib.load()
    dtype = np.dtype(dtype)
    if dtype not in (np.dtype("float64"), np.dtype("int64")):
        raise TypeError("constant device columns are float64 or int64")
    c = DeviceColumn.empty(nrows, dtype)
    bits = f64_bits(value) if dtype == np.float64 else i64_bits(value)
    _lib.check(lib.mb200_fill_u64(c.ptr, nrows, bits, current_stream()))
    return c


def sort_pairs(keys: DeviceColumn, payload: DeviceColumn):
    """In-place stable sort of (keys, payload) by key."""
    lib = _lib.load()
    n = len(keys)
    sb = lib.mb200_sort_scratch_bytes(n)
    scratch = _scratch(sb, "sort")
    _lib.check(lib.mb200_sort_pairs_i64(keys.ptr, payload.ptr, n, scratch.data_ptr(), sb, current_stream()))
