"""Tagged device functors: what the operator templates hand to the partitions.

The reference's templates wrap *pandas methods* in closures (``lambda x: function(x, *args,
**kwargs)``, alg/map.py:64-66, alg/tree_reduce.py:76-77, alg/binary.py:399-401, 422) and the
partition calls them on a ``pandas.DataFrame``.  The B200 query compiler registers these
functors through the same templates instead (SURVEY.md §8b-4): each is a callable with the
pandas method's calling convention that takes ``DeviceBlock`` operands and launches
libmodin_b200 kernels.  They carry an ``op`` tag so that the partition call-queue can fuse
adjacent ones (``x*b`` then ``+c`` -> one AFFINE sweep; ``a*b`` then ``+c`` -> one FMA3 sweep).

Anything a functor cannot do on the device raises ``NotImplementedError`` -- there is no
silent pandas fallback on this path.
"""

from __future__ import annotations

import numbers
from typing import NamedTuple, Optional

import numpy as np
import pandas

from . import _lib, ops
from .block import DeviceBlock, DeviceColumn
from .config import ReduceVariant

MODIN_UNNAMED_SERIES_LABEL = "__reduced__"  # modin/utils.py:98

_BINARY_TO_SCALAR = {
    "add": "add_s", "radd": "add_s", "sub": "sub_s", "rsub": "rsub_s", "mul": "mul_s", "rmul": "mul_s",
    "truediv": "div_s", "rtruediv": "rdiv_s", "eq": "eq_s", "ne": "ne_s", "lt": "lt_s", "le": "le_s",
    "gt": "gt_s", "ge": "ge_s",
}  # fmt: skip
_BINARY_TO_FRAME = {
    "add": "add", "radd": "add", "sub": "sub", "mul": "mul", "rmul": "mul", "truediv": "div",
    "eq": "eq", "ne": "ne", "lt": "lt", "le": "le", "gt": "gt", "ge": "ge",
}  # fmt: skip
_REFLECTED_FRAME = {"rsub": "sub", "rtruediv": "div"}


def _spans_ranks(block) -> bool:
    """True when ``block`` is this rank's part of a frame whose rows are sharded over several GPUs: the reduce phase
    of a template then has to finish with a collective.  The reference gathers every block of the axis into ONE task
    (axis_partition.py:445-452); here the other ranks hold the rest of the axis, so the reduce-phase functors issue
    the collective themselves -- also when Modin's own templates call them through an opaque lambda
    (``lambda y: reduce_function(y, *args, **kwargs)``, alg/tree_reduce.py:77-80)."""
    from . import dist

    return dist.is_distributed() and not getattr(block, "replicated", False)


class DevFn:
    """Base of all device functors."""

    op: str = ""
    fusable: bool = False

    def __call__(self, block, *args, **kwargs):  # pragma: no cover - interface
        raise NotImplementedError


def _is_scalar(x) -> bool:
    return isinstance(x, (numbers.Number, np.number, np.bool_)) and not isinstance(x, bool) or isinstance(x, bool)


def _check_block(x, who):
    if not isinstance(x, DeviceBlock):
        raise TypeError(f"{who} expects a DeviceBlock partition payload, got {type(x).__name__}")
    if x._pending is not None:
        x.nrows  # sized on the device: read the count back (and trim the buffers) before any kernel sees the block


class DevMap(DevFn):
    """Unary elementwise map: abs / neg / isna / notna (qc.py:2036, 2063-2106)."""

    def __init__(self, op: str):
        if op not in ("abs", "neg", "isna", "notna", "copy", "not"):
            raise ValueError(op)
        self.op = op

    def __call__(self, block, *args, **kwargs):
        _check_block(block, f"DevMap({self.op})")
        if self.op == "not" and any(c.dtype != np.bool_ for c in block.cols):
            raise NotImplementedError("~frame on the B200 path needs bool columns (bitwise integer NOT is not on it)")
        if not block.cols or block.nrows == 0:
            return self._empty(block)
        if self.op in ("isna", "notna"):
            # int64 columns hold no nulls: constant answer, computed by the compare kernel (x == x)
            cols = []
            for c in block.cols:
                if c.dtype == np.float64:
                    cols.extend(ops.map_columns(self.op, [c]))
                else:
                    cols.extend(ops.map_columns("ne" if self.op == "isna" else "eq", [c], [c]))
            return block.with_cols(cols)
        return block.with_cols(ops.map_columns(self.op, block.cols))

    def _empty(self, block):
        if self.op in ("isna", "notna"):
            return block.with_cols([DeviceColumn.empty(block.nrows, np.bool_) for _ in block.cols])
        return block


class DevRound(DevFn):
    """``df.round(decimals)`` -- ``Map.register(pandas.DataFrame.round)`` qc.py:2438; numpy.round semantics
    (``rint(x * 10**d) / 10**d``, half to even), integer columns unchanged for d >= 0."""

    op = "round"

    def __call__(self, block, *args, decimals=0, **kwargs):
        _check_block(block, "DevRound")
        if args:
            decimals = args[0]
        if not isinstance(decimals, numbers.Integral) or abs(int(decimals)) > 22:
            raise NotImplementedError("device round takes one integer `decimals` in [-22, 22]")
        d = int(decimals)
        if not block.cols or block.nrows == 0:
            return block
        out = list(block.cols)
        fidx = [j for j, c in enumerate(block.cols) if c.dtype == np.float64]
        if any(c.dtype == np.int64 for c in block.cols) and d < 0:
            raise NotImplementedError("round(decimals < 0) on int64 columns is not on the B200 path")
        if any(c.dtype == np.bool_ for c in block.cols):
            raise NotImplementedError("round on bool columns is not on the B200 path")
        if fidx:
            res = ops.map_columns("round_s", [block.cols[j] for j in fidx], s0=[10.0 ** abs(d)] * len(fidx),
                                  s1=[1.0 if d >= 0 else -1.0] * len(fidx))  # fmt: skip
            for j, r in zip(fidx, res):
                out[j] = r
        return block.with_cols(out)


class DevAstype(DevFn):
    """``df.astype(dtype)`` -- qc.py ``astype`` (a Map over ``pandas.DataFrame.astype``) for the widening casts the
    map kernels already carry: int64 / bool -> float64 (the ``x / 1`` division kernel, round to nearest even above
    2**53 exactly as numpy) and bool -> int64 (the widening copy).  A column already of the target dtype shares its
    buffer.  float64 -> int64 (pandas raises on NaN / inf, truncates otherwise) and anything -> bool have no kernel
    on this path and are refused."""

    op = "astype"

    @staticmethod
    def target(dtype) -> np.dtype:
        try:
            dt = np.dtype(pandas.api.types.pandas_dtype(dtype))
        except TypeError:
            raise NotImplementedError(f"astype({dtype!r}) is not on the B200 path") from None
        if dt not in (np.dtype("float64"), np.dtype("int64"), np.dtype("bool")):
            raise NotImplementedError(f"astype({dt}) is not on the B200 path (float64 / int64 / bool columns only)")
        return dt

    @classmethod
    def validate(cls, have: pandas.Series, col_dtypes) -> dict:
        """{label: dtype} for ``col_dtypes`` (one dtype for every column, or a mapping) after checking every cast
        against the current dtypes ``have`` -- called by the query compilers BEFORE anything is launched, so a
        refused cast cannot leave a half-converted frame.  An unknown label raises pandas' KeyError."""
        if not isinstance(col_dtypes, dict):
            col_dtypes = {label: col_dtypes for label in have.index}
        for label, dt in col_dtypes.items():
            if label not in have.index:
                raise KeyError("Only a column name can be used for the key in a dtype mappings argument. "
                               f"'{label}' not found in columns.")  # fmt: skip
            src, dst = np.dtype(have[label]), cls.target(dt)
            if src != dst and not (dst == np.float64 or (dst == np.int64 and src == np.bool_)):
                raise NotImplementedError(f"astype {src} -> {dst} is not on the B200 path")
        return dict(col_dtypes)

    def __call__(self, block, *args, col_dtypes=None, **kwargs):
        _check_block(block, "DevAstype")
        if args:
            col_dtypes = args[0]
        if not isinstance(col_dtypes, dict):
            raise TypeError("DevAstype takes a {column label: dtype} mapping")
        out = list(block.cols)
        for j, label in enumerate(block.columns):
            if label not in col_dtypes:
                continue
            src, dst = block.cols[j].dtype, self.target(col_dtypes[label])
            if src == dst:
                continue
            if not (dst == np.float64 or (dst == np.int64 and src == np.bool_)):
                raise NotImplementedError(f"astype {src} -> {dst} is not on the B200 path")
            if block.nrows == 0:  # nothing to launch, but the dtype still changes
                out[j] = DeviceColumn.empty(0, dst)
            elif dst == np.float64:
                out[j] = ops.cast_columns_f64([block.cols[j]])[0]
            elif dst == np.int64 and src == np.bool_:
                out[j] = ops.cast_columns_i64([block.cols[j]])[0]
            else:
                raise NotImplementedError(f"astype {src} -> {dst} is not on the B200 path")
        return block.with_cols(out)


class DevClip(DevFn):
    """``df.clip(lower, upper)`` with scalar bounds -- ``Map.register(pandas.DataFrame.clip)`` (qc.py clip);
    NaNs stay NaN, a missing bound is -inf / +inf."""

    op = "clip"

    def __call__(self, block, *args, lower=None, upper=None, axis=None, inplace=False, **kwargs):
        _check_block(block, "DevClip")
        if args:
            lower = args[0]
            upper = args[1] if len(args) > 1 else upper
        for b in (lower, upper):
            if b is not None and not isinstance(b, numbers.Real):
                raise NotImplementedError("device clip takes scalar bounds")
        if lower is not None and upper is not None and lower > upper:
            lower, upper = upper, lower  # pandas swaps crossed scalar bounds
        if not block.cols or block.nrows == 0 or (lower is None and upper is None):
            return block
        out = list(block.cols)
        for code, lo_def, hi_def in ((np.float64, -np.inf, np.inf), (np.int64, np.iinfo(np.int64).min, np.iinfo(np.int64).max)):
            idx = [j for j, c in enumerate(block.cols) if c.dtype == code]
            if not idx:
                continue
            lo = lo_def if lower is None or (code == np.float64 and lower != lower) else lower
            hi = hi_def if upper is None or (code == np.float64 and upper != upper) else upper
            if code == np.int64 and (float(lo) != int(lo) or float(hi) != int(hi)):
                raise NotImplementedError("clip of int64 columns with fractional bounds upcasts to float64 in pandas; "
                                          "not on the B200 path")  # fmt: skip
            conv = float if code == np.float64 else int
            res = ops.map_columns("clip_s", [block.cols[j] for j in idx], s0=[conv(lo)] * len(idx), s1=[conv(hi)] * len(idx))
            for j, r in zip(idx, res):
                out[j] = r
        if any(c.dtype == np.bool_ for c in block.cols):
            raise NotImplementedError("clip on bool columns is not on the B200 path")
        return block.with_cols(out)


class DevFillna(DevFn):
    """``df.fillna(value=scalar|dict)`` -- the Map branch of qc.fillna (qc.py:2710-2813)."""

    op = "fillna"

    def __call__(self, block, *args, value=None, method=None, axis=None, inplace=False, limit=None, **kwargs):
        _check_block(block, "DevFillna")
        if args:
            value = args[0]
        if method is not None or limit is not None:
            raise NotImplementedError("fillna(method=/limit=) is a Fold in the reference; not on the B200 path")
        if value is None:
            raise ValueError("Must specify a fill 'value' or 'method'.")
        if isinstance(value, dict) or isinstance(value, pandas.Series):
            lookup = dict(value)
        elif _is_scalar(value):
            lookup = None
        else:
            raise NotImplementedError("fillna with a frame value goes through broadcast_apply; use DevBinary('fillna')")
        out = []
        for label, c in zip(block.columns, block.cols):
            v = value if lookup is None else lookup.get(label)
            if v is None or c.dtype != np.float64 or block.nrows == 0:
                out.append(c)  # nothing to fill: share the buffer
            else:
                out.extend(ops.map_columns("fillna_s", [c], s0=[float(v)]))
        return block.with_cols(out)


class DevBinary(DevFn):
    """Binary operator against a scalar, a row vector (list / Series along axis=1) or another
    block -- the three shapes Binary.caller produces (alg/binary.py:334-458)."""

    fusable = True

    def __init__(self, op: str):
        if op not in _BINARY_TO_SCALAR and op not in _REFLECTED_FRAME and op != "fillna":
            raise ValueError(f"binary op {op!r} is not implemented on the B200 path")
        self.op = op

    # -- helpers -------------------------------------------------------------------------------
    @staticmethod
    def _promote(cols, scalar_is_float):
        """pandas type promotion for arithmetic: int64 (op) float -> float64."""
        if scalar_is_float and any(c.dtype == np.int64 for c in cols):
            return ops.cast_columns_f64(cols)
        return list(cols)

    def _scalar(self, block, scalars):
        """`scalars`: one python scalar per column."""
        kop = _BINARY_TO_SCALAR[self.op]
        is_pred = kop in _lib.PREDICATES
        any_float = any(isinstance(s, (float, np.floating)) for s in scalars)
        if is_pred:
            # an int64 column against a FLOAT scalar is compared in float64, as numpy / pandas do (the column is
            # converted, rounding included above 2**53); int against int stays an exact integer compare
            cols = [ops.cast_columns_f64([c])[0] if c.dtype == np.int64 and isinstance(s, (float, np.floating)) else c
                    for c, s in zip(block.cols, scalars)]  # fmt: skip
        else:
            cols = self._promote(block.cols, any_float)
        # group by dtype handled inside map_columns; scalars must match the column dtype
        svals = [float(s) if c.dtype == np.float64 else int(s) for c, s in zip(cols, scalars)]
        out = ops.map_columns(kop, cols, s0=svals)
        return block.with_cols(out)

    def _frame(self, left, right):
        if self.op == "fillna":
            kop, a, b = "fillna", left.cols, right.cols
        elif self.op in _REFLECTED_FRAME:
            kop, a, b = _REFLECTED_FRAME[self.op], right.cols, left.cols
        else:
            kop, a, b = _BINARY_TO_FRAME[self.op], left.cols, right.cols
        if left.nrows != right.nrows:
            raise ValueError("device binary op needs identically shaped, co-partitioned operands")
        if len(right.cols) == 1 and len(left.cols) != 1 and self.op not in _REFLECTED_FRAME:
            # frame (op) column vector: the broadcast_apply shape of Binary.caller (alg/binary.py:396-408,
            # `df.mul(series, axis=0)`): the single right column is paired with every left column
            b = [right.cols[0]] * len(left.cols)
            a = left.cols
        elif len(right.cols) == 1 and len(left.cols) != 1:
            a = [right.cols[0]] * len(left.cols)
            b = left.cols
        elif len(a) != len(b):
            raise ValueError("device binary op needs identically shaped, co-partitioned operands")
        elif not left.columns.equals(right.columns):
            raise NotImplementedError("binary op between blocks with different column labels (needs copartition)")
        if kop not in _lib.PREDICATES and kop != "div":
            mixed = any(x.dtype != y.dtype for x, y in zip(a, b))
            if mixed:
                a, b = ops.cast_columns_f64(a), ops.cast_columns_f64(b)
        return left.with_cols(ops.map_columns(kop, a, b))

    def _empty(self, block, other):
        """Zero rows: nothing to launch, but the result still has the dtypes the rules above give it (a comparison of
        an empty frame is an empty BOOL frame -- ``df[df.x > 100][df.y > 0]`` and ``(empty > 0).any()`` depend on it)."""
        f64, i64 = np.dtype("float64"), np.dtype("int64")
        ldt = [c.dtype for c in block.cols]
        if isinstance(other, DeviceBlock):
            kop = "fillna" if self.op == "fillna" else _REFLECTED_FRAME.get(self.op) or _BINARY_TO_FRAME[self.op]
            rdt = [c.dtype for c in other.cols]
            rdt = rdt * len(ldt) if len(rdt) == 1 else rdt
            if kop in _lib.PREDICATES:
                dts = [np.dtype("bool")] * len(ldt)
            elif kop == "div":
                dts = [f64] * len(ldt)
            elif kop != "fillna" and any(x != y for x, y in zip(ldt, rdt)):
                dts = [f64] * len(ldt)  # mixed int64 / float64 operands are all promoted
            else:
                dts = ldt
        else:
            scalars = list(other) if isinstance(other, (list, tuple, np.ndarray, pandas.Series)) else [other]
            kop = _BINARY_TO_SCALAR.get(self.op)
            if kop is None:  # frame-only ops ("fillna"): nothing to decide without the frame
                return block
            any_float = any(isinstance(s, (float, np.floating)) for s in scalars)
            if kop in _lib.PREDICATES:
                dts = [np.dtype("bool")] * len(ldt)
            elif kop in ("div_s", "rdiv_s"):
                dts = [f64] * len(ldt)
            else:
                dts = [f64 if (any_float and d == i64) else d for d in ldt]
        return block.with_cols([c if c.dtype == d else DeviceColumn.empty(0, d) for c, d in zip(block.cols, dts)])

    def __call__(self, block, other, *args, axis=None, level=None, fill_value=None, **kwargs):
        _check_block(block, f"DevBinary({self.op})")
        if level is not None or fill_value is not None:
            raise NotImplementedError("level= / fill_value= are not implemented on the B200 path")
        if not block.cols:
            return block
        if block.nrows == 0:
            return self._empty(block, other)
        if isinstance(other, DeviceBlock):
            return self._frame(block, other)
        if _is_scalar(other):
            return self._scalar(block, [other] * len(block.cols))
        if isinstance(other, pandas.Series):
            if axis in (0, "index"):
                raise NotImplementedError("column-vector broadcast (axis=0) is not on the B200 path")
            other = other.reindex(block.columns)
            if other.isna().any():
                raise NotImplementedError("row vector does not cover every column label")
            other = other.to_list()
        if isinstance(other, (list, tuple, np.ndarray)):
            if len(other) != len(block.cols):
                raise ValueError(f"Unable to coerce to Series, length must be {len(block.cols)}: given {len(other)}")
            return self._scalar(block, list(other))
        raise NotImplementedError(f"binary op with {type(other).__name__} operand is not on the B200 path")


class DevLogical(DevFn):
    """``a & b``, ``a | b``, ``a ^ b`` between co-partitioned BOOL frames -- ``Binary.register(pandas.DataFrame.__and__
    / __or__ / __xor__)`` (qc.py:541-571).  Bool columns are uint8 0 / 1 buffers; the result stays bool."""

    def __init__(self, op: str):
        if op not in ("and", "or", "xor"):
            raise ValueError(op)
        self.op = op

    def __call__(self, block, other, *args, axis=None, level=None, fill_value=None, **kwargs):
        _check_block(block, f"DevLogical({self.op})")
        if not isinstance(other, DeviceBlock):
            raise NotImplementedError("logical ops on the B200 path take another bool frame")
        if block.nrows != other.nrows or len(block.cols) != len(other.cols) or not block.columns.equals(other.columns):
            raise NotImplementedError("logical op between differently shaped / labelled blocks")
        if any(c.dtype != np.bool_ for c in list(block.cols) + list(other.cols)):
            raise NotImplementedError("logical ops on the B200 path need bool columns (bitwise integer ops are not on it)")
        if block.nrows == 0 or not block.cols:
            return block
        return block.with_cols(ops.map_columns(self.op, block.cols, other.cols))


class DevIsin(DevFn):
    """``frame.isin(values)`` for int64 columns and a list of integers -- ``Map.register(pandas.DataFrame.isin)``
    (qc.py `isin`): a membership test is a join probe without payload: build a (dense or hashed) table over the
    distinct values once, probe every column, ``index >= 0`` is the answer."""

    op = "isin"

    def __init__(self, values):
        vals = np.asarray(list(values))
        if vals.size and vals.dtype.kind not in "iu":
            raise NotImplementedError("device isin takes integer values")
        self.values = np.unique(vals.astype(np.int64))
        self._tables = {}

    def _table(self, device):
        tab = self._tables.get(device)
        if tab is None:
            tab = ops.JoinTable(DeviceColumn.from_numpy(self.values))
            self._tables[device] = tab
        return tab

    def __call__(self, block, *args, **kwargs):
        _check_block(block, "DevIsin")
        if any(c.dtype != np.int64 for c in block.cols):
            raise NotImplementedError("device isin tests int64 columns")
        if not block.cols or block.nrows == 0:
            return block.with_cols([DeviceColumn.empty(block.nrows, np.bool_) for _ in block.cols])
        if self.values.size == 0:
            return block.with_cols(ops.map_columns("ne", list(block.cols), list(block.cols)))  # all False
        tab = self._table(str(block.cols[0].data.device))
        out = []
        for c in block.cols:
            idx, _ = tab.probe(c)
            out.extend(ops.map_columns("ge_s", [idx], s0=[0]))
        return block.with_cols(out)


class DevRowLogical(DevFn):
    """Row-wise ``all`` / ``any`` over the BOOL columns of a block -> one bool column (``df.all(axis=1)`` on the
    result of a predicate; what ``dropna`` needs).  W - 1 logical sweeps."""

    def __init__(self, op: str, label="__reduced__"):
        if op not in ("all", "any"):
            raise ValueError(op)
        self.op, self.label = op, label

    def __call__(self, block, *args, **kwargs):
        _check_block(block, f"DevRowLogical({self.op})")
        if not block.cols:
            raise NotImplementedError("row-wise all / any of a frame without columns")
        if any(c.dtype != np.bool_ for c in block.cols):
            raise NotImplementedError("row-wise all / any on the B200 path needs bool columns")
        acc = block.cols[0]
        kop = "and" if self.op == "all" else "or"
        for c in block.cols[1:]:
            acc = ops.map_columns(kop, [acc], [c])[0] if block.nrows else acc
        return block.with_cols([acc], pandas.Index([self.label]))


class DevRowFilter(DevFn):
    """``block[mask]`` for a co-partitioned bool column: boolean row selection (``df[bool_series]``,
    ``df.dropna()``; the reference reaches it through ``getitem_array`` -> ``take_2d_labels_or_positional``,
    df.py:1188-1389).  mask -> hit positions (ranked compaction) -> one gather per column; the surviving row
    labels travel as a device index column."""

    op = "row_filter"

    def __call__(self, block, mask_block=None, *args, **kwargs):
        _check_block(block, "DevRowFilter")
        if not isinstance(mask_block, DeviceBlock) or len(mask_block.cols) != 1 or mask_block.cols[0].dtype != np.bool_:
            raise NotImplementedError("row selection on the B200 path takes one co-partitioned bool column")
        if mask_block.nrows != block.nrows:
            raise ValueError("Item wrong length: the mask has to cover the rows of the frame one to one")
        if any(c.dtype == np.bool_ for c in block.cols):
            raise NotImplementedError("row selection of frames with bool columns is not on the B200 path")
        if block.index_host is not None:
            raise NotImplementedError("row selection keeps numeric / range row labels only")
        if block.index_cols and len(block.index_cols) != 1:
            raise NotImplementedError("row selection of a frame with a MultiIndex is not on the B200 path")
        if block.nrows == 0:
            return block
        flags = ops.cast_columns_i64([mask_block.cols[0]])
        idx = ops.map_columns("add_s", flags, s0=[-1])[0]  # 0 -> -1 (drop), 1 -> 0 (keep)
        pos, k = ops.compact_hits(idx)
        cols = ops.take_columns(block.cols, pos) if block.cols else []
        if block.index_cols:
            labels = ops.take_columns(block.index_cols, pos)[0]
            names = block.index_names
        else:
            labels = ops.map_columns("add_s", [pos], s0=[int(block.range_start)])[0] if k else pos
            names = [None]
        return DeviceBlock(cols, block.columns, nrows=k, index_cols=[labels], index_names=names)


class DevSortRows(DevFn):
    """``df.sort_values(by=one column)`` on one block holding all the rows -- the block-function form of
    ``B200Dataframe.sort_by`` for callers that apply functions to full-axis partitions (the Modin plug-in's
    ``qc.sort_rows_by_column_values``).  Nothing is re-implemented: the block is wrapped in a one-partition frame and
    handed to ``sort_by`` (order-preserving key image, stable LSD radix sort of (image, row id), one gather)."""

    op = "sort_rows"

    @staticmethod
    def resolve(columns: pandas.Index, by, ascending=True, **kwargs):
        """(key position, ascending) after the argument checks both query compilers share."""
        cols = [by] if not isinstance(by, (list, tuple)) else list(by)
        asc = ascending[0] if isinstance(ascending, (list, tuple)) else ascending
        if len(cols) != 1:
            raise NotImplementedError("device sort_values sorts by one column")
        if kwargs.get("na_position", "last") != "last":
            raise NotImplementedError("sort_values(na_position='first') is not on the B200 path")
        if kwargs.get("key") is not None:
            raise NotImplementedError("sort_values(key=) is not on the B200 path")
        if cols[0] not in columns:
            raise KeyError(cols[0])
        return int(columns.get_loc(cols[0])), bool(asc)

    def __call__(self, block, key_position=0, ascending=True, ignore_index=False, **kwargs):
        from .dataframe import B200Dataframe

        _check_block(block, "DevSortRows")
        frame = B200Dataframe.from_blocks([block])
        return frame.sort_by(int(key_position), bool(ascending), bool(ignore_index))._partitions[0, 0].get()


class DevDropDuplicates(DevFn):
    """``df.drop_duplicates(subset=[one int64 column], keep="first" | "last")`` on one block holding all the rows.
    The reference (modin/pandas/base.py:1600-1623 -> qc.unique, qc.py:2231-2270 -> BaseQueryCompiler.unique,
    base/query_compiler.py:2410-2435) computes ``duplicated(keep)`` over the subset, inverts it, selects the rows
    with that mask and optionally resets the index.  Same result here without materialising the mask in row order
    (there is no scatter on this path); composed from the sort, compaction and gather kernels, nothing of its own:

    1. stable sort of (key, row id): equal keys become runs, row ids ascending inside a run;
    2. run edges: ``sorted[i + 1] != sorted[i]`` (one elementwise sweep over two views shifted by a row);
    3. the row ids at the edges (first or last of every run) by ranked compaction + gather;
    4. those K row ids sorted back into row order, and one gather per column.

    Original row order and row labels are kept, as in pandas."""

    op = "drop_duplicates"

    @staticmethod
    def resolve(columns: pandas.Index, subset, keep) -> int:
        """Position of the ONE subset column, after the argument checks both query compilers share (``subset=None``
        means all columns, so it is accepted only for a one-column frame).  pandas' error types where it has one."""
        cols = list(columns) if subset is None else ([subset] if not isinstance(subset, (list, tuple)) else list(subset))
        if len(cols) != 1:
            raise NotImplementedError("device drop_duplicates compares one int64 column (pass subset=[column])")
        if cols[0] not in columns:
            raise KeyError(pandas.Index([cols[0]]))
        if keep not in ("first", "last"):
            if keep is False:
                raise NotImplementedError("drop_duplicates(keep=False) is not on the B200 path")
            raise ValueError('keep must be either "first", "last" or False')
        return int(columns.get_loc(cols[0]))

    def __call__(self, block, key_position=0, keep="first", ignore_index=False, **kwargs):
        _check_block(block, "DevDropDuplicates")
        if _spans_ranks(block):
            return self._across_ranks(block, key_position, keep, ignore_index)
        self._validate(block, key_position, keep, ignore_index)
        if block.nrows <= 1:
            return DeviceBlock(block.cols, block.columns, nrows=block.nrows, range_start=0) if ignore_index else block
        return self._rows(block, self._winners(block.cols[key_position], keep), ignore_index, 0)

    def _across_ranks(self, block, key_position, keep, ignore_index):
        """Rows sharded over ranks: equal keys may sit on different GPUs, so a shard-local answer is not the answer.
        Every rank finds its own first / last occurrence per key; only the KEYS of those survivors (one int64 per
        rank and distinct key) are all-gathered, in rank order -- which is row order, shards are contiguous; the
        same pass over the gathered keys names the job-wide winners, and every rank keeps the winners that came
        from its own survivors.  The result stays row-sharded and in row order like any other frame; no row moves."""
        from . import dist

        self._validate(block, key_position, keep, ignore_index)
        t = ops.torch_mod()
        key = block.cols[key_position]
        mine = self._winners(key, keep)  # positions inside this shard, ascending
        dev = key.data.device
        counts = [c[0] for c in dist.all_gather_small(t.tensor([len(mine)], dtype=t.int64, device=dev))]
        surv_keys = ops.take_columns([key], mine)[0] if len(mine) else DeviceColumn.empty(0, np.int64)
        all_keys = DeviceColumn(dist.all_gather_rows([surv_keys.data])[0], np.int64)
        win = self._winners(all_keys, keep)  # positions inside the gathered survivors, ascending
        start = int(sum(counts[: dist.rank()]))
        stop = start + int(counts[dist.rank()])
        keep_ids = DeviceColumn.empty(0, np.int64)
        if len(win) and stop > start:
            # winners that are this rank's survivors: positions in [start, stop) (digitize against the two bounds)
            bins = ops.digitize(win, [start, stop])
            hit = ops.map_columns("eq_s", [bins], s0=[1])[0]
            idx = ops.map_columns("add_s", ops.cast_columns_i64([hit]), s0=[-1])[0]  # 0 -> -1 (skip), 1 -> 0 (hit)
            pos, k = ops.compact_hits(idx)
            if k:
                local = ops.map_columns("add_s", ops.take_columns([win], pos), s0=[-start])[0]
                keep_ids = ops.take_columns([mine], local)[0]
        offset = dist.exclusive_row_offset(len(keep_ids)) if ignore_index else 0
        return self._rows(block, keep_ids, ignore_index, offset)

    @staticmethod
    def _validate(block, key_position, keep, ignore_index):
        if keep not in ("first", "last"):
            raise NotImplementedError("drop_duplicates(keep=False) is not on the B200 path")
        if block.cols[key_position].dtype != np.int64:
            raise NotImplementedError("device drop_duplicates needs an int64 subset column")
        if any(c.dtype == np.bool_ for c in block.cols):
            raise NotImplementedError("drop_duplicates of frames with bool columns is not on the B200 path")
        if block.index_host is not None and not ignore_index:
            raise NotImplementedError("drop_duplicates keeps numeric / range row labels only (or ignore_index=True)")
        if block.index_cols and len(block.index_cols) != 1 and not ignore_index:
            raise NotImplementedError("drop_duplicates of a frame with a MultiIndex is not on the B200 path")

    @staticmethod
    def _winners(key: DeviceColumn, keep: str) -> DeviceColumn:
        """Row positions holding the first / last occurrence of every key value, ascending (steps 1-4 above)."""
        t = ops.torch_mod()
        n = len(key)
        if n <= 1:
            return ops.iota(0, n)
        image = ops.map_columns("ordered_s", [key], s0=[0])[0]  # fresh buffer: the sort is in place
        perm = ops.iota(0, n)  # mb200_iota_i64: the row ids the sort carries along
        ops.sort_pairs(image, perm)
        edge = ops.map_columns("ne", [image.slice(1, n)], [image.slice(0, n - 1)])[0]  # edge[i]: run ends at i
        idx = ops.map_columns("add_s", ops.cast_columns_i64([edge]), s0=[-1])[0]  # 0 -> -1 (skip), 1 -> 0 (hit)
        pos, k = ops.compact_hits(idx)
        if keep == "first":  # sorted row 0 opens the first run; every edge i opens a run at i + 1
            always = perm.slice(0, 1)
            if k:
                pos = ops.map_columns("add_s", [pos], s0=[1])[0]
        else:  # every edge i closes a run at i; sorted row n - 1 closes the last one
            always = perm.slice(n - 1, n)
        picked = [ops.take_columns([perm], pos)[0].data] if k else []
        rid = DeviceColumn(t.cat([always.data] + picked), np.int64)  # K = k + 1 row ids, in key order
        ops.sort_pairs(rid, DeviceColumn.empty(k + 1, np.int64))  # back into row order (payload unused)
        return rid

    @staticmethod
    def _rows(block, rid: DeviceColumn, ignore_index: bool, new_start: int) -> DeviceBlock:
        """The rows ``rid`` of ``block`` with their labels (or renumbered from ``new_start``)."""
        k = len(rid)
        cols = ops.take_columns(block.cols, rid) if block.cols else []
        if ignore_index:
            return DeviceBlock(cols, block.columns, nrows=k, range_start=int(new_start))
        if block.index_cols:
            labels, names = ops.take_columns(block.index_cols, rid)[0], block.index_names
        else:
            labels, names = ops.map_columns("add_s", [rid], s0=[int(block.range_start)])[0], [None]
        return DeviceBlock(cols, block.columns, nrows=k, index_cols=[labels], index_names=names)


class DevBoolReduce(DevFn):
    """``df.any()`` / ``df.all()`` over BOOL columns -- ``TreeReduce.register(pandas.DataFrame.any / all)``
    (qc.py:986-987): any = max, all = min of the 0 / 1 values, per partition and again over the partials
    (and over the GPUs with one packed all_reduce).  An empty column gives any = False, all = True like pandas."""

    def __init__(self, op: str, phase: str = "map"):
        if op not in ("any", "all"):
            raise ValueError(op)
        self.op, self.phase = op, phase
        self.kop = "max" if op == "any" else "min"

    def _ints(self, block):
        if self.phase == "map":
            if any(c.dtype != np.bool_ for c in block.cols):
                raise NotImplementedError("any / all on the B200 path reduce bool columns (compare first)")
            return ops.cast_columns_i64(block.cols)
        return list(block.cols)  # partials are int64 0 / 1 (or the +-max identities of empty partitions)

    def _finish(self, vals, block):
        ints = [DeviceColumn(v, np.int64) for v in vals]
        if self.phase == "map":
            return _reduced_block(ints, block.columns)
        # reduce phase: int64 -> bool.  An all-empty frame leaves the identity: INT64_MIN for max (any -> False),
        # INT64_MAX for min (all -> True); both fall out of "> 0".
        return _reduced_block(ops.map_columns("gt_s", ints, s0=[0] * len(ints)), block.columns)

    def __call__(self, block, *args, axis=0, skipna=True, **kwargs):
        from . import dist

        _check_block(block, f"DevBoolReduce({self.op})")
        if axis not in (0, "index", None):
            raise NotImplementedError("row-wise any / all is not on the B200 path")
        if not block.cols:
            return _reduced_block([], block.columns)
        vals, _ = ops.reduce_columns(self.kop, self._ints(block), skipna=True, variant=1)
        if self.phase != "reduce" or not _spans_ranks(block):
            return self._finish(vals, block)
        dist.all_reduce_values(vals, [self.kop] * len(vals))
        res = self._finish(vals, block)
        res.replicated = True
        return res


class DevAffine(DevFn):
    """Fused ``x * s + t`` (two roundings) produced by the call-queue fusion pass."""

    op = "affine"

    def __init__(self, mul, add):
        self.mul, self.add = mul, add  # per-column lists or scalars

    def __call__(self, block, *args, **kwargs):
        _check_block(block, "DevAffine")
        W = len(block.cols)
        mul = list(self.mul) if isinstance(self.mul, (list, tuple, np.ndarray)) else [self.mul] * W
        add = list(self.add) if isinstance(self.add, (list, tuple, np.ndarray)) else [self.add] * W
        if block.nrows == 0 or not block.cols:
            # nothing to sweep, but the RESULT DTYPES still follow pandas (int64 * 2 + 1.5 is float64 on an empty frame
            # too): the two un-fused steps know how to answer for empty blocks
            return DevBinary("add")(DevBinary("mul")(block, self.mul), self.add)
        is_int = lambda v: isinstance(v, (int, np.integer)) and not isinstance(v, bool)  # noqa: E731
        cols, s0, s1 = [], [], []
        for c, m, a in zip(block.cols, mul, add):
            if c.dtype == np.int64 and is_int(m) and is_int(a):
                cols.append(c)  # int64 * int + int stays int64 (wrapping), like pandas
                s0.append(int(m))
                s1.append(int(a))
            else:
                cols.append(ops.cast_columns_f64([c])[0])
                s0.append(float(m))
                s1.append(float(a))
        return block.with_cols(ops.map_columns("affine", cols, s0=s0, s1=s1))


class DevFma3(DevFn):
    """Fused ``a * b + c`` over three co-partitioned blocks (two roundings)."""

    op = "fma3"

    def __call__(self, a, b, c, *args, **kwargs):
        for x in (a, b, c):
            _check_block(x, "DevFma3")
        if not (a.nrows == b.nrows == c.nrows and len(a.cols) == len(b.cols) == len(c.cols)):
            raise ValueError("fma3 needs identically shaped operands")
        if any(x.dtype != np.float64 for blk in (a, b, c) for x in blk.cols):
            raise NotImplementedError("fused a*b+c needs float64 columns")
        return a.with_cols(ops.map_columns("fma3", a.cols, b.cols, c.cols))


# ------------------------------------------------------------------ TreeReduce functors
def _reduced_block(cols, columns, label=MODIN_UNNAMED_SERIES_LABEL):
    return DeviceBlock(cols, columns, nrows=1, index_host=pandas.Index([label]))


class DevReduce(DevFn):
    """``pandas.DataFrame.sum/count/min/max(axis=0)`` of one block -> 1 x W block.

    Used both as map and as reduce function of TreeReduce (qc.py:976-1035): the reduce phase
    sees the row-concatenation of the per-partition 1 x W partials.
    """

    def __init__(self, op: str, phase: str = "map"):
        if op not in ("sum", "count", "min", "max", "prod"):
            raise ValueError(op)
        self.op = op
        self.phase = phase  # "map" | "reduce"

    def _kernel_op(self):
        if self.phase == "reduce" and self.op == "count":
            return "sum"  # counts add up (qc.py:976: TreeReduce.register(count, sum))
        return self.op

    @staticmethod
    def _widen_bools(block, kop):
        """sum / count of bool columns: pandas sums booleans as int64 (``(df > 0).sum()``); min / max / prod of
        booleans would have to return bool and are left out."""
        if not any(c.dtype == np.bool_ for c in block.cols):
            return block
        if kop not in ("sum", "count"):
            raise NotImplementedError(f"{kop} over bool columns is not on the B200 path (use any / all / sum)")
        return block.with_cols(ops.cast_columns_i64(block.cols))

    def _check(self, block, axis, min_count):
        _check_block(block, f"DevReduce({self.op})")
        if axis not in (0, "index", None):
            raise NotImplementedError("row-wise (axis=1) reductions are not on the B200 path")
        if min_count and min_count > 1:
            raise NotImplementedError("sum(min_count>1) is a full-axis Reduce in the reference; not on the B200 path")

    def __call__(self, block, *args, axis=0, skipna=True, numeric_only=False, min_count=0, **kwargs):
        self._check(block, axis, min_count)
        if not block.cols:
            return _reduced_block([], block.columns)
        spans = self.phase == "reduce" and _spans_ranks(block)
        kop = self._kernel_op()
        block = self._widen_bools(block, kop)
        vals, cnts = ops.reduce_columns(kop, block.cols, skipna=bool(skipna), variant=ReduceVariant.get())
        if spans:
            return self._across_ranks(block, kop, vals, cnts, skipna, min_count)
        out = []
        for j, c in enumerate(block.cols):
            if kop == "count":
                out.append(DeviceColumn(cnts[j], np.int64))
            elif kop == "sum" and min_count == 1 and c.dtype == np.float64 and skipna:
                # pandas min_count=1: no valid value -> NaN.  Works through the tree exactly like the
                # reference: an all-NaN block yields a NaN partial, which the reduce phase skips.
                out.append(_nan_where_empty(vals[j], cnts[j]))
            else:
                out.append(DeviceColumn(vals[j], c.dtype))
        res = _reduced_block(out, block.columns)
        res.replicated = block.replicated  # a partial of rows every rank holds in full is such a partial too
        return res

    @staticmethod
    def _across_ranks(block, kop, vals, cnts, skipna, min_count):
        """Reduce phase when rows are sharded over several GPUs: this rank's reduction of its partials (``vals`` /
        ``cnts``) goes into ONE packed all_reduce of the W-vector (sum / min / max) -- the collective that replaces
        the reference's gather-to-one-task (axis_partition.py:445-452)."""
        from . import dist

        t = ops.torch_mod()
        W = len(block.cols)
        if kop == "count":
            dist.all_reduce_values(cnts, ["sum"] * W)
            out = [DeviceColumn(c, np.int64) for c in cnts]
        elif kop == "prod":
            # gather every rank's partial product per column (world_size values) and multiply locally
            vals = [dist.all_gather_rows([v.reshape(1)])[0].prod().reshape(1) for v in vals]
            out = [DeviceColumn(v, c.dtype) for v, c in zip(vals, block.cols)]
        elif kop == "sum":
            dist.all_reduce_values(vals, ["sum"] * W)
            if min_count == 1 and skipna:
                dist.all_reduce_values(cnts, ["sum"] * W)
                vals = [t.where(n == 0, t.full_like(v, float("nan")), v) if v.dtype == t.float64 else v
                        for v, n in zip(vals, cnts)]  # fmt: skip
            out = [DeviceColumn(v, c.dtype) for v, c in zip(vals, block.cols)]
        else:
            # min / max: a shard without valid values must not poison the others -> +-inf locally,
            # NaN decided from the job-wide counts (pandas: all-NaN -> NaN; skipna=False & any NaN -> NaN)
            nrows = t.full((1,), block.nrows, dtype=t.int64, device=vals[0].device)
            rows = [nrows.clone() for _ in range(W)]
            for j, c in enumerate(block.cols):
                if c.dtype == np.float64:
                    inf = float("inf") if kop == "min" else float("-inf")
                    vals[j] = t.where(cnts[j] > 0, t.nan_to_num(vals[j], nan=inf), t.full_like(vals[j], inf))
            dist.all_reduce_values(vals, [kop] * W)
            dist.all_reduce_values(cnts + rows, ["sum"] * (2 * W))
            out = []
            for j, c in enumerate(block.cols):
                v = vals[j]
                if c.dtype == np.float64:
                    bad = (cnts[j] == 0) if skipna else ((cnts[j] == 0) | (cnts[j] < rows[j]))
                    v = t.where(bad, t.full_like(v, float("nan")), v)
                out.append(DeviceColumn(v, c.dtype))
        res = _reduced_block(out, block.columns)
        res.replicated = True
        return res


def _nan_where_empty(val, cnt):
    """val if cnt > 0 else NaN, on device, for a 1-element tensor (min_count=1 semantics)."""
    v = DeviceColumn(val, np.float64)
    c = DeviceColumn(cnt, np.int64)
    cf = ops.cast_columns_f64([c])[0]
    # cf/cf is 1.0 when count > 0 and NaN when count == 0 ; multiply keeps val or makes NaN
    one_or_nan = ops.map_columns("div", [cf], [cf])[0]
    return ops.map_columns("mul", [v], [one_or_nan])[0]


class DevMeanMap(DevFn):
    """Map phase of mean: per-column (sum, count) -- qc.py:1046-1058 builds a 2-row frame with
    rows "sum"/"count"; here the partial is 1 x 2W: W float sums followed by W int64 counts."""

    op = "mean_map"

    def __call__(self, block, *args, axis=0, skipna=True, numeric_only=False, **kwargs):
        _check_block(block, "DevMeanMap")
        if axis not in (0, "index", None):
            raise NotImplementedError("row-wise mean is not on the B200 path")
        cols = ops.cast_columns_f64(block.cols)
        vals, cnts = ops.reduce_columns("sum", cols, skipna=bool(skipna), variant=ReduceVariant.get())
        out = [DeviceColumn(v, np.float64) for v in vals]
        if skipna:
            out += [DeviceColumn(c, np.int64) for c in cnts]
        else:  # count of rows, NaNs included (qc.py:1049-1053 uses len when skipna=False)
            import torch

            n = block.nrows
            out += [DeviceColumn(torch.full((1,), n, dtype=torch.int64, device=vals[0].device), np.int64)
                    for _ in cnts]  # fmt: skip
        return _reduced_block(out, _mean_partial_labels(block.columns))


_MEAN_LABELS: dict = {}


def _mean_partial_labels(columns: pandas.Index) -> pandas.MultiIndex:
    """("sum", c) ... ("count", c) ... for the 1 x 2W partial of a mean.  Building a MultiIndex costs the host more
    than the launch it labels (~0.6 ms), and a frame asks for the same one on every call: remembered per column set."""
    try:
        key = tuple(columns)
        hit = _MEAN_LABELS.get(key)
    except TypeError:  # unhashable labels: build, do not remember
        key = hit = None
    if hit is None:
        hit = pandas.MultiIndex.from_tuples([("sum", c) for c in columns] + [("count", c) for c in columns])
        if key is not None:
            if len(_MEAN_LABELS) >= 64:
                _MEAN_LABELS.clear()
            _MEAN_LABELS[key] = hit
    return hit


class DevMeanReduce(DevFn):
    """Reduce phase of mean: add the partial sums and counts, divide (qc.py:1060-1075)."""

    op = "mean_reduce"

    def _local(self, block):
        W = len(block.cols) // 2
        sums, _ = ops.reduce_columns("sum", block.cols[:W], skipna=False, variant=1)
        cnts, _ = ops.reduce_columns("sum", block.cols[W:], skipna=False, variant=1)
        labels = pandas.Index([t[1] for t in block.columns[:W]]) if isinstance(block.columns, pandas.MultiIndex) \
            else block.columns[:W]  # fmt: skip
        return sums, cnts, labels

    @staticmethod
    def _divide(sums, cnts, labels):
        s = [DeviceColumn(v, np.float64) for v in sums]
        c = ops.cast_columns_f64([DeviceColumn(v, np.int64) for v in cnts])
        return _reduced_block(ops.map_columns("div", s, c), labels)

    def __call__(self, block, *args, axis=0, skipna=True, **kwargs):
        from . import dist

        _check_block(block, "DevMeanReduce")
        sums, cnts, labels = self._local(block)
        if not _spans_ranks(block):
            return self._divide(sums, cnts, labels)
        # across ranks, sums and counts are all_reduced BEFORE the division (mean of shard means would be wrong)
        dist.all_reduce_values(sums + cnts, ["sum"] * (len(sums) + len(cnts)))
        res = self._divide(sums, cnts, labels)
        res.replicated = True
        return res


class DevVar(DevFn):
    """``pandas.DataFrame.var / std`` of one FULL column partition -> 1 x W block: the device body of the Reduce
    template (alg/reduce.py:32-71 -> PandasDataframe.reduce, df.py:2171-2205; qc.py:1155-1156 registers
    ``Reduce.register(pandas.DataFrame.std / var)``, i.e. pandas' two-pass nanops.nanvar over the gathered column).

    Two sweeps over the block, nothing leaves the device: (sum, count) -> means -> sums of squared deviations from
    those means (``mb200_reduce_columns_centered``) -> ``ssd / (count - ddof)``.  When the rows are sharded over
    ranks the W sums / counts and the W sums of squares are all-reduced in between -- the Reduce template's
    "gather the whole axis into one task" (axis_partition.py:445-452) becomes two packed W-vector collectives."""

    def __init__(self, sqrt: bool = False):
        self.sqrt = bool(sqrt)
        self.op = "std" if sqrt else "var"

    def __call__(self, block, *args, axis=0, skipna=True, ddof=1, numeric_only=False, **kwargs):
        from . import dist

        _check_block(block, f"DevVar({self.op})")
        if axis not in (0, "index", None) or args:
            raise NotImplementedError("row-wise var / std is not on the B200 path")
        if not block.cols:
            return _reduced_block([], block.columns)
        spans = _spans_ranks(block)
        t = ops.torch_mod()
        W = len(block.cols)
        cols = ops.cast_columns_f64(block.cols)
        sums, cnts = ops.reduce_columns("sum", cols, skipna=bool(skipna), variant=ReduceVariant.get())
        if spans:
            dist.all_reduce_values(list(sums) + list(cnts), ["sum"] * (2 * W))
        n = t.cat([c.reshape(1) for c in cnts]).to(t.float64)
        centers = t.cat([v.reshape(1) for v in sums]) / n
        ssd, _ = ops.reduce_columns("ssd", cols, skipna=bool(skipna), variant=ReduceVariant.get(), centers=centers)
        if spans:
            dist.all_reduce_values(list(ssd), ["sum"] * W)
        d = n - float(ddof)
        out = t.where(d > 0, t.cat([v.reshape(1) for v in ssd]) / d, t.full_like(d, float("nan")))
        if self.sqrt:
            out = t.sqrt(out)
        res = _reduced_block([DeviceColumn(out[j : j + 1], np.float64) for j in range(W)], block.columns)
        res.replicated = spans
        return res


_LABEL_EMPTY, _LABEL_I64, _LABEL_F64, _LABEL_REFUSED = 0, 1, 2, 3


class DevArgReduce(DevFn):
    """``pandas.DataFrame.idxmax / idxmin`` of one FULL column partition -> 1 x W block of row labels: the device body
    of the Reduce template (alg/reduce.py:32-71; qc.py:1101-1102 registers ``Reduce.register(pandas.DataFrame.idxmax
    / idxmin)``).

    One pass over the block (``mb200_reduce_arg_columns``) gives per column the extreme value, the first row holding it
    and the number of non-NaN values; the row becomes its label on the device (range start + row, or a gather from the
    device index column) and the counts decide pandas' errors.  When the rows are sharded over ranks every rank
    all-gathers its (value, label, count) W-vectors plus its row count -- one collective -- and combines them in rank
    order: the better value wins and a tie goes to the lower rank, which holds the earlier rows.  Ranks without a
    valid value in a column do not take part in it, and the errors are decided from the job-wide counts, so every rank
    raises the same error after the same collective.  Labels are int64 (range or int64 index) or float64; string
    labels, several index levels and ``axis=1`` are refused."""

    def __init__(self, op: str):
        if op not in ("max", "min"):
            raise ValueError(op)
        self.op = op

    @staticmethod
    def _label_kind(block):
        """(kind code, refusal message) of the block's row labels."""
        if block.nrows == 0:
            return _LABEL_EMPTY, None
        if block.has_range_index():
            return _LABEL_I64, None
        if block.index_cols:
            if len(block.index_cols) != 1:
                return _LABEL_REFUSED, "idxmax / idxmin over several index levels is not on the B200 path"
            return (_LABEL_F64 if block.index_cols[0].dtype == np.float64 else _LABEL_I64), None
        idx = block.index_host
        if isinstance(idx, pandas.MultiIndex):
            return _LABEL_REFUSED, "idxmax / idxmin over several index levels is not on the B200 path"
        if idx.dtype.kind not in "if":
            return _LABEL_REFUSED, f"idxmax / idxmin over {idx.dtype} row labels is not on the B200 path"
        return (_LABEL_F64 if idx.dtype.kind == "f" else _LABEL_I64), None

    @staticmethod
    def _labels(block, kind, pos):
        """Row labels at the W positions ``pos`` (int64 device tensor; -1 gives an arbitrary label)."""
        t = ops.torch_mod()
        if kind == _LABEL_EMPTY:
            return t.zeros_like(pos)
        p = DeviceColumn(pos, np.int64)
        if block.has_range_index():
            return ops.map_columns("add_s", [p], s0=[block.range_start])[0].data
        if block.index_cols:
            return ops.take_columns([block.index_cols[0]], p)[0].data
        host = block.index_host.to_numpy().astype(np.float64 if kind == _LABEL_F64 else np.int64)
        at = pos.tolist()
        return t.tensor([host[i] if i >= 0 else 0 for i in at], dtype=t.float64 if kind == _LABEL_F64 else t.int64,
                        device=pos.device)  # fmt: skip

    def _raise_for(self, counts, nrows, skipna):
        """pandas' errors (nanops._maybe_arg_null_out and the empty check), from the counts of the whole axis."""
        if nrows == 0:
            raise ValueError(f"attempt to get arg{self.op} of an empty sequence")
        if skipna and min(counts) == 0:
            raise ValueError("Encountered all NA values")
        if not skipna and min(counts) < nrows:
            raise ValueError("Encountered an NA value with skipna=False")

    def __call__(self, block, *args, axis=0, skipna=True, numeric_only=False, **kwargs):
        _check_block(block, f"DevArgReduce({self.op})")
        if axis not in (0, "index", None) or args:
            raise NotImplementedError(f"row-wise idx{self.op} (axis=1) is not on the B200 path")
        if not block.cols:
            return _reduced_block([], block.columns)
        spans = _spans_ranks(block)
        kind, refusal = self._label_kind(block)
        if refusal and not spans:
            raise NotImplementedError(refusal)
        t = ops.torch_mod()
        W = len(block.cols)
        cols = ops.cast_columns_i64(block.cols)
        vals, poss, cnts = ops.arg_reduce_columns(self.op, cols, ReduceVariant.get())
        pos = t.cat([p.reshape(1) for p in poss])
        cnt = t.cat([c.reshape(1) for c in cnts])
        labels = self._labels(block, kind, pos) if not refusal else t.zeros_like(pos)
        nrows = block.nrows
        if spans:
            labels, cnt, nrows, kind = self._combine_ranks(vals, labels, cnt, nrows, kind, cols)
        host = t.cat([cnt, t.full((1,), nrows, dtype=t.int64, device=cnt.device)]).tolist()  # one D2H
        self._raise_for(host[:W], host[W], bool(skipna))
        dtype = np.float64 if kind == _LABEL_F64 else np.int64
        out = [DeviceColumn(labels[j : j + 1], dtype) for j in range(W)]
        res = _reduced_block(out, block.columns)
        res.replicated = spans
        return res

    def _combine_ranks(self, vals, labels, cnt, nrows, kind, cols):
        """All-gather (value bits, label bits, count) per column and (rows, label kind) per rank, combine in rank
        order.  Returns the job-wide (labels, counts, rows, label kind); raises on every rank alike."""
        from . import dist

        t = ops.torch_mod()
        W = len(cols)
        bits = lambda x: x.view(t.int64) if x.dtype == t.float64 else x  # noqa: E731
        vb = t.cat([bits(v.reshape(1)) for v in vals])
        meta = t.tensor([nrows, kind], dtype=t.int64, device=vb.device)
        g = dist.all_gather_fixed(t.cat([vb, bits(labels), cnt, meta])).view(-1, 3 * W + 2)
        rank_meta = g[:, 3 * W :].tolist()  # [rows, label kind] per rank
        kinds = {k for _, k in rank_meta} - {_LABEL_EMPTY}
        if _LABEL_REFUSED in kinds or len(kinds) > 1:
            raise NotImplementedError("idxmax / idxmin on the B200 path need int64 or float64 row labels of one kind "
                                      "on every rank")  # fmt: skip
        is_f = t.tensor([c.dtype == np.float64 for c in cols], device=vb.device)
        v_i, lab, cn = g[:, :W].contiguous(), g[:, W : 2 * W].contiguous(), g[:, 2 * W : 3 * W]
        v_f = v_i.view(t.float64)
        best_i, best_f, best_l, have = v_i[0], v_f[0], lab[0], cn[0] > 0
        for r in range(1, g.shape[0]):
            ok = cn[r] > 0
            if self.op == "max":
                better = t.where(is_f, v_f[r] > best_f, v_i[r] > best_i)
            else:
                better = t.where(is_f, v_f[r] < best_f, v_i[r] < best_i)
            take = ok & (~have | better)  # strict: a tie stays with the lower rank
            best_i, best_f = t.where(take, v_i[r], best_i), t.where(take, v_f[r], best_f)
            best_l = t.where(take, lab[r], best_l)
            have = have | ok
        kind = kinds.pop() if kinds else _LABEL_I64
        out = best_l.view(t.float64) if kind == _LABEL_F64 else best_l
        return out, cn.sum(0), sum(n for n, _ in rank_meta), kind


# ------------------------------------------------------------------ Fold functor
class DevCumulative(DevFn):
    """``pandas.DataFrame.cumsum / cummax / cummin`` (qc.py:2429-2431) and ``DataFrame.ffill`` (``fillna(method=
    "ffill")``, qc.py:2809-2810) of one full column partition: the device body of the Fold template
    (alg/fold.py:32-95 -> PandasDataframe.fold, df.py:2357-2400).

    The reference gathers every row block of the column partition into one pandas frame and runs the sequential
    function over it.  Here the block is scanned by tiles (csrc/cum.cu: tile aggregates -> per-column scan of the
    aggregates -> tiles with their prefix); when the rows are sharded over ranks each rank scans its own shard and the
    rows before it arrive as ONE number per column: the ranks all-gather their column totals (W x 8 bytes each) and
    combine those of the lower ranks in rank order into the carry of the second pass.  NaN are skipped like pandas
    does (``skipna=True`` only); bool columns are refused (pandas returns object / int columns for them)."""

    def __init__(self, op: str):
        if op not in ("sum", "max", "min", "ffill"):
            raise ValueError(op)
        self.op = op

    def __call__(self, block, *args, axis=0, skipna=True, **kwargs):
        _check_block(block, f"DevCumulative({self.op})")
        if axis not in (0, "index", None) or args:
            raise NotImplementedError("row-wise (axis=1) cumulative functions are not on the B200 path")
        if not skipna:
            raise NotImplementedError("cumulative functions with skipna=False are not on the B200 path")
        if self.op == "ffill" and (kwargs.get("limit") is not None or kwargs.get("limit_area") is not None):
            raise NotImplementedError("ffill(limit=) is not on the B200 path")
        return self._run(block, _spans_ranks(block))

    def _run(self, block, distributed: bool):
        from . import dist

        if any(c.dtype == np.bool_ for c in block.cols):
            raise NotImplementedError(f"cumulative {self.op} over bool columns is not on the B200 path")
        # forward fill leaves integer columns as they are (they hold no NaN)
        sel = [j for j, c in enumerate(block.cols) if not (self.op == "ffill" and c.dtype != np.float64)]
        if not sel or (block.nrows == 0 and not distributed):
            return block
        cols = [block.cols[j] for j in sel]
        state = ops.cum_partials(self.op, cols)
        carries = None
        if distributed:
            gathered = [dist.all_gather_fixed(g[3]) for g in state.groups]
            carries = ops.cum_carry(state, gathered, dist.rank())
        outs = ops.cum_apply(state, cols, carries)
        new_cols = list(block.cols)
        for j, c in zip(sel, outs):
            new_cols[j] = c
        return block.with_cols(new_cols)


# ------------------------------------------------------------------ label alignment (the reindexing half of _copartition)
def _labels_block(block, cols, labels: pandas.Index, replicated=False):
    """``cols`` under new row ``labels`` (RangeIndex -> O(1) metadata, numeric -> device index column, else host)."""
    n = len(labels)
    if isinstance(labels, pandas.RangeIndex) and labels.step == 1 and labels.name is None:
        out = DeviceBlock(cols, block.columns, nrows=n, range_start=labels.start)
    elif not isinstance(labels, pandas.MultiIndex) and labels.dtype.kind in "if" and n > 0:
        arr = labels.to_numpy()
        arr = arr.astype(np.int64) if arr.dtype.kind == "i" else arr.astype(np.float64)
        out = DeviceBlock(cols, block.columns, nrows=n, index_cols=[DeviceColumn.from_numpy(arr)], index_names=[labels.name])
    else:
        out = DeviceBlock(cols, block.columns, nrows=n, index_host=labels)
    out.replicated = replicated
    return out


class DevReindex(DevFn):
    """``df.reindex(labels, axis=axis)`` of one full-axis block -- the function ``PandasDataframe._copartition``
    ships to ``map_axis_partitions`` for every frame whose labels differ from the joined index (df.py:3799-3840,
    ``make_reindexer`` df.py:2058-2073).  Rows: a join table over the block's own labels is probed with the target
    labels and the columns are gathered (``mb200_join_build`` / ``probe`` / ``take``); labels that the block does not
    have become NaN rows, which promotes int64 columns to float64 exactly as pandas does.  Columns: buffers are
    re-ordered by reference, missing labels become NaN columns."""

    op = "reindex"

    def __call__(self, block, labels, axis=0, fill_value=None, **kwargs):
        _check_block(block, "DevReindex")
        if fill_value is not None and not (isinstance(fill_value, float) and np.isnan(fill_value)):
            raise NotImplementedError("reindex(fill_value=) is not on the B200 path")
        labels = labels if isinstance(labels, pandas.Index) else pandas.Index(labels)
        if axis in (1, "columns"):
            return self._columns(block, labels)
        if axis not in (0, "index"):
            raise ValueError(f"No axis named {axis}")
        return self._rows(block, labels)

    @staticmethod
    def with_indexer(block, labels, indexer):
        """Rows gathered by a HOST-computed positional indexer (-1 = no such row -> NaN): what
        ``df._reindex_with_indexers({0: [joined_index, indexer]}, allow_dups=True)`` does for frames whose labels
        repeat (``make_reindexer``, df.py:2064-2072 -- the reference computes those indexers on the host too)."""
        labels = labels if isinstance(labels, pandas.Index) else pandas.Index(labels)
        if indexer is None:
            return _labels_block(block, list(block.cols), labels, replicated=block.replicated)
        pos = np.asarray(indexer, dtype=np.int64)
        misses = int((pos < 0).sum())
        cols = []
        for c in block.cols:
            if misses and c.dtype == np.bool_:
                raise NotImplementedError("re-indexing would put NaN into a bool column (object dtype in pandas)")
            cols.append(ops.cast_columns_f64([c])[0] if misses and c.dtype == np.int64 else c)
        idx = DeviceColumn.from_numpy(pos) if len(pos) else DeviceColumn.empty(0, np.int64)
        out = ops.take_columns(cols, idx) if cols else []
        return _labels_block(block, out, labels, replicated=block.replicated)

    @staticmethod
    def _columns(block, labels):
        if not block.columns.is_unique:
            raise ValueError("cannot reindex on an axis with duplicate labels")
        pos = block.columns.get_indexer(labels)
        cols = [block.cols[p] if p >= 0 else ops.full_column(block.nrows, np.float64, float("nan")) for p in pos]
        return block.with_cols(cols, labels)

    @staticmethod
    def _rows(block, labels):
        n_t = len(labels)
        numeric = (not isinstance(labels, pandas.MultiIndex) and labels.dtype.kind in "if"
                   and block.index_host is None and (not block.index_cols or len(block.index_cols) == 1))  # fmt: skip
        if n_t == 0 or block.nrows == 0 or not numeric:
            src = block.index  # host labels (small blocks, non-numeric labels): the indexer is computed on the host
            if not src.is_unique:
                raise ValueError("cannot reindex on an axis with duplicate labels")
            pos = src.get_indexer(labels).astype(np.int64)
            misses = int((pos < 0).sum())
            idx = DeviceColumn.from_numpy(pos) if n_t else DeviceColumn.empty(0, np.int64)
        else:
            src = block.index_cols[0] if block.index_cols else ops.iota(block.range_start, block.nrows)
            tgt_np = labels.to_numpy()
            if src.dtype == np.float64 or tgt_np.dtype.kind == "f":
                # float labels (or int against float): compare through the order-preserving int64 image, in which
                # -0.0 and 0.0 are one label
                from .groupkeys import float_image

                tgt = float_image(DeviceColumn.from_numpy(tgt_np.astype(np.float64)))
                src = float_image(ops.cast_columns_f64([src])[0])
            else:
                tgt = DeviceColumn.from_numpy(tgt_np.astype(np.int64))
            table = ops.JoinTable(src)
            try:
                if not table.is_unique():
                    raise ValueError("cannot reindex on an axis with duplicate labels")
                idx, nmatch = table.probe(tgt)
                misses = n_t - int(nmatch.item())
            finally:
                table.close()
        cols = []
        for c in block.cols:
            if misses and c.dtype == np.bool_:
                raise NotImplementedError("re-indexing would put NaN into a bool column (object dtype in pandas)")
            cols.append(ops.cast_columns_f64([c])[0] if misses and c.dtype == np.int64 else c)
        out = ops.take_columns(cols, idx) if cols else []
        return _labels_block(block, out, labels, replicated=block.replicated)


# ------------------------------------------------------------------ GroupByReduce functors
class _Partial(NamedTuple):
    """What a partial group table of one aggregation carries: the table flags, and the emitted arrays in column order
    (``sums`` / ``cnts``: one column per value column, under the value labels -- or under ``("sum", label)`` /
    ``("count", label)`` when there are both; ``sizes``: one column labelled "size")."""

    flags: int
    arrays: tuple


_PARTIALS = {
    "min": _Partial(_lib.GB_MIN, ("sums",)),
    "max": _Partial(_lib.GB_MAX, ("sums",)),
    "sum": _Partial(_lib.GB_SUM, ("sums",)),
    "count": _Partial(_lib.GB_COUNT, ("cnts",)),
    "size": _Partial(_lib.GB_SIZE, ("sizes",)),
    "mean": _Partial(_lib.GB_SUM | _lib.GB_COUNT, ("sums", "cnts")),  # mean = sums / counts, in _finished_block
}


def _partial_cols(agg, sums, cnts, sizes):
    """The emitted arrays of a table in the partial layout of ``agg``."""
    got = {"sums": sums, "cnts": cnts, "sizes": [sizes]}
    return [c for name in _PARTIALS[agg].arrays for c in got[name]]


def _partial_labels(agg, labels):
    arrays = _PARTIALS[agg].arrays
    if arrays == ("sizes",):
        return pandas.Index(["size"])
    if len(arrays) == 1:
        return labels
    tags = {"sums": "sum", "cnts": "count"}
    return pandas.MultiIndex.from_tuples([(tags[name], c) for name in arrays for c in labels])


_VALUE_POSITIONS: dict = {}


def _value_positions(columns: pandas.Index, key_label):
    """Positions and labels of the columns other than ``key_label``.  Iterating and slicing a pandas Index (Arrow-backed
    strings under pandas 3) costs ~0.15 ms of host time per query; a frame asks the same question on every query, so the
    answer is remembered per Index object (identity + the label; Index objects are immutable)."""
    memo = _VALUE_POSITIONS.get(id(columns))
    if memo is not None and memo[0] is columns and memo[1] == key_label:
        return memo[2], memo[3]
    keep = [i for i, lab in enumerate(columns) if lab != key_label]
    labels = columns[keep]
    if len(_VALUE_POSITIONS) >= 64:
        _VALUE_POSITIONS.clear()
    _VALUE_POSITIONS[id(columns)] = (columns, key_label, keep, labels)  # holding `columns` keeps the id from being reused
    return keep, labels


def _split_key_values(block: DeviceBlock, by_block: Optional[DeviceBlock], who: str):
    """Key column, its label, value columns and their labels of one row block (alg/groupby.py:186-206: with
    drop=True the `by` column is taken out of the data, or concatenated in when it lives in another frame)."""
    _check_block(block, who)
    if by_block is None:
        raise NotImplementedError("groupby needs a `by` block on the B200 path")
    if len(by_block.cols) != 1:
        raise NotImplementedError("multi-column `by` is not on the B200 path yet")
    key = by_block.cols[0]
    keep, labels = _value_positions(block.columns, by_block.columns[0])
    if key.dtype != np.int64:
        raise NotImplementedError("device groupby needs an int64 key column")
    return key, by_block.columns[0], [block.cols[i] for i in keep], labels


def _aggregated_values(agg, vals):
    """The value columns ``agg`` aggregates: none for size, float64 images for count / mean (the table counts non-NaN
    float64 values); the others take float64 columns only."""
    if agg == "size":
        return []
    vals = ops.cast_columns_f64(vals) if agg in ("count", "mean") else vals
    if any(v.dtype != np.float64 for v in vals):
        raise NotImplementedError(f"device groupby.{agg} aggregates float64 value columns only")
    return vals


def _group_block(cols, labels, keys, key_label, count_dev=None):
    """One row per group, ascending by key (the device index column).  With ``count_dev`` the columns have room for
    more rows than there are groups; the count stays on the device until it is read."""
    if count_dev is not None:
        blk = DeviceBlock.with_device_count(cols, labels, count_dev, index_cols=[keys], index_names=[key_label],
                                            check=ops.refuse_dense_overflow)  # fmt: skip
    else:
        blk = DeviceBlock(cols, labels, nrows=len(keys), index_cols=[keys], index_names=[key_label])
    blk.keys_sorted_unique = True
    return blk


def _finished_block(agg, keys, key_label, cols, labels):
    """The groupby result from merged partial columns ``cols`` (the layout of ``agg``); ``labels`` are the value
    labels.  A mean divides its sums by its counts."""
    if agg == "mean":
        W = len(cols) // 2
        cf = ops.cast_columns_f64(cols[W:])
        cols = ops.map_columns("div", cols[:W], cf) if len(keys) else cols[:W]
        return _group_block(cols, labels, keys, key_label)
    return _group_block(cols, _partial_labels(agg, labels), keys, key_label)


class DevGroupbyMap(DevFn):
    """GroupByReduce.map (alg/groupby.py:124-208): hash-aggregate one row block against its
    slice of `by` into a partial table (index = keys, ascending)."""

    def __init__(self, agg: str, capacity_hint: int = 1 << 20):
        if agg not in _PARTIALS:
            raise NotImplementedError(f"groupby.{agg} is not on the B200 path")
        self.agg = agg
        self.op = f"groupby_{agg}_map"
        self.capacity_hint = capacity_hint

    def __call__(self, block, by_block=None, *args, **kwargs):
        key, key_label, vals, labels = _split_key_values(block, by_block, self.op)
        vals = _aggregated_values(self.agg, vals)
        keys, sums, cnts, sizes = ops.hash_aggregate([(key, vals)], _PARTIALS[self.agg].flags, self.capacity_hint)
        return _group_block(_partial_cols(self.agg, sums, cnts, sizes), _partial_labels(self.agg, labels), keys, key_label)


def keys_to_columns(block: DeviceBlock, offset: int = 0) -> DeviceBlock:
    """``groupby(..., as_index=False)``: the group keys (device index columns) become the leading columns and the rows
    get a fresh RangeIndex starting at ``offset`` (``GroupBy.handle_as_index_for_dataframe``, alg/groupby.py:278-294)
    -- buffers are shared, nothing is copied."""
    if not block.index_cols:
        return block
    names = list(block.index_names or [None] * len(block.index_cols))
    clash = [n for n in names if n in set(block.columns)]
    if clash:
        raise ValueError(f"cannot insert {clash[0]}, already exists")
    labels = pandas.Index(names).append(block.columns)
    return DeviceBlock(list(block.index_cols) + list(block.cols), labels, nrows=block.nrows, range_start=offset)


class DevGroupbyReduce(DevFn):
    """GroupByReduce.reduce (alg/groupby.py:211-300): regroup the concatenated partial tables by
    key (level 0) with the reduce aggregation (sum of sums / counts / sizes; mean = sum/count)."""

    def __init__(self, agg: str):
        self.agg = agg
        self.op = f"groupby_{agg}_reduce"

    def _merge(self, keys, cols):
        """Regroup partial rows by key -> ascending unique keys + merged partial columns (same layout as the input).
        Partial sums add up, partial minima / maxima reduce with min / max, counts and sizes add up."""
        layout = _PARTIALS[self.agg]
        W = len(cols) // len(layout.arrays)
        got = {name: list(cols[i * W : (i + 1) * W]) for i, name in enumerate(layout.arrays)}
        sums, cnts, sizes = got.get("sums"), got.get("cnts"), got.get("sizes", [None])[0]
        if sums is None:
            # partial counts are merged through the count accumulators, which want value columns (ignored)
            sums = ops.cast_columns_f64(cnts) if cnts is not None else []
        k, s, c, z = ops.hash_aggregate([(keys, sums, cnts, sizes)], layout.flags, len(keys), partial=True)
        return k, _partial_cols(self.agg, s, c, z)

    def _finalize(self, k, cols, columns, key_label):
        labels = pandas.Index([t[1] for t in columns[: len(cols) // 2]]) if self.agg == "mean" else columns
        return _finished_block(self.agg, k, key_label, cols, labels)

    def __call__(self, block, *args, partition_idx=0, **kwargs):
        _check_block(block, self.op)
        if not block.index_cols:
            raise ValueError("groupby reduce expects partial tables keyed by device index columns")
        keys, key_label = block.index_cols[0], (block.index_names[0] if block.index_names else None)
        # a single partial table (one row partition on this GPU) is already one row per key, ascending:
        # nothing to regroup -- the reference would re-run groupby(level=0) on it to the same effect
        k, cols = (keys, list(block.cols)) if block.keys_sorted_unique else self._merge(keys, block.cols)
        if _spans_ranks(block):
            k, cols = self._across_ranks(k, cols)
        return self._finalize(k, cols, block.columns, key_label)

    def _across_ranks(self, k, cols):
        """The groupby shuffle: range-partition this rank's merged table by key over the ranks (all-to-all of <= G
        pre-aggregated rows per GPU, never raw rows) and merge what arrives.  Rank r ends up owning the r-th key
        range, ascending -- the concatenation over ranks is the reference's key-sorted result."""
        from . import dist

        rk, rcols = dist.exchange_by_key_range(k.data, [c.data for c in cols])
        rkeys = DeviceColumn(rk, np.int64)
        rc = [DeviceColumn(t_, c.dtype) for t_, c in zip(rcols, cols)]
        return self._merge(rkeys, rc) if len(rkeys) else (rkeys, rc)


def fused_dense_groupby(map_fn: "DevGroupbyMap", reduce_fn: "DevGroupbyReduce", blocks, by_blocks):
    """GroupByReduce with map and reduce fused for keys in a narrow range: ONE direct-addressed table per
    GPU absorbs every row partition resident on it (no per-partition emit, no regroup), the tables of
    all GPUs are merged in place by element-wise collectives (NCCL SUM / MIN / MAX over NVLink; no
    key exchange at all), and each rank emits its slice of the key range, ascending.

    Returns the finished result block, or None when the keys are not dense-able (the caller then runs
    the general map -> exchange -> reduce path).  Every rank takes the same decision: it is made on the
    job-wide key range and row count (``ops.plan_table``)."""
    from . import dist
    from .config import GroupbyAsyncEmit

    agg = map_fn.agg
    if agg != reduce_fn.agg or not blocks or len(blocks) != len(by_blocks):
        return None
    inputs = [_split_key_values(block, by_block, map_fn.op) for block, by_block in zip(blocks, by_blocks)]
    key_label, labels = inputs[0][1], (inputs[0][3] if agg != "size" else inputs[0][3][:0])
    if len(labels) > _lib.MAX_COLS:
        return None
    plan = ops.plan_table([inp[0] for inp in inputs], len(labels), _PARTIALS[agg].flags, map_fn.capacity_hint,
                          job_wide=True)  # fmt: skip
    if plan is None:
        return None
    table, mine = plan.create(), None
    try:
        ops.fill_table(table, [(key, _aggregated_values(agg, vals)) for key, _, vals, _ in inputs])
        if plan.chunk:
            # the reduce phase: rank r receives the merged accumulators of ITS key slice only (no keys move,
            # no sort, no pivots) and emits it; the rank-ordered results are the reference's key-sorted frame
            mine = table.reduce_scatter(plan.chunk, dist.reduce_scatter, dist.rank())
        emitter = mine if mine is not None else table
        if agg != "mean" and GroupbyAsyncEmit.get():
            # no host round trip: the result block is sized on the device and learns its row count when somebody
            # asks (DeviceBlock.with_device_count) -- the host is free to prepare the next query meanwhile
            keys, sums, cnts, sizes, count = emitter.emit_async()
            return _group_block(_partial_cols(agg, sums, cnts, sizes), _partial_labels(agg, labels), keys, key_label,
                                count_dev=count)  # fmt: skip
        keys, sums, cnts, sizes = ops.emit_counted(emitter, sort=False)
    finally:
        table.close()
        if mine is not None:
            mine.close()
    return _finished_block(agg, keys, key_label, _partial_cols(agg, sums, cnts, sizes), labels)


# ------------------------------------------------------------------ broadcast merge functor
_BOOL_MISSES = "device merge(how='left') with a bool payload column and unmatched left rows (pandas gives object dtype)"


class DevMerge(DevFn):
    """Per-row-partition ``pandas.merge(left_block, right, how, on / left_on / right_on, sort=False)`` of
    MergeImpl.row_axis_merge (merge.py:139-168) as a join-table probe + payload gather.

    * distinct right keys (many-to-one): probe + fused payload gather, the fact columns of a left join shared by
      reference;
    * repeated right keys (many-to-many): every left row yields one row per matching right row, left order kept, the
      matches in their order on the right (``ops.expand_matches``), then two gathers;
    * ``left_on != right_on``: both key columns appear in the result, like pandas.

    ``promote_ints``: whether int64 payload columns of a LEFT join become float64 (pandas does that when some left
    row finds no match, for the NaN).  The caller decides it ONCE for the whole job (all row partitions, all ranks:
    ``count_misses`` + all_reduce), so that every partition of the result carries the same dtypes; ``None`` = decide
    per block (single-partition callers)."""

    op = "merge"

    def __init__(self, on=None, how="left", suffixes=("_x", "_y"), left_on=None, right_on=None, promote_ints=None,
                 table_cache=None):  # fmt: skip
        if how not in ("left", "inner"):
            raise NotImplementedError("device merge supports how='left' and how='inner'")
        self.left_on = on if left_on is None else left_on
        self.right_on = on if right_on is None else right_on
        if self.left_on is None or self.right_on is None:
            raise NotImplementedError("device merge needs `on` (or `left_on` and `right_on`)")
        self.on, self.how, self.suffixes, self.promote_ints = self.left_on, how, suffixes, promote_ints
        # {right key label: (right block, table, unique)}.  Handed in by ``merge.row_axis_merge`` it lives on the
        # combined (broadcast) right frame, so that a dim frame is built into a table ONCE however often it is merged
        self._cache = table_cache if table_cache is not None else {}

    def _table(self, right: DeviceBlock):
        """(join table over the right keys, are they distinct) -- built once per right block and kept (the library
        also keeps the key-ordered payload copies of a dense table with it)."""
        keys = right.column(self.right_on)
        ident = (keys.ptr, len(keys))  # the key BUFFER identifies the table: blocks are re-wrapped freely, buffers are immutable
        ent = self._cache.get(self.right_on)
        if ent is None or ent[0] != ident:
            if ent is not None:
                ent[1].close()
            table = ops.JoinTable(keys)
            ent = (ident, table, table.is_unique())
            self._cache[self.right_on] = ent
        return ent[1], ent[2]

    _LABELS: dict = {}

    def result_labels(self, left_columns, right_columns):
        """(positions of the right columns that enter the result, left labels, right labels) with pandas' suffixes.
        Asked twice per merge (frame metadata, then the block functor) with the same two Index objects on every query
        of a stream: remembered per (Index identities, keys, suffixes) -- iterating pandas Indexes is host time the
        probe kernel does not have at 8 GPUs."""
        key = (id(left_columns), id(right_columns), self.left_on, self.right_on, tuple(self.suffixes))
        try:
            memo = DevMerge._LABELS.get(key)
        except TypeError:
            key = memo = None
        if memo is not None and memo[0] is left_columns and memo[1] is right_columns:
            return memo[2]
        out = self._result_labels(left_columns, right_columns)
        if key is not None:
            if len(DevMerge._LABELS) >= 64:
                DevMerge._LABELS.clear()
            DevMerge._LABELS[key] = (left_columns, right_columns, out)  # the references keep the ids from being reused
        return out

    def _result_labels(self, left_columns, right_columns):
        same = self.left_on == self.right_on
        pay_pos = [i for i, lab in enumerate(right_columns) if not (same and lab == self.right_on)]
        pay_labels = [right_columns[i] for i in pay_pos]
        left_labels = list(left_columns)
        overlap = set(left_labels) & set(pay_labels)
        ll = [f"{x}{self.suffixes[0]}" if x in overlap else x for x in left_labels]
        rl = [f"{x}{self.suffixes[1]}" if x in overlap else x for x in pay_labels]
        return pay_pos, ll, rl

    def count_misses(self, left: DeviceBlock, right: DeviceBlock) -> int:
        """Left rows of this block whose key is not on the right (host int; one probe pass, one sync)."""
        table, _ = self._table(right)
        _, nmatch = table.probe(left.column(self.left_on))
        return left.nrows - int(nmatch.item())

    def __call__(self, left, right, *args, **kwargs):
        _check_block(left, "DevMerge")
        _check_block(right, "DevMerge")
        table, unique = self._table(right)
        fact_keys = left.column(self.left_on)
        pay_pos, ll, rl = self.result_labels(left.columns, right.columns)
        pay_cols = [right.cols[i] for i in pay_pos]
        has_int = any(c.dtype == np.int64 for c in pay_cols)
        # a left row without a match gets NaN in every payload column, which turns a bool column into pandas' object
        # dtype: not on the device path.  Without misses, bool payload is gathered like any other column.
        has_bool = self.how == "left" and any(c.dtype == np.bool_ for c in pay_cols)
        if not unique:
            lrows, rrows, misses = ops.expand_matches(fact_keys, right.column(self.right_on), keep_misses=self.how == "left")
            if has_bool and misses:
                raise NotImplementedError(_BOOL_MISSES)
            promote = self.how == "left" and has_int and (self.promote_ints if self.promote_ints is not None else misses > 0)
            pay = ops.cast_columns_f64(pay_cols) if promote else pay_cols
            cols = ops.take_columns(left.cols, lrows) + ops.take_columns(pay, rrows)
            return DeviceBlock(cols, pandas.Index(ll + rl), nrows=len(lrows), range_start=0)
        if self.how == "left":
            promote = self.promote_ints
            if has_bool:
                idx, nmatch = table.probe(fact_keys)
                if promote or int(nmatch.item()) != left.nrows:
                    raise NotImplementedError(_BOOL_MISSES)
                return DeviceBlock(list(left.cols) + ops.take_columns(pay_cols, idx), pandas.Index(ll + rl),
                                   nrows=left.nrows, range_start=left.range_start)  # fmt: skip
            if has_int and promote is None:
                gathered, nmatch = table.probe_gather(fact_keys, pay_cols)
                promote = int(nmatch.item()) != left.nrows  # misses: pandas promotes int payload to float64 NaN
                if not promote:
                    return DeviceBlock(list(left.cols) + gathered, pandas.Index(ll + rl), nrows=left.nrows,
                                       range_start=left.range_start)  # fmt: skip
            if has_int and promote:
                idx, _ = table.probe(fact_keys)
                gathered = ops.take_columns(ops.cast_columns_f64(pay_cols), idx)
            else:
                gathered, _ = table.probe_gather(fact_keys, pay_cols)
            cols = list(left.cols) + gathered  # fact columns shared by reference
            return DeviceBlock(cols, pandas.Index(ll + rl), nrows=left.nrows, range_start=left.range_start)
        idx, _ = table.probe(fact_keys)
        pos, k = ops.compact_hits(idx)
        lcols = ops.take_columns(left.cols, pos)
        hit_idx = ops.take_columns([idx], pos)[0]
        rcols = ops.take_columns(pay_cols, hit_idx)
        return DeviceBlock(lcols + rcols, pandas.Index(ll + rl), nrows=k, range_start=0)


class DevMergePacked(DevMerge):
    """``DevMerge`` on SEVERAL int64 key columns (pandas.merge(on=[k1, k2, ...]), merge.py:139-168 per block): the
    left block's key tuples are packed into one order-preserving int64 (``groupkeys.pack``: one subtract + multiply
    per key column and k - 1 adds per row) with the plan that also packed the right frame, the single-key join runs
    on that image, and the image column is dropped from the result."""

    op = "merge_packed"

    def __init__(self, left_keys, plan, how="left", suffixes=("_x", "_y"), promote_ints=None, table_cache=None):
        from .groupkeys import PACKED_KEY

        super().__init__(how=how, suffixes=suffixes, left_on=PACKED_KEY, right_on=PACKED_KEY, promote_ints=promote_ints,
                         table_cache=table_cache)  # fmt: skip
        self.left_keys, self.plan = list(left_keys), plan

    def _with_image(self, left: DeviceBlock) -> DeviceBlock:
        from . import groupkeys as gk

        keys = DeviceBlock([left.column(k) for k in self.left_keys], pandas.Index(range(len(self.left_keys))), nrows=left.nrows)
        if any(c.dtype != np.int64 for c in keys.cols):
            raise NotImplementedError("device merge joins on int64 key columns")
        return left.with_cols(list(left.cols) + [gk.pack(keys, self.plan)], left.columns.append(pandas.Index([gk.PACKED_KEY])))

    def count_misses(self, left: DeviceBlock, right: DeviceBlock) -> int:
        return super().count_misses(self._with_image(left), right)

    def __call__(self, left, right, *args, **kwargs):
        from .groupkeys import PACKED_KEY

        _check_block(left, "DevMergePacked")
        out = super().__call__(self._with_image(left), right, *args, **kwargs)
        return out.select_columns([i for i, lab in enumerate(out.columns) if lab != PACKED_KEY])

