"""``modin_b200.pandas``: the pandas-API layer over the B200 query compiler.

A thin mirror of ``modin.pandas`` for the operations on the hot path, written the way the
reference's API layer is: every method validates arguments, forwards to
``self._query_compiler.<op>`` and wraps the resulting query compiler
(modin/pandas/base.py:485-542 ``_binary_op``, :660-665 ``abs``; modin/pandas/dataframe.py:2188-2247
``sum``, :484-603 ``groupby``, :1365-1403 ``merge``; modin/pandas/groupby.py:1330-1345, 1829-1886).

With real Modin installed, ``modin_b200.modin_plugin.register()`` plugs the same execution in
behind ``modin.pandas`` itself; this module is what runs where Modin is absent (the GPU box).
"""

from __future__ import annotations

import numbers
from typing import Optional

import numpy as np
import pandas

from ..functors import MODIN_UNNAMED_SERIES_LABEL
from ..dataframe import B200Dataframe
from ..query_compiler import B200QueryCompiler


def _is_scalar(x):
    return isinstance(x, (numbers.Number, np.number)) or np.isscalar(x)


class BasePandasDataset:
    _query_compiler: B200QueryCompiler

    # ---- plumbing --------------------------------------------------------------------------------
    def _create_or_update_from_compiler(self, new_query_compiler):
        return type(self)(query_compiler=new_query_compiler)

    def _validate_other(self, other):
        if isinstance(other, BasePandasDataset):
            return other._query_compiler
        return other

    def _binary_op(self, op, other, **kwargs):
        """modin/pandas/base.py:485-542."""
        other_qc = self._validate_other(other)
        if isinstance(other, Series) and isinstance(self, Series) and self.name != other.name:
            # Series (op) Series aligns on the row labels, not on the names; pandas drops the name when they differ
            unnamed = pandas.Index([MODIN_UNNAMED_SERIES_LABEL])
            new_qc = getattr(self._query_compiler.relabel_columns(unnamed), op)(other_qc.relabel_columns(unnamed), **kwargs)
            return self._create_or_update_from_compiler(new_qc)
        if isinstance(other, Series) and isinstance(self, DataFrame):
            if kwargs.get("axis") in (0, "index"):
                # frame (op) Series along the rows: a column vector co-partitioned with the frame -> the
                # broadcast_apply branch of Binary.caller (alg/binary.py:396-408)
                new_qc = getattr(self._query_compiler, op)(other_qc, broadcast=True, **kwargs)
                return self._create_or_update_from_compiler(new_qc)
            # along the columns == per-column scalars: hand the (W) values over as a row vector
            other_qc = other._to_pandas()
        new_qc = getattr(self._query_compiler, op)(other_qc, **kwargs)
        return self._create_or_update_from_compiler(new_qc)

    def _reduce_dimension(self, query_compiler):
        """1 x W frame -> pandas.Series (modin/pandas/dataframe.py ``_reduce_dimension``): the result of
        a reduction is small, so it is returned as a host ``pandas.Series``."""
        df = query_compiler.to_pandas()
        ser = df.iloc[0] if len(df) else pandas.Series(dtype="float64", index=df.columns)
        ser.name = None
        if len(set(df.dtypes)) == 1:
            ser = ser.astype(df.dtypes.iloc[0])
        return ser

    # ---- Map -------------------------------------------------------------------------------------
    def abs(self):
        return self._create_or_update_from_compiler(self._query_compiler.abs())

    def __abs__(self):
        return self.abs()

    def __neg__(self):
        return self._create_or_update_from_compiler(self._query_compiler.negative())

    def round(self, decimals=0, *args, **kwargs):
        return self._create_or_update_from_compiler(self._query_compiler.round(decimals=decimals))

    def drop_duplicates(self, subset=None, *, keep="first", inplace=False, ignore_index=False):
        """modin/pandas/base.py ``drop_duplicates`` -> qc.drop_duplicates; row order and row labels as pandas."""
        if inplace:
            raise NotImplementedError("drop_duplicates(inplace=True) is not on the B200 path")
        if isinstance(self, Series) and subset is not None:
            raise TypeError("Series.drop_duplicates() got an unexpected keyword argument 'subset'")
        qc = self._query_compiler.drop_duplicates(subset=subset, keep=keep, ignore_index=ignore_index)
        return self._create_or_update_from_compiler(qc)

    def astype(self, dtype, copy=None, errors="raise"):
        """modin/pandas/base.py ``astype`` -> qc.astype: one dtype for all columns, or {label: dtype}."""
        if isinstance(dtype, (pandas.Series, BasePandasDataset)):
            raise NotImplementedError("astype on the B200 path takes a dtype or a {column: dtype} dict")
        if isinstance(self, Series) and isinstance(dtype, dict):
            raise NotImplementedError("Series.astype on the B200 path takes a single dtype")
        return self._create_or_update_from_compiler(self._query_compiler.astype(dtype, errors=errors))

    def clip(self, lower=None, upper=None, *, axis=None, inplace=False, **kwargs):
        if inplace:
            raise NotImplementedError("clip(inplace=True) is not on the B200 path")
        return self._create_or_update_from_compiler(self._query_compiler.clip(lower=lower, upper=upper))

    def isin(self, values):
        if isinstance(values, (BasePandasDataset, pandas.Series, pandas.DataFrame, dict)):
            raise NotImplementedError("isin on the B200 path takes a list / array of integers")
        return self._create_or_update_from_compiler(self._query_compiler.isin(values))

    def isna(self):
        return self._create_or_update_from_compiler(self._query_compiler.isna())

    isnull = isna

    def notna(self):
        return self._create_or_update_from_compiler(self._query_compiler.notna())

    notnull = notna

    def fillna(self, value=None, *, method=None, axis=None, inplace=False, limit=None, downcast=None):
        if value is None and method is None:
            raise ValueError("Must specify a fill 'value' or 'method'.")
        if isinstance(value, (list, tuple)):
            raise TypeError(f'"value" parameter must be a scalar or dict, but you passed a "{type(value).__name__}"')
        if inplace:
            raise NotImplementedError("inplace=True is not supported by modin_b200.pandas")
        if isinstance(value, BasePandasDataset):
            value = value._query_compiler
        return self._create_or_update_from_compiler(
            self._query_compiler.fillna(value=value, method=method, axis=axis, limit=limit)
        )

    # ---- Binary ----------------------------------------------------------------------------------
    def add(self, other, axis="columns", level=None, fill_value=None):
        return self._binary_op("add", other, axis=axis, level=level, fill_value=fill_value)

    def radd(self, other, axis="columns", level=None, fill_value=None):
        return self._binary_op("radd", other, axis=axis, level=level, fill_value=fill_value)

    def sub(self, other, axis="columns", level=None, fill_value=None):
        return self._binary_op("sub", other, axis=axis, level=level, fill_value=fill_value)

    def rsub(self, other, axis="columns", level=None, fill_value=None):
        return self._binary_op("rsub", other, axis=axis, level=level, fill_value=fill_value)

    def mul(self, other, axis="columns", level=None, fill_value=None):
        return self._binary_op("mul", other, axis=axis, level=level, fill_value=fill_value)

    def rmul(self, other, axis="columns", level=None, fill_value=None):
        return self._binary_op("rmul", other, axis=axis, level=level, fill_value=fill_value)

    def truediv(self, other, axis="columns", level=None, fill_value=None):
        return self._binary_op("truediv", other, axis=axis, level=level, fill_value=fill_value)

    def rtruediv(self, other, axis="columns", level=None, fill_value=None):
        return self._binary_op("rtruediv", other, axis=axis, level=level, fill_value=fill_value)

    div = divide = truediv
    multiply = mul
    subtract = sub

    def eq(self, other, axis="columns", level=None):
        return self._binary_op("eq", other, axis=axis, level=level)

    def ne(self, other, axis="columns", level=None):
        return self._binary_op("ne", other, axis=axis, level=level)

    def lt(self, other, axis="columns", level=None):
        return self._binary_op("lt", other, axis=axis, level=level)

    def le(self, other, axis="columns", level=None):
        return self._binary_op("le", other, axis=axis, level=level)

    def gt(self, other, axis="columns", level=None):
        return self._binary_op("gt", other, axis=axis, level=level)

    def ge(self, other, axis="columns", level=None):
        return self._binary_op("ge", other, axis=axis, level=level)

    __add__ = lambda self, o: self.add(o)  # noqa: E731
    __radd__ = lambda self, o: self.radd(o)  # noqa: E731
    __sub__ = lambda self, o: self.sub(o)  # noqa: E731
    __rsub__ = lambda self, o: self.rsub(o)  # noqa: E731
    __mul__ = lambda self, o: self.mul(o)  # noqa: E731
    __rmul__ = lambda self, o: self.rmul(o)  # noqa: E731
    __truediv__ = lambda self, o: self.truediv(o)  # noqa: E731
    __rtruediv__ = lambda self, o: self.rtruediv(o)  # noqa: E731
    __eq__ = lambda self, o: self.eq(o)  # noqa: E731
    __ne__ = lambda self, o: self.ne(o)  # noqa: E731
    __lt__ = lambda self, o: self.lt(o)  # noqa: E731
    __le__ = lambda self, o: self.le(o)  # noqa: E731
    __gt__ = lambda self, o: self.gt(o)  # noqa: E731
    __ge__ = lambda self, o: self.ge(o)  # noqa: E731
    __hash__ = None

    # ---- logical ops on bool frames (what comparisons produce) --------------------------------------
    __and__ = lambda self, o: self._binary_op("__and__", o)  # noqa: E731
    __or__ = lambda self, o: self._binary_op("__or__", o)  # noqa: E731
    __xor__ = lambda self, o: self._binary_op("__xor__", o)  # noqa: E731

    def __invert__(self):
        return self._create_or_update_from_compiler(self._query_compiler.invert())

    def any(self, axis=0, bool_only=False, skipna=True, **kwargs):
        return self._stat("any", axis, skipna, False)

    def all(self, axis=0, bool_only=False, skipna=True, **kwargs):
        return self._stat("all", axis, skipna, False)

    # ---- TreeReduce --------------------------------------------------------------------------------
    def _stat(self, name, axis=0, skipna=True, numeric_only=False, **kwargs):
        if axis not in (0, "index", None):
            raise NotImplementedError(f"{name}(axis=1) is not on the B200 path")
        qc = getattr(self._query_compiler, name)(axis=0, skipna=skipna, numeric_only=numeric_only, **kwargs)
        return self._reduce_dimension(qc)

    def sum(self, axis=0, skipna=True, numeric_only=False, min_count=0, **kwargs):
        return self._stat("sum", axis, skipna, numeric_only, min_count=min_count)

    def prod(self, axis=0, skipna=True, numeric_only=False, min_count=0, **kwargs):
        if min_count:
            raise NotImplementedError("prod(min_count>0) is not on the B200 path")
        return self._stat("prod", axis, skipna, numeric_only)

    product = prod

    def mean(self, axis=0, skipna=True, numeric_only=False, **kwargs):
        return self._stat("mean", axis, skipna, numeric_only)

    def var(self, axis=0, skipna=True, ddof=1, numeric_only=False, **kwargs):
        """modin/pandas/base.py ``var`` -> ``_stat_operation``; two device passes (mean, squared deviations)."""
        if axis not in (0, "index", None):
            raise NotImplementedError("var(axis=1) is not on the B200 path")
        return self._finish_host_stat(self._query_compiler.var(axis=0, skipna=skipna, ddof=ddof, numeric_only=numeric_only))

    def std(self, axis=0, skipna=True, ddof=1, numeric_only=False, **kwargs):
        if axis not in (0, "index", None):
            raise NotImplementedError("std(axis=1) is not on the B200 path")
        return self._finish_host_stat(self._query_compiler.std(axis=0, skipna=skipna, ddof=ddof, numeric_only=numeric_only))

    def _finish_host_stat(self, ser):
        ser.name = None
        return ser

    def min(self, axis=0, skipna=True, numeric_only=False, **kwargs):
        return self._stat("min", axis, skipna, numeric_only)

    def max(self, axis=0, skipna=True, numeric_only=False, **kwargs):
        return self._stat("max", axis, skipna, numeric_only)

    def count(self, axis=0, numeric_only=False):
        if axis not in (0, "index", None):
            raise NotImplementedError("count(axis=1) is not on the B200 path")
        return self._reduce_dimension(self._query_compiler.count(axis=0, numeric_only=numeric_only))

    # ---- Reduce: label of the first extreme value (modin/pandas/base.py ``idxmax`` / ``idxmin``) ----------------
    def _arg_stat(self, name, axis, skipna, numeric_only):
        if axis not in (0, "index", None):
            raise NotImplementedError(f"{name}(axis=1) is not on the B200 path")
        if not len(self._query_compiler.columns):
            return pandas.Series([], index=self._query_compiler.columns, dtype=np.int64)
        return self._reduce_dimension(getattr(self._query_compiler, name)(axis=0, skipna=skipna, numeric_only=numeric_only))

    def idxmax(self, axis=0, skipna=True, numeric_only=False):
        return self._arg_stat("idxmax", axis, skipna, numeric_only)

    def idxmin(self, axis=0, skipna=True, numeric_only=False):
        return self._arg_stat("idxmin", axis, skipna, numeric_only)

    # ---- misc --------------------------------------------------------------------------------------
    def _to_pandas(self):
        return self._query_compiler.to_pandas()

    def to_numpy(self, **kwargs):
        return self._query_compiler.to_numpy(**kwargs)

    def execute(self):
        """modin.utils.execute (modin/utils.py:740-753): drain call queues and wait for the device."""
        self._query_compiler.execute()
        return self

    @property
    def dtypes(self):
        return self._query_compiler.dtypes


class DataFrame(BasePandasDataset):
    """modin.pandas.DataFrame for the hot path (modin/pandas/dataframe.py:147-266 constructor)."""

    def __init__(self, data=None, index=None, columns=None, dtype=None, copy=None, query_compiler=None):
        if query_compiler is not None:
            self._query_compiler = query_compiler
            return
        if isinstance(data, DataFrame):
            self._query_compiler = data._query_compiler
            return
        if not isinstance(data, pandas.DataFrame) or index is not None or columns is not None or dtype is not None:
            data = pandas.DataFrame(data=data, index=index, columns=columns, dtype=dtype)
        self._query_compiler = B200QueryCompiler.from_pandas(data)

    # metadata
    columns = property(lambda self: self._query_compiler.columns)
    index = property(lambda self: self._query_compiler.index)
    shape = property(lambda self: (self._query_compiler.get_axis_len(0), len(self.columns)))

    def __len__(self):
        return self._query_compiler.get_axis_len(0)

    # ---- structure (metadata only: buffers are shared, nothing is copied or launched) --------------------------
    def copy(self, deep=True):
        return DataFrame(query_compiler=self._query_compiler)  # blocks are immutable values

    def __setitem__(self, key, value):
        """``df["d"] = df["a"] * 2`` -- a co-partitioned Series (or one-column frame) becomes / replaces a column."""
        if isinstance(key, (list, tuple)):
            raise NotImplementedError("assigning several columns at once is not on the B200 path")
        if isinstance(value, (Series, DataFrame)):
            vqc = value._query_compiler
            if len(vqc.columns) != 1:
                raise ValueError("Cannot set a DataFrame with multiple columns to the single column " + str(key))
        else:
            raise NotImplementedError("column assignment on the B200 path takes a device Series")
        self._query_compiler = self._query_compiler.set_column(key, vqc)

    def assign(self, **kwargs):
        out = self.copy()
        for k, v in kwargs.items():
            out[k] = v(out) if callable(v) else v
        return out

    def drop(self, labels=None, *, axis=0, index=None, columns=None, inplace=False, errors="raise", **kwargs):
        if inplace or index is not None or (labels is not None and axis in (0, "index")):
            raise NotImplementedError("drop on the B200 path removes columns")
        cols = columns if columns is not None else labels
        cols = [cols] if not isinstance(cols, (list, tuple, pandas.Index)) else list(cols)
        missing = [c for c in cols if c not in self.columns]
        if missing and errors == "raise":
            raise KeyError(f"{missing} not found in axis")
        return self[[c for c in self.columns if c not in cols]]

    def rename(self, mapper=None, *, columns=None, axis=None, inplace=False, **kwargs):
        if inplace or (mapper is not None and axis not in (1, "columns")) or kwargs.get("index") is not None:
            raise NotImplementedError("rename on the B200 path renames columns")
        mapping = columns if columns is not None else mapper
        new = [mapping(c) if callable(mapping) else mapping.get(c, c) for c in self.columns]
        return DataFrame(query_compiler=self._query_compiler.relabel_columns(new))

    def head(self, n=5):
        return DataFrame(query_compiler=self._query_compiler.head(n))

    def tail(self, n=5):
        return DataFrame(query_compiler=self._query_compiler.tail(n))

    def nunique(self, axis=0, dropna=True):
        """Distinct values per column: one device group table per column, the answer is its row count.  int64
        columns only -- a float column would need pandas' NaN handling (``dropna``), which the group tables do not
        have.  The W counts come back as a host Series, like the other column reductions."""
        if axis not in (0, "index"):
            raise NotImplementedError("nunique(axis=1) is not on the B200 path")
        bad = [c for c, dt in zip(self.columns, self.dtypes) if np.dtype(dt) != np.int64]
        if bad:
            raise NotImplementedError(f"nunique on the B200 path counts int64 columns only (got {bad!r})")
        counts = [self[c].nunique() for c in self.columns]
        return pandas.Series(counts, index=self.columns, dtype=np.int64)

    def dropna(self, *, axis=0, how="any", subset=None, inplace=False, ignore_index=False, **kwargs):
        """Drop rows with missing values: ``notna()`` -> row-wise all / any -> boolean row selection, all on the
        device (the reference: qc.dropna, a full-axis apply of ``pandas.DataFrame.dropna``)."""
        if axis not in (0, "index") or inplace or ignore_index or kwargs.get("thresh") is not None:
            raise NotImplementedError("dropna on the B200 path: rows only, how='any'|'all', optional subset")
        if how not in ("any", "all"):
            raise ValueError(f"invalid how option: {how}")
        cols = list(self.columns) if subset is None else ([subset] if not isinstance(subset, (list, tuple)) else list(subset))
        probe = self[cols].notna()._query_compiler
        keep = probe.row_all() if how == "any" else probe.row_any()
        return DataFrame(query_compiler=self._query_compiler.getitem_row_mask(keep))

    def __getitem__(self, key):
        if isinstance(key, Series) or (isinstance(key, DataFrame) and len(key.columns) == 1 and
                                       key._query_compiler.dtypes.iloc[0] == np.bool_):  # fmt: skip
            # boolean row selection: df[df["c0"] > 0]
            if key._query_compiler.dtypes.iloc[0] != np.bool_:
                raise NotImplementedError("indexing a frame with a non-bool Series is not on the B200 path")
            return DataFrame(query_compiler=self._query_compiler.getitem_row_mask(key._query_compiler))
        if isinstance(key, (list, pandas.Index, np.ndarray)):
            return DataFrame(query_compiler=self._query_compiler.getitem_column_array(list(key)))
        if key not in self.columns:
            raise KeyError(key)
        qc = self._query_compiler.getitem_column_array([key])
        return Series(query_compiler=qc)

    def groupby(self, by=None, axis=0, level=None, as_index=True, sort=True, group_keys=True, observed=True,
                dropna=True):  # fmt: skip
        """modin/pandas/dataframe.py:484-603: a column label resolves to ``self[by]``'s query compiler
        with ``drop=True``."""
        if axis not in (0, "index"):
            raise NotImplementedError("groupby(axis=1) is not on the B200 path")
        if level is not None:
            raise NotImplementedError("groupby(level=) is not on the B200 path")
        for key, value, allowed in (("as_index", as_index, (True, False)), ("observed", observed, (True, False, None))):
            if value not in allowed:
                raise NotImplementedError(f"groupby({key}={value!r}) is not on the B200 path")
        kwargs = dict(as_index=as_index, sort=sort, group_keys=group_keys, observed=observed, dropna=dropna, level=level)
        if isinstance(by, (list, tuple)) and len(by) != 1:
            # several int64 keys: the query compiler groups by their packed image, and drops the key columns
            for k in by:
                if k not in self.columns:
                    raise KeyError(k)
            if len(set(by)) != len(by):
                raise ValueError("duplicate key columns")
            if any(np.dtype(self.dtypes[k]) != np.int64 for k in by):
                raise NotImplementedError("multi-column groupby on the B200 path needs int64 key columns")
            return DataFrameGroupBy(self, self._query_compiler.getitem_column_array(list(by)), drop=True,
                                    groupby_kwargs=kwargs)  # fmt: skip
        if isinstance(by, (list, tuple)):
            by = by[0]
        drop = False
        if isinstance(by, Series):
            by_qc = by._query_compiler
        elif isinstance(by, str) or not callable(by):
            if by not in self.columns:
                raise KeyError(by)
            by_qc = self[by]._query_compiler
            drop = True
        else:
            raise NotImplementedError("callable `by` is not on the B200 path")
        return DataFrameGroupBy(self, by_qc, drop=drop,
                                groupby_kwargs=dict(as_index=as_index, sort=sort, group_keys=group_keys,
                                                    observed=observed, dropna=dropna, level=level))  # fmt: skip

    def sort_values(self, by, *, axis=0, ascending=True, inplace=False, kind="quicksort", na_position="last",
                    ignore_index=False, key=None):  # fmt: skip
        """modin/pandas/base.py ``sort_values`` -> ``qc.sort_rows_by_column_values``."""
        if axis not in (0, "index"):
            raise NotImplementedError("sort_values(axis=1) is not on the B200 path")
        if inplace:
            raise NotImplementedError("sort_values(inplace=True) is not on the B200 path")
        qc = self._query_compiler.sort_rows_by_column_values(by, ascending=ascending, kind=kind, na_position=na_position,
                                                             ignore_index=ignore_index, key=key)  # fmt: skip
        return DataFrame(query_compiler=qc)

    def merge(self, right, how="inner", on=None, left_on=None, right_on=None, left_index=False, right_index=False,
              sort=False, suffixes=("_x", "_y"), copy=None, indicator=False, validate=None):  # fmt: skip
        """modin/pandas/dataframe.py:1365-1403."""
        if isinstance(right, Series):
            raise NotImplementedError("merging with a Series is not on the B200 path")
        if not isinstance(right, DataFrame):
            raise TypeError(f"Can only merge Series or DataFrame objects, a {type(right)} was passed")
        if indicator or validate is not None or sort:
            raise NotImplementedError("merge(indicator=/validate=/sort=True) is not on the B200 path")
        return DataFrame(
            query_compiler=self._query_compiler.merge(
                right._query_compiler, how=how, on=on, left_on=left_on, right_on=right_on, left_index=left_index,
                right_index=right_index, sort=sort, suffixes=suffixes,
            )
        )  # fmt: skip

    def __repr__(self):
        return f"<modin_b200.pandas.DataFrame shape={self.shape} columns={list(self.columns)!r}>"


class Series(BasePandasDataset):
    """One-column frame viewed as a Series (modin/pandas/series.py keeps a 1-column query compiler)."""

    def __init__(self, data=None, index=None, name=None, query_compiler=None):
        if query_compiler is not None:
            self._query_compiler = query_compiler
            return
        ser = data if isinstance(data, pandas.Series) else pandas.Series(data, index=index, name=name)
        label = ser.name if ser.name is not None else MODIN_UNNAMED_SERIES_LABEL
        self._query_compiler = B200QueryCompiler.from_pandas(ser.to_frame(label))

    @property
    def name(self):
        label = self._query_compiler.columns[0]
        return None if label == MODIN_UNNAMED_SERIES_LABEL else label

    def __len__(self):
        return self._query_compiler.get_axis_len(0)

    def _to_pandas(self):
        df = self._query_compiler.to_pandas()
        ser = df.iloc[:, 0]
        ser.name = self.name
        return ser

    def _reduce_dimension(self, query_compiler):
        res = super()._reduce_dimension(query_compiler)
        return res.iloc[0]

    def _finish_host_stat(self, ser):
        return ser.iloc[0]

    # ---- the frame surface that only re-wraps: a Series is a one-column frame, so these delegate to it -----------
    @property
    def dtype(self):
        return self._query_compiler.dtypes.iloc[0]

    def _as_frame(self) -> "DataFrame":
        return DataFrame(query_compiler=self._query_compiler)

    @staticmethod
    def _of(frame: "DataFrame") -> "Series":
        return Series(query_compiler=frame._query_compiler)

    def head(self, n=5):
        return self._of(self._as_frame().head(n))

    def tail(self, n=5):
        return self._of(self._as_frame().tail(n))

    def copy(self, deep=True):
        return self._of(self._as_frame().copy())

    def dropna(self, *, axis=0, inplace=False, how=None, ignore_index=False):
        if inplace or ignore_index or axis not in (0, "index"):
            raise NotImplementedError("Series.dropna(inplace= / ignore_index= / axis=1) is not on the B200 path")
        return self._of(self._as_frame().dropna())

    def sort_values(self, *, axis=0, ascending=True, inplace=False, kind="quicksort", na_position="last",
                    ignore_index=False, key=None):  # fmt: skip
        if inplace:
            raise NotImplementedError("sort_values(inplace=True) is not on the B200 path")
        label = self._query_compiler.columns[0]
        return self._of(self._as_frame().sort_values(label, axis=axis, ascending=ascending, kind=kind, na_position=na_position,
                                                     ignore_index=ignore_index, key=key))  # fmt: skip

    def rename(self, index=None, **kwargs):
        """``Series.rename(name)``: a new name over the same buffer (relabelling the row labels is not on the path)."""
        if kwargs or callable(index) or isinstance(index, dict):
            raise NotImplementedError("Series.rename on the B200 path only changes the name")
        label = MODIN_UNNAMED_SERIES_LABEL if index is None else index
        return Series(query_compiler=self._query_compiler.relabel_columns([label]))

    def argmax(self, axis=None, skipna=True, *args, **kwargs):
        """Position of the first largest value: ``idxmax`` over the rows renumbered 0..n-1, as modin/pandas/series.py
        ``argmax`` does with ``reset_index(drop=True)`` (metadata only, no copy)."""
        return self._positions().idxmax(skipna=skipna)

    def argmin(self, axis=None, skipna=True, *args, **kwargs):
        return self._positions().idxmin(skipna=skipna)

    def _positions(self) -> "Series":
        from ..query_compiler import _reset_row_index

        return Series(query_compiler=self._query_compiler.__constructor__(_reset_row_index(self._query_compiler._modin_frame)))

    def __getitem__(self, key):
        """``s[bool_series]``: boolean row selection, as on a frame."""
        if isinstance(key, Series):
            return self._of(self._as_frame()[key])
        raise NotImplementedError("indexing a Series on the B200 path takes a bool Series")

    # ---- distinct values of an int64 Series, through the group tables (qc.py:1109-1142 nunique / unique; the
    # reference's range-partitioning variants are built on the same shuffle as sort_values) ----------------------
    def _as_key_frame(self):
        label = self._query_compiler.columns[0]
        return DataFrame(query_compiler=self._query_compiler), label

    def nunique(self, dropna=True):
        """Number of distinct values = number of groups (int64 values only; int64 holds no NaN)."""
        df, label = self._as_key_frame()
        frame = df.groupby(label).size()._query_compiler._modin_frame
        return int(frame.global_nrows)

    def value_counts(self, normalize=False, sort=True, ascending=False, bins=None, dropna=True):
        """``Series.value_counts`` (modin/pandas/base.py -> qc.value_counts): group sizes keyed by value, most
        frequent first.  Ties come out in ascending value order (pandas leaves tie order unspecified)."""
        if normalize or bins is not None:
            raise NotImplementedError("value_counts(normalize= / bins=) is not on the B200 path")
        df, label = self._as_key_frame()
        sizes = df.groupby(label).size()  # Series over the group keys
        if not sort:
            return sizes
        frame = DataFrame(query_compiler=sizes._query_compiler).sort_values(sizes._query_compiler.columns[0],
                                                                            ascending=ascending)  # fmt: skip
        return Series(query_compiler=frame._query_compiler)


class DataFrameGroupBy:
    """modin/pandas/groupby.py (``_wrap_aggregation`` :1829-1886)."""

    def __init__(self, df: DataFrame, by_qc, drop, groupby_kwargs):
        self._df = df
        self._query_compiler = df._query_compiler
        self._by = by_qc
        self._drop = drop
        self._kwargs = groupby_kwargs

    def _check_keys(self):
        if len(self._by.columns) == 1 and self._by.dtypes.iloc[0] == np.float64:  # float keys are not on this front door
            raise NotImplementedError("device groupby needs an int64 key column")

    def _wrap_aggregation(self, qc_method, numeric_only=False, agg_args=None, agg_kwargs=None):
        self._check_keys()
        result_qc = qc_method(self._query_compiler, by=self._by, axis=0, groupby_kwargs=self._kwargs,
                              agg_args=agg_args or [], agg_kwargs=agg_kwargs or {}, drop=self._drop)  # fmt: skip
        return DataFrame(query_compiler=result_qc)

    def sum(self, numeric_only=False, min_count=0):
        if min_count:
            raise NotImplementedError("groupby.sum(min_count>0) is not on the B200 path")
        return self._wrap_aggregation(type(self._query_compiler).groupby_sum, numeric_only)

    def count(self):
        return self._wrap_aggregation(type(self._query_compiler).groupby_count)

    def mean(self, numeric_only=False):
        return self._wrap_aggregation(type(self._query_compiler).groupby_mean, numeric_only)

    def min(self, numeric_only=False, min_count=-1):
        return self._wrap_aggregation(type(self._query_compiler).groupby_min, numeric_only)

    def max(self, numeric_only=False, min_count=-1):
        return self._wrap_aggregation(type(self._query_compiler).groupby_max, numeric_only)

    def first(self, numeric_only=False, min_count=-1, skipna=True):
        """The first non-NaN value of every column per group (every row's value under ``skipna=False``), passed on as
        modin/pandas/groupby.py:904-915 does."""
        return self._wrap_aggregation(type(self._query_compiler).groupby_first, numeric_only,
                                      agg_kwargs=dict(min_count=min_count, skipna=skipna))  # fmt: skip

    def last(self, numeric_only=False, min_count=-1, skipna=True):
        return self._wrap_aggregation(type(self._query_compiler).groupby_last, numeric_only,
                                      agg_kwargs=dict(min_count=min_count, skipna=skipna))  # fmt: skip

    def idxmax(self, skipna=True, numeric_only=False):
        """The label of the first row holding each group's maximum, per column (NaN skipped; a group whose values in a
        column are all NaN raises ValueError), passed on as modin/pandas/groupby.py:607-618 does."""
        return self._wrap_aggregation(type(self._query_compiler).groupby_idxmax, numeric_only,
                                      agg_kwargs=dict(axis=0, skipna=skipna))  # fmt: skip

    def idxmin(self, skipna=True, numeric_only=False):
        return self._wrap_aggregation(type(self._query_compiler).groupby_idxmin, numeric_only,
                                      agg_kwargs=dict(axis=0, skipna=skipna))  # fmt: skip

    def var(self, ddof=1, engine=None, engine_kwargs=None, numeric_only=False):
        """The sample variance of every column per group (NaN skipped; NaN where a group has ``ddof`` values or
        fewer), passed on as modin/pandas/groupby.py:1264-1278 does.  Only pandas' own engine."""
        if engine not in ("cython", None) or engine_kwargs is not None:
            raise NotImplementedError(f"groupby.var(engine={engine!r}) is not on the B200 path")
        return self._wrap_aggregation(type(self._query_compiler).groupby_var, numeric_only, agg_kwargs=dict(ddof=ddof))

    def std(self, ddof=1, engine=None, engine_kwargs=None, numeric_only=False):
        if engine not in ("cython", None) or engine_kwargs is not None:
            raise NotImplementedError(f"groupby.std(engine={engine!r}) is not on the B200 path")
        return self._wrap_aggregation(type(self._query_compiler).groupby_std, numeric_only, agg_kwargs=dict(ddof=ddof))

    def nunique(self, dropna=True):
        """The number of distinct values of every column per group (int64; NaN left out under ``dropna``, else counted
        once), passed on as modin/pandas/groupby.py:1399-1406 does."""
        return self._wrap_aggregation(type(self._query_compiler).groupby_nunique, agg_kwargs=dict(dropna=dropna))

    def size(self):
        res = self._wrap_aggregation(type(self._query_compiler).groupby_size)
        return Series(query_compiler=res._query_compiler)

    def agg(self, func, *args, **kwargs):
        if isinstance(func, str) and func in ("var", "std", "nunique") and not args:
            return getattr(self, func)(**kwargs)
        if isinstance(func, str) and func in ("sum", "count", "mean", "size", "min", "max", "first", "last", "idxmax",
                                                 "idxmin"):
            return getattr(self, func)()
        if isinstance(func, dict):
            return self._dict_agg(func)
        raise NotImplementedError(f"groupby.agg({func!r}) is not on the B200 path")

    def _dict_agg(self, spec):
        """``groupby(key).agg({column: function})`` -- qc._groupby_dict_reduce (qc.py:3876-3970) splits a dictionary
        aggregation into per-function map / reduce tables.  Here: one device aggregation per distinct function over
        the columns that ask for it, zipped column-wise in the dictionary's order (``qc.groupby_agg``)."""
        if not self._drop:
            raise NotImplementedError("dictionary aggregation needs the key column inside the frame")
        self._check_keys()
        return DataFrame(query_compiler=self._query_compiler.groupby_agg(self._by, spec, 0, self._kwargs, (), {},
                                                                         drop=self._drop))  # fmt: skip

    aggregate = agg


def concat(objs, *, axis=0, join="outer", ignore_index=False, **kwargs):
    """``pandas.concat`` of device frames (modin/pandas/general.py ``concat`` -> qc.concat -> PandasDataframe.concat,
    df.py:3952-4096) for the two shapes that need no label alignment: rows of frames with identical columns
    (axis=0: the row partitions are simply lined up, buffers shared) and columns of frames with identical rows and
    distinct labels (axis=1: ``hstack``)."""
    from .. import dist
    from ..dataframe import B200Dataframe

    objs = list(objs)
    if not objs or not all(isinstance(o, DataFrame) for o in objs):
        raise NotImplementedError("concat on the B200 path takes a list of device DataFrames")
    if axis in (1, "columns"):
        # PandasDataframe.concat(axis=1) (df.py:3952-4096) co-partitions the frames along the rows first: the row
        # labels are joined (outer, in order of appearance -- pandas.concat does not sort) and frames whose labels
        # differ are re-indexed on the device
        if join != "outer":
            raise NotImplementedError("concat(axis=1, join='inner') is not on the B200 path")
        frames = [o._query_compiler._modin_frame for o in objs]
        frame, rest = frames[0]._copartition_rows(frames[1:], how="outer", sort=False)
        for o in rest:
            frame = frame.hstack(o)
        return DataFrame(query_compiler=type(objs[0]._query_compiler)(frame))
    if axis not in (0, "index"):
        raise ValueError(f"No axis named {axis}")
    if dist.is_distributed():
        raise NotImplementedError("row-wise concat of sharded frames would interleave the shards; not on the B200 path")
    cols = objs[0].columns
    for o in objs[1:]:
        if not o.columns.equals(cols):
            raise NotImplementedError("row-wise concat on the B200 path needs identical column labels")
        if list(o.dtypes) != list(objs[0].dtypes):  # pandas would promote; shared buffers cannot
            raise NotImplementedError("row-wise concat on the B200 path needs identical column dtypes")
    from ..block import DeviceBlock, concat_cols

    first = objs[0]._query_compiler._modin_frame
    pc = first._partition_mgr_cls._partition_class
    blocks, pos = [], 0
    for o in objs:
        f = o._query_compiler._modin_frame
        if len(f) == 0:
            continue
        for row in f._partitions:
            b = concat_cols([p.get() for p in row]) if len(row) > 1 else row[0].get()
            if ignore_index:  # fresh 0..n labels; the column buffers are shared, not copied
                b = DeviceBlock(b.cols, b.columns, nrows=b.nrows, range_start=pos)
            blocks.append(b)
            pos += b.nrows
    if not blocks:
        return objs[0].copy()
    # from_blocks assumes the blocks' range labels run on from each other, which only holds after ignore_index;
    # otherwise leave the index cache empty so the labels are read from the blocks (each keeps its own)
    index = pandas.RangeIndex(0, pos) if ignore_index else None
    parts = np.array([[pc.put(b)] for b in blocks], dtype=object)
    frame = B200Dataframe(parts, index, cols, [b.nrows for b in blocks], [len(cols)], dtypes=None)
    return DataFrame(query_compiler=type(objs[0]._query_compiler)(frame))


# ---- zero-copy interchange with other GPU libraries (SURVEY 8f-1: DLPack; the reference's wire format for
# this is the dataframe interchange protocol, df.py:4803-4867, whose buffers also export __dlpack__) -------------
def from_dlpack(columns: dict, range_start: int = 0) -> DataFrame:
    """Frame over device buffers owned by another library: ``{label: object with __dlpack__ (or a torch tensor)}``,
    1-D contiguous float64 / int64 / bool of equal length on this process's GPU.  Nothing is copied; the frame is
    ONE row partition (this rank's shard under torchrun)."""
    import torch

    from ..block import DeviceBlock, DeviceColumn, current_device
    from ..dataframe import B200Dataframe

    dev = current_device()
    cols, labels, n = [], [], None
    for label, obj in columns.items():
        ten = obj if isinstance(obj, torch.Tensor) else torch.from_dlpack(obj)
        if ten.dim() != 1 or not ten.is_contiguous():
            raise ValueError(f"column {label!r}: need a 1-D contiguous buffer")
        if ten.device != dev:
            raise ValueError(f"column {label!r} lives on {ten.device}, this process computes on {dev}")
        np_dtype = {torch.float64: np.float64, torch.int64: np.int64, torch.bool: np.bool_, torch.uint8: np.bool_}.get(ten.dtype)
        if np_dtype is None:
            raise TypeError(f"column {label!r}: dtype {ten.dtype} is not on the B200 path (float64 / int64 / bool)")
        if ten.dtype == torch.bool:
            ten = ten.view(torch.uint8)
        if n is None:
            n = ten.shape[0]
        elif ten.shape[0] != n:
            raise ValueError("columns of different lengths")
        cols.append(DeviceColumn(ten, np.dtype(np_dtype)))
        labels.append(label)
    block = DeviceBlock(cols, pandas.Index(labels), nrows=n or 0, range_start=range_start)
    return DataFrame(query_compiler=B200QueryCompiler(B200Dataframe.from_blocks([block])))


def to_dlpack(df: DataFrame) -> dict:
    """``{label: torch tensor}`` views of the frame's device buffers (each exports ``__dlpack__``).  Zero-copy
    for a frame with one row partition; several row partitions are concatenated on the device first."""
    from ..block import concat_cols, concat_rows

    frame = df._query_compiler._modin_frame
    rows = [concat_cols([p.get() for p in row]) if len(row) > 1 else row[0].get() for row in frame._partitions]
    block = concat_rows(rows) if len(rows) > 1 else rows[0]
    import torch

    out = {}
    for label, c in zip(block.columns, block.cols):
        out[label] = c.data.view(torch.bool) if c.dtype == np.bool_ else c.data
    return out
