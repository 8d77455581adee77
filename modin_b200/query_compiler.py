"""The device surface both query compilers share, and ``B200QueryCompiler``, the Modin-free one that holds a
``B200Dataframe``.

``device_operations(alg)`` returns the one definition of every device operation: the Map / Binary / TreeReduce /
Reduce / Fold registrations with their device functors, ``fillna`` / ``astype`` / ``merge``, and the groupby
aggregations.  ``alg`` is the module of operator templates the registrations go through: ``modin_b200.algebra`` for
the mirror below, ``modin.core.dataframe.algebra`` for the Modin plug-in (``modin_plugin.py``), whose query compiler
puts the class in front of ``PandasQueryCompiler`` so that these entries replace Modin's.

Reference registrations being mirrored (modin/core/storage_formats/pandas/query_compiler.py):
Binary ops ``:535-624``; ``count/sum/max/min/mean`` TreeReduce ``:976-1096``; ``abs`` ``:2036``;
``isna/notna/negative`` ``:2063-2106``; ``fillna`` ``:2710-2813``; ``groupby_*`` ``:3741-3748``
with GroupbyReduceImpl (storage_formats/pandas/groupby.py:26-248); ``merge`` ``:657-667`` with
MergeImpl.row_axis_merge (merge.py:104-252).

Operations outside this list raise ``NotImplementedError`` instead of defaulting to pandas: the
north-star forbids a CPU fallback on this path, and a silent D2H -> pandas -> H2D round trip would
hide exactly the cost this backend exists to remove.
"""

from __future__ import annotations

import numpy as np
import pandas

from . import algebra, dist
from . import groupkeys as gk
from .block import concat_cols
from .dataframe import B200Dataframe
from .functors import (
    arg_label_dtype,
    DevArgReduce,
    DevAstype,
    DevBinary,
    DevBoolReduce,
    DevClip,
    DevCumulative,
    DevFillna,
    DevGroupbyMap,
    DevGroupbyReduce,
    DevLogical,
    DevMap,
    DevMeanMap,
    DevMeanReduce,
    DevReduce,
    DevRound,
    DevVar,
    groupby_nunique,
)


def _dtypes_sum(dtypes: pandas.Series, *func_args, **func_kwargs):
    """qc.py:961-974: result dtype of sum = common type of the columns."""
    return np.result_type(*dtypes.values) if len(dtypes) else np.dtype("float64")


def _position_agg_skipna(agg: str, agg_kwargs) -> bool:
    """``skipna`` of ``groupby.first`` / ``last`` from the ``agg_kwargs`` Modin passes (modin/pandas/groupby.py:904-915).
    ``min_count`` of -1, 0 or 1 leaves the result as it is (every group has a row); a larger one makes pandas put NaN
    into groups with fewer values and change the dtypes of int64 / bool columns, which is not on the device path."""
    kw = dict(agg_kwargs or {})
    skipna, min_count = kw.pop("skipna", True), kw.pop("min_count", -1)
    if kw:
        raise NotImplementedError(f"groupby.{agg}({', '.join(kw)}=) is not on the B200 path")
    if not isinstance(skipna, (bool, np.bool_)):
        raise ValueError(f"skipna must be a boolean, got {skipna!r}")
    if min_count not in (-1, 0, 1):
        raise NotImplementedError(f"groupby.{agg}(min_count={min_count!r}) is not on the B200 path")
    return bool(skipna)


def _arg_agg_kwargs(agg: str, agg_kwargs) -> None:
    """``groupby.idxmax`` / ``idxmin`` take ``skipna=True`` and ``axis=0`` from the ``agg_kwargs`` Modin passes
    (modin/pandas/groupby.py:607-631).  ``skipna=False`` is refused: pandas 3.0.2 raises there when a NaN is present
    anywhere, even in a row whose key is dropped, and otherwise returns NaN for every group."""
    kw = dict(agg_kwargs or {})
    skipna, axis = kw.pop("skipna", True), kw.pop("axis", 0)
    kw.pop("numeric_only", None)
    if kw:
        raise NotImplementedError(f"groupby.{agg}({', '.join(kw)}=) is not on the B200 path")
    if not isinstance(skipna, (bool, np.bool_)):
        raise ValueError(f"skipna must be a boolean, got {skipna!r}")
    if not skipna:
        raise NotImplementedError(f"groupby.{agg}(skipna=False) is not on the B200 path")
    if axis not in (0, "index", None):
        raise NotImplementedError(f"groupby.{agg}(axis={axis!r}) is not on the B200 path")


def _var_ddof(agg: str, agg_kwargs):
    """``ddof`` of ``groupby.var`` / ``std`` from the ``agg_kwargs`` Modin passes (modin/pandas/groupby.py:1264-1278),
    truncated towards zero as pandas does.  ``numeric_only`` is dropped (the caller has selected the columns); any
    other argument, such as another engine, is refused."""
    kw = dict(agg_kwargs or {})
    ddof = kw.pop("ddof", 1)
    kw.pop("numeric_only", None)
    if kw.get("engine") in ("cython", None) and kw.get("engine_kwargs") is None:  # pandas' own engine
        kw.pop("engine", None)
        kw.pop("engine_kwargs", None)
    if kw:
        raise NotImplementedError(f"groupby.{agg}({', '.join(kw)}=) is not on the B200 path")
    if not isinstance(ddof, (int, float, np.integer, np.floating)):
        raise TypeError(f"ddof must be a number, got {ddof!r}")
    return int(ddof)  # pandas 3.0.2's group_var takes ddof as an integer: 1.5 acts as 1, -0.5 as 0


def _nunique_dropna(agg_kwargs) -> bool:
    """``dropna`` of ``groupby.nunique`` from the ``agg_kwargs`` Modin passes (modin/pandas/groupby.py:1399-1406): whether
    NaN is left out of the count.  Any other argument is refused."""
    kw = dict(agg_kwargs or {})
    dropna = kw.pop("dropna", True)
    if kw:
        raise NotImplementedError(f"groupby.nunique({', '.join(kw)}=) is not on the B200 path")
    if not isinstance(dropna, (bool, np.bool_)):
        raise ValueError(f"dropna must be a boolean, got {dropna!r}")
    return bool(dropna)


def _nunique_frame(frame, by_frame, dropna: bool):
    """``groupby.nunique`` of ``frame`` by the one int64 key column of ``by_frame`` (``functors.groupby_nunique``): a
    frame of one row block.  It is not a GroupByReduce: distinct counts do not merge as partial tables."""
    blocks = [concat_cols([p.get() for p in row]) if len(row) > 1 else row[0].get() for row in frame._partitions]
    by_blocks = [row[0].get() for row in by_frame._partitions]
    if [b.nrows for b in blocks] != [b.nrows for b in by_blocks]:
        raise NotImplementedError("group keys partitioned unlike the frame's rows are not on the B200 path")
    block = groupby_nunique(blocks, by_blocks, frame.columns, dropna)
    pc = frame._partition_mgr_cls._partition_class
    return type(frame)(np.array([[pc(block)]], dtype=object), None, None, None, None)


def _groupby_reduce(agg: str):
    """``qc.groupby_<agg>`` (qc.py:3741-3748, alg/groupby.py) over device blocks.  ``by`` is a query compiler of key
    columns with the frame's rows; ``key_names`` replaces the names of the result's keys (``groupby(level=)``).
    ``agg_kwargs`` are read by first / last (``skipna``, ``min_count``), idxmax / idxmin (``skipna``, ``axis``), var /
    std (``ddof``) and nunique (``dropna``) only; the other aggregations ignore them.  nunique is not a GroupByReduce:
    it runs ``_nunique_frame``."""
    map_f, red_f = (DevGroupbyMap(agg), DevGroupbyReduce(agg)) if agg != "nunique" else (None, None)

    def caller(query_compiler, by, axis, groupby_kwargs, agg_args, agg_kwargs, drop=False, key_names=None, **kwargs):
        if by is None and groupby_kwargs.get("level") is not None and hasattr(query_compiler, "_b200_level_key"):
            # groupby(level=) through the plug-in: its query compiler turns the row labels into the key column
            by, name = query_compiler._b200_level_key(groupby_kwargs["level"])
            key_names = [name]
        if axis != 0 or not isinstance(by, type(query_compiler)) or len(by.columns) < 1:
            raise NotImplementedError("device groupby: key columns of the same frame, axis=0")
        fns = (map_f, red_f)
        if agg in ("first", "last"):
            skipna = _position_agg_skipna(agg, agg_kwargs)
            fns = (DevGroupbyMap(agg, skipna=skipna), DevGroupbyReduce(agg, skipna=skipna))
        if agg in ("idxmax", "idxmin"):
            _arg_agg_kwargs(agg, agg_kwargs)
        if agg in ("var", "std"):
            fns = (map_f, DevGroupbyReduce(agg, ddof=_var_ddof(agg, agg_kwargs)))
        if agg == "nunique":
            dropna = _nunique_dropna(agg_kwargs)
        frame, by_frame = query_compiler._modin_frame, by._modin_frame
        # a float64 key or several int64 keys: the single-key groupby runs on their int64 image and the G result keys
        # are restored afterwards (groupkeys.py); one int64 key is its own image
        keys = [concat_cols([p.get() for p in row]) if len(row) > 1 else row[0].get() for row in by_frame._partitions]
        images, image = gk.key_image(keys)
        if image is not None:
            pc = by_frame._partition_mgr_cls._partition_class
            by_frame = type(by_frame)(np.array([[pc(b)] for b in images], dtype=object), by_frame.copy_index_cache(),
                                      images[0].columns, by_frame.row_lengths, [1])  # fmt: skip
        if drop and len(by.columns) > 1:  # the packed key has a label of its own: the key columns leave here
            keep = [c for c in query_compiler.columns if c not in set(by.columns)]
            frame = query_compiler.getitem_column_array(keep)._modin_frame
        if agg in ("idxmax", "idxmin"):
            # labels of one dtype on every rank; the NaN group of a float key is dropped below under dropna, so it is
            # left out of the all-NaN check
            labels = arg_label_dtype([row[0].get() for row in frame._partitions])
            nan_key = image == gk.FLOAT_KEY and groupby_kwargs.get("dropna", True)
            fns = (DevGroupbyMap(agg, label_dtype=labels), DevGroupbyReduce(agg, nan_key=nan_key))
        # the functors themselves, not lambdas around them: the partition manager recognises them and fuses map +
        # reduce into one direct-addressed table per GPU when the key range allows (pm.groupby_reduce)
        if agg == "nunique":
            new_frame = _nunique_frame(frame, by_frame, dropna)
        else:
            new_frame = frame.groupby_reduce(axis, by_frame, *fns)
        if image is not None or key_names is not None:
            blocks = gk.restore_keys([row[0].get() for row in new_frame._partitions], image,
                                     groupby_kwargs.get("dropna", True), key_names)  # fmt: skip
            pc = new_frame._partition_mgr_cls._partition_class
            new_frame = type(new_frame)(np.array([[pc(b)] for b in blocks], dtype=object), None, None, None, None)
        if not groupby_kwargs.get("as_index", True):
            new_frame = group_keys_to_columns(new_frame)  # alg/groupby.py:278-294
        return query_compiler.__constructor__(new_frame)

    return caller


def device_operations(alg):
    """The device operations of a query compiler, registered through the operator templates of ``alg``."""

    class DeviceOperations:
        # ---- Map (qc.py:2036-2106) ----------------------------------------------------------------------
        abs = alg.Map.register(DevMap("abs"), dtypes="copy")
        negative = alg.Map.register(DevMap("neg"), dtypes="copy")
        isna = alg.Map.register(DevMap("isna"), dtypes=np.bool_)
        notna = alg.Map.register(DevMap("notna"), dtypes=np.bool_)
        round = alg.Map.register(DevRound(), dtypes="copy")  # qc.py:2438
        clip = alg.Map.register(DevClip(), dtypes="copy")  # qc.py `clip = Map.register(pandas.DataFrame.clip)`
        invert = alg.Map.register(DevMap("not"), dtypes=np.bool_)
        _astype_map = alg.Map.register(DevAstype())  # result dtypes are read back from the blocks

        def astype(self, col_dtypes, errors: str = "raise"):
            """qc.py ``astype(col_dtypes, errors)``: ``col_dtypes`` is one dtype for every column or a
            {column label: dtype} mapping.  Only the widening casts of ``DevAstype``; checked here, before any launch,
            so that a refused cast leaves no half-converted frame."""
            if errors != "raise":
                raise NotImplementedError("astype(errors='ignore') is not on the B200 path")
            return self._astype_map(col_dtypes=DevAstype.validate(self.dtypes, col_dtypes))

        def fillna(self, **kwargs):
            """qc.py:2710-2813: scalar / dict values are a Map, a frame value is an n-ary op; forward fill is a Fold."""
            value = kwargs.get("value")
            if kwargs.get("method") is not None:  # qc.py:2809-2810
                if kwargs["method"] not in ("ffill", "pad") or value is not None or kwargs.get("limit") is not None \
                        or kwargs.get("axis") not in (0, "index", None):  # fmt: skip
                    raise NotImplementedError("fillna(method=) on the B200 path: forward fill down the rows, no limit=")
                return self._ffill(0)
            if kwargs.get("limit") is not None:
                raise NotImplementedError("fillna(limit=) is not on the B200 path")
            if isinstance(value, type(self)):
                return self.__constructor__(
                    # PandasDataframe.n_ary_op takes the dtypes themselves: the "copy" shorthand is only understood by
                    # the Binary template and broadcast_apply
                    self._modin_frame.n_ary_op(lambda x, y: DevBinary("fillna")(x, y), [value._modin_frame],
                                               join_type="left", dtypes=self._modin_frame.copy_dtypes_cache())
                )  # fmt: skip
            return self.__constructor__(self._modin_frame.map(lambda x: DevFillna()(x, value=value), dtypes="copy"))

        # ---- Binary (qc.py:535-624) ---------------------------------------------------------------------
        add = alg.Binary.register(DevBinary("add"), infer_dtypes="common_cast")
        radd = alg.Binary.register(DevBinary("radd"), infer_dtypes="common_cast")
        sub = alg.Binary.register(DevBinary("sub"), infer_dtypes="common_cast")
        rsub = alg.Binary.register(DevBinary("rsub"), infer_dtypes="common_cast")
        mul = alg.Binary.register(DevBinary("mul"), infer_dtypes="common_cast")
        rmul = alg.Binary.register(DevBinary("rmul"), infer_dtypes="common_cast")
        truediv = alg.Binary.register(DevBinary("truediv"), infer_dtypes="common_cast")
        rtruediv = alg.Binary.register(DevBinary("rtruediv"), infer_dtypes="common_cast")
        eq = alg.Binary.register(DevBinary("eq"), infer_dtypes="bool")
        ne = alg.Binary.register(DevBinary("ne"), infer_dtypes="bool")
        lt = alg.Binary.register(DevBinary("lt"), infer_dtypes="bool")
        le = alg.Binary.register(DevBinary("le"), infer_dtypes="bool")
        gt = alg.Binary.register(DevBinary("gt"), infer_dtypes="bool")
        ge = alg.Binary.register(DevBinary("ge"), infer_dtypes="bool")
        # logical ops between bool frames (qc.py:541-571)
        __and__ = alg.Binary.register(DevLogical("and"), infer_dtypes="bool")
        __or__ = alg.Binary.register(DevLogical("or"), infer_dtypes="bool")
        __xor__ = alg.Binary.register(DevLogical("xor"), infer_dtypes="bool")

        # ---- TreeReduce (qc.py:976-1096) ----------------------------------------------------------------
        count = alg.TreeReduce.register(DevReduce("count"), DevReduce("count", phase="reduce"),
                                        compute_dtypes=lambda *a, **k: np.dtype("int64"))  # fmt: skip
        sum = alg.TreeReduce.register(DevReduce("sum"), DevReduce("sum", phase="reduce"), compute_dtypes=_dtypes_sum)
        prod = alg.TreeReduce.register(DevReduce("prod"), DevReduce("prod", phase="reduce"), compute_dtypes=_dtypes_sum)
        max = alg.TreeReduce.register(DevReduce("max"), DevReduce("max", phase="reduce"))
        min = alg.TreeReduce.register(DevReduce("min"), DevReduce("min", phase="reduce"))
        mean = alg.TreeReduce.register(DevMeanMap(), DevMeanReduce(), compute_dtypes=lambda *a, **k: np.dtype("float64"))
        any = alg.TreeReduce.register(DevBoolReduce("any"), DevBoolReduce("any", phase="reduce"),
                                      compute_dtypes=lambda *a, **k: np.dtype("bool"))  # qc.py:986
        all = alg.TreeReduce.register(DevBoolReduce("all"), DevBoolReduce("all", phase="reduce"),
                                      compute_dtypes=lambda *a, **k: np.dtype("bool"))  # qc.py:987

        # ---- Reduce: one function over FULL column partitions ---------------------------------------------
        # qc.py:1155-1156: std / var = Reduce.register(pandas.DataFrame.std / var) -- two sweeps over each full column
        # partition, two packed all-reduces when the rows span ranks
        # qc.py:1101-1102: idxmax / idxmin = Reduce.register(pandas.DataFrame.idxmax / idxmin) -- one arg-reduction
        # pass per column partition, one W-vector all-gather when the rows span ranks
        idxmax = alg.Reduce.register(DevArgReduce("max"))
        idxmin = alg.Reduce.register(DevArgReduce("min"))
        var = alg.Reduce.register(DevVar(sqrt=False))
        std = alg.Reduce.register(DevVar(sqrt=True))

        # ---- Fold (qc.py:2429-2431; forward fill is fillna(method="ffill"), qc.py:2809-2810) ----------------------
        cumsum = alg.Fold.register(DevCumulative("sum"), shape_preserved=True)
        cummax = alg.Fold.register(DevCumulative("max"), shape_preserved=True)
        cummin = alg.Fold.register(DevCumulative("min"), shape_preserved=True)
        _ffill = alg.Fold.register(DevCumulative("ffill"), shape_preserved=True)

        # ---- GroupByReduce (qc.py:3741-3748; impl table storage_formats/pandas/groupby.py:237-248) ------
        groupby_sum = _groupby_reduce("sum")
        groupby_count = _groupby_reduce("count")
        groupby_size = _groupby_reduce("size")
        groupby_mean = _groupby_reduce("mean")
        groupby_min = _groupby_reduce("min")
        groupby_max = _groupby_reduce("max")
        groupby_first = _groupby_reduce("first")
        groupby_last = _groupby_reduce("last")
        groupby_idxmax = _groupby_reduce("idxmax")
        groupby_idxmin = _groupby_reduce("idxmin")
        groupby_var = _groupby_reduce("var")
        groupby_std = _groupby_reduce("std")
        groupby_nunique = _groupby_reduce("nunique")  # a full-axis groupby, as in Modin (qc.groupby_nunique)

        _DEVICE_AGGS = ("sum", "count", "size", "mean", "min", "max", "first", "last", "idxmax", "idxmin", "var", "std",
                        "nunique")  # fmt: skip
        _KWARG_AGGS = ("first", "last", "idxmax", "idxmin", "var", "std", "nunique")  # aggregations that read agg_kwargs

        def groupby_agg(self, by, agg_func, axis, groupby_kwargs, agg_args, agg_kwargs, how="axis_wise", drop=False,
                        series_groupby=False):  # fmt: skip
            """qc.py:4236-4527.  The reference sends ``{column: function}`` dictionaries whose functions all have a
            map / reduce form through ``_groupby_dict_reduce`` (qc.py:3876-3970: one map table and one reduce table
            per function) and everything else through a full-axis ``groupby.agg`` on pandas blocks.  Here a dictionary
            over the device aggregations becomes one device aggregation per DISTINCT function over the columns that
            ask for it; every result carries the same ascending group keys, so the result blocks are zipped
            column-wise (buffers shared) in the dictionary's order.  A function name alone goes to its registered
            template.  Anything else has no device form and is refused -- there is no pandas block to fall back to."""
            if how != "axis_wise" or agg_args or (agg_kwargs and agg_func not in self._KWARG_AGGS):
                raise NotImplementedError(f"groupby ({how}) with extra arguments is not on the B200 path")
            if isinstance(agg_func, str) and agg_func in self._DEVICE_AGGS:
                return getattr(self, f"groupby_{agg_func}")(
                    by=by, axis=axis, groupby_kwargs=groupby_kwargs, agg_args=agg_args, agg_kwargs=agg_kwargs, drop=drop
                )
            if not isinstance(agg_func, dict) or not agg_func:
                raise NotImplementedError(f"groupby.agg({agg_func!r}) is not on the B200 path")
            if not isinstance(by, type(self)):
                raise NotImplementedError("device groupby: key columns of the same frame, axis=0")
            spec = {col: fn[0] if isinstance(fn, (list, tuple)) and len(fn) == 1 else fn for col, fn in agg_func.items()}
            by_func = gk.split_aggregations(spec, self.columns, set(by.columns) if drop else ())
            if len(by_func) > 1 and set(by_func) & {"first", "last", "idxmax", "idxmin", "var", "std", "nunique"} \
                    and dist.is_distributed():  # fmt: skip
                # across ranks the fused dense path of the other functions and the key-range exchange of first / last /
                # idxmax / idxmin / var / std / nunique give each rank a different key range
                raise NotImplementedError("groupby.agg mixing first / last / idxmax / idxmin / var / std / nunique with "
                                          "other functions across ranks")  # fmt: skip
            if any(isinstance(fn, (list, tuple)) for fn in agg_func.values()):
                raise NotImplementedError("groupby.agg with lists of functions (two-level result columns)")
            kw = dict(groupby_kwargs, as_index=True)
            results = []
            for fn, cols in by_func.items():
                res = getattr(self.getitem_column_array(cols), f"groupby_{fn}")(
                    by=by, axis=axis, groupby_kwargs=kw, agg_args=(), agg_kwargs={}, drop=False
                )
                results.append([[p.get() for p in row] for row in res._modin_frame._partitions])
            pc = self._modin_frame._partition_mgr_cls._partition_class
            rows = [[pc(b)] for b in gk.zip_aggregations(spec, by_func, results)]
            new_frame = type(self._modin_frame)(np.array(rows, dtype=object), None, None, None, None)
            if not groupby_kwargs.get("as_index", True):
                new_frame = group_keys_to_columns(new_frame)  # alg/groupby.py:278-294
            return self.__constructor__(new_frame)

        # ---- merge (qc.py:657-667 -> MergeImpl.row_axis_merge merge.py:104-252) --------------------------
        def merge(self, right, **kwargs):
            """The per-block ``pandas.merge`` replaced by the device join functor (``modin_b200.merge``): many-to-one
            and many-to-many keys, ``on`` or ``left_on`` / ``right_on``, how in {left, inner}."""
            from .merge import row_axis_merge

            return self.__constructor__(row_axis_merge(self, right, _reset_row_index, **kwargs))

    return DeviceOperations


class B200QueryCompiler(device_operations(algebra)):
    """Query compiler holding a ``B200Dataframe`` (qc.py:279-302)."""

    _modin_frame: B200Dataframe
    _shape_hint = None

    def __init__(self, modin_frame: B200Dataframe, shape_hint=None):
        self._modin_frame = modin_frame
        self._shape_hint = shape_hint

    @property
    def __constructor__(self):
        return type(self)

    storage_format = property(lambda self: self._modin_frame.storage_format)
    engine = property(lambda self: self._modin_frame.engine)

    # ---- metadata ----------------------------------------------------------------------------------
    index = property(lambda self: self._modin_frame.index)
    columns = property(lambda self: self._modin_frame.columns)
    dtypes = property(lambda self: self._modin_frame.dtypes)
    frame_has_materialized_dtypes = property(lambda self: self._modin_frame.has_materialized_dtypes)
    frame_has_materialized_columns = property(lambda self: self._modin_frame.has_materialized_columns)

    def get_axis_len(self, axis):
        return len(self._modin_frame) if axis == 0 else len(self.columns)

    # ---- lifecycle (qc.py:366-387) ------------------------------------------------------------------
    def finalize(self):
        self._modin_frame.finalize()

    def execute(self):
        self.finalize()
        self._modin_frame.wait_computations()

    def free(self):
        pass

    @classmethod
    def from_pandas(cls, df, data_cls=B200Dataframe):
        return cls(data_cls.from_pandas(df))

    @classmethod
    def from_arrow(cls, at, data_cls=B200Dataframe):
        return cls(data_cls.from_arrow(at))

    def to_pandas(self):
        return self._modin_frame.to_pandas()

    def to_numpy(self, **kwargs):
        return self._modin_frame.to_numpy(**kwargs)

    def default_to_pandas(self, pandas_op, *args, **kwargs):
        name = getattr(pandas_op, "__name__", str(pandas_op))
        raise NotImplementedError(
            f"`{name}` has no device implementation in modin_b200 and this execution never defaults to pandas"
        )

    def sort_rows_by_column_values(self, columns, ascending=True, **kwargs):
        """qc.py ``sort_rows_by_column_values`` -> ``PandasDataframe.sort_by`` (df.py:2741-2791): one float64 / int64
        key column, NaN last, ties in original row order (pandas ``kind="stable"``; the default quicksort leaves
        tie order unspecified, so a stable result is a valid answer for every ``kind``)."""
        from .functors import DevSortRows

        pos, asc = DevSortRows.resolve(self.columns, columns, ascending, **kwargs)
        return self.__constructor__(self._modin_frame.sort_by(pos, asc, bool(kwargs.get("ignore_index", False))))

    def drop_duplicates(self, subset=None, keep="first", ignore_index=False):
        """What ``BasePandasDataset.drop_duplicates`` (modin/pandas/base.py:1600-1623) asks of the query compiler --
        ``qc.unique(keep, ignore_index, subset)``, qc.py:2231-2270: rows with the first / last occurrence of every
        value of ONE int64 subset column (``subset=None`` means all columns, so it is accepted only for a
        one-column frame)."""
        from .functors import DevDropDuplicates

        pos = DevDropDuplicates.resolve(self.columns, subset, keep)
        return self.__constructor__(self._modin_frame.drop_duplicate_rows(pos, keep, bool(ignore_index)))

    def relabel_columns(self, new_labels):
        """Same buffers, new column labels (metadata only; ``qc.columns = ...`` in the reference)."""
        new_labels = pandas.Index(new_labels)
        if len(new_labels) != len(self.columns):
            raise ValueError("Length mismatch: expected axis has %d elements, new values have %d elements"
                             % (len(self.columns), len(new_labels)))  # fmt: skip
        return self.__constructor__(self._modin_frame.relabel_columns(new_labels))

    def set_column(self, label, value_qc):
        """``df[label] = series``: append (or replace) one column, sharing every buffer (qc.setitem / insert)."""
        value_qc = value_qc.relabel_columns([label])
        labels = list(self.columns)
        if label in labels:
            pos = labels.index(label)
            others = [i for i in range(len(labels)) if i != pos]
            base = self.__constructor__(self._modin_frame.take_2d_labels_or_positional(col_positions=others))
            stacked = self.__constructor__(base._modin_frame.hstack(value_qc._modin_frame))
            order = list(range(pos)) + [len(others)] + list(range(pos, len(others)))
            return self.__constructor__(stacked._modin_frame.take_2d_labels_or_positional(col_positions=order))
        return self.__constructor__(self._modin_frame.hstack(value_qc._modin_frame))

    def head(self, n):
        return self.__constructor__(self._modin_frame.head_rows(n))

    def tail(self, n):
        return self.__constructor__(self._modin_frame.tail_rows(n))

    def isin(self, values, **kwargs):
        """qc.py ``isin = Map.register(pandas.DataFrame.isin, dtypes=np.bool_)``: integer values, int64 columns."""
        from .functors import DevIsin

        return self.__constructor__(self._modin_frame.map(DevIsin(values), dtypes=np.bool_))

    def getitem_row_mask(self, mask_qc):
        """``df[bool_series]`` (qc.getitem_array with a boolean key, qc.py:2907-2960): rows where the mask holds."""
        return self.__constructor__(self._modin_frame.filter_rows(mask_qc._modin_frame))

    def row_all(self):
        """Row-wise AND over bool columns -> one bool column (``(...).all(axis=1)``; used by dropna)."""
        from .functors import DevRowLogical

        return self.__constructor__(self._modin_frame.rowwise_to_column(DevRowLogical("all")))

    def row_any(self):
        from .functors import DevRowLogical

        return self.__constructor__(self._modin_frame.rowwise_to_column(DevRowLogical("any")))

    def getitem_column_array(self, key, numeric=False, ignore_order=False):
        """qc.py:2885-2905."""
        if numeric:
            positions = list(key)
        else:
            positions = [int(p) for p in self.columns.get_indexer_for(list(key))]
            if any(p < 0 for p in positions):
                missing = [k for k, p in zip(key, positions) if p < 0]
                raise KeyError(f"{missing} not in index")
        return self.__constructor__(self._modin_frame.take_2d_labels_or_positional(col_positions=positions))

    copy_data = algebra.Map.register(DevMap("copy"), dtypes="copy")

    def var(self, axis=0, skipna=True, ddof=1, numeric_only=False, **kwargs):
        """The W variances as a host ``pandas.Series``: the API layer of the mirror takes reductions of this kind as W
        host numbers (identical on every rank)."""
        return self._host_series(super().var(axis=axis, skipna=skipna, ddof=ddof, numeric_only=numeric_only))

    def std(self, axis=0, skipna=True, ddof=1, numeric_only=False, **kwargs):
        return self._host_series(super().std(axis=axis, skipna=skipna, ddof=ddof, numeric_only=numeric_only))

    def _host_series(self, qc):
        return pandas.Series(qc.to_pandas().iloc[0].to_numpy(dtype=np.float64), index=self.columns, dtype="float64")

def group_keys_to_columns(frame):
    """Result frame of a device groupby with ``as_index=False``: keys as leading columns, rows renumbered 0..G-1 over
    all row partitions (and ranks, in rank order = key order).  Metadata only."""
    from . import dist
    from .functors import keys_to_columns

    lengths = [row[0].length() for row in frame._partitions]
    offset = dist.exclusive_row_offset(sum(lengths)) if dist.is_distributed() else 0
    pc = frame._partition_mgr_cls._partition_class
    rows = []
    for row, n in zip(frame._partitions, lengths):
        if len(row) != 1:
            raise NotImplementedError("groupby(as_index=False) results wider than one column partition")
        rows.append([pc(keys_to_columns(row[0].get(), offset))])
        offset += n
    first = rows[0][0].get()
    start = offset - sum(lengths)
    return type(frame)(np.array(rows, dtype=object), pandas.RangeIndex(start, offset), first.columns, lengths,
                       [len(first.cols)], None)  # fmt: skip


def _frame_device(frame):
    """Device of the frame's first non-empty block (works for the mirror frame and for Modin's ``PandasDataframe``)."""
    from .block import current_device

    for p in frame._partitions.flatten():
        b = p.get()
        if b.cols:
            return b.cols[0].data.device
    return current_device()


def _reset_row_index(frame: B200Dataframe, offset_hint=None) -> B200Dataframe:
    """``reset_index(drop=True)`` on range-indexed device blocks: renumber ``range_start`` so that
    the row partitions of this rank form one contiguous RangeIndex (metadata only, no kernel).
    ``offset_hint``: this rank's first global row position when the caller already knows it (a left merge keeps
    the left frame's rows, so the left shard's own range start is the answer) -- saves the collective + D2H that
    counting the other ranks' rows costs."""
    from . import dist
    from .block import DeviceBlock

    lengths = frame.row_lengths
    offset = 0
    if offset_hint is not None:
        offset = int(offset_hint)
    elif dist.is_distributed():
        import torch

        dev = _frame_device(frame)
        mine = torch.zeros(dist.world_size(), dtype=torch.int64, device=dev)
        mine[dist.rank()] = sum(lengths)
        dist.all_reduce_values([mine], ["sum"])
        offset = int(mine[: dist.rank()].sum().item())
    pc = frame._partition_mgr_cls._partition_class
    rows = []
    for row, n in zip(frame._partitions, lengths):
        new_row = []
        for p in row:
            b = p.get()
            new_row.append(pc(DeviceBlock(b.cols, b.columns, nrows=b.nrows, range_start=offset)))
        rows.append(new_row)
        offset += n
    start = offset - sum(lengths)
    return type(frame)(np.array(rows, dtype=object), pandas.RangeIndex(start, offset), frame._columns_cache,
                       lengths, frame._column_widths_cache, frame._dtypes)  # fmt: skip
