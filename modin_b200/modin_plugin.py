"""Plug the B200 execution in behind the real ``modin.pandas`` (when Modin is importable).

``register()`` adds an execution ``(storage_format="Arrow", engine="B200")`` to Modin through its
public hooks only -- no reference file is edited (SURVEY.md §8b-1):

* ``StorageFormat.add_option`` / ``Engine.add_option`` / ``Backend.register_backend``
  (modin/config/envvars.py:271-277, 449-472);
* a factory class injected as ``factories.ArrowOnB200Factory`` -- the dispatcher looks factories up
  by exactly that name (modin/core/execution/dispatching/factories/dispatcher.py:143-172);
* ``BaseIO`` subclass naming the frame and query-compiler classes (modin/core/io/io.py:51-52).

The classes are Modin's OWN ``PandasDataframe`` / ``PandasDataframePartitionManager`` /
``PandasQueryCompiler`` with this package's device classes mixed in in front, so every non-hot
method keeps Modin's behaviour while the hot path (Map / Binary / TreeReduce / GroupByReduce /
broadcast merge) is re-registered with device functors through Modin's unchanged operator
templates.  ``modin.set_execution(engine="B200", storage_format="Arrow")`` then makes
``import modin.pandas as pd`` a drop-in.

The image ships pandas 3 while the reference pins pandas<2.4; ``apply_pandas3_shims()`` restores the
five removed names / keyword arguments Modin's import and hot path need (SURVEY.md §8c).  It touches
only pandas attributes, never Modin.
"""

from __future__ import annotations

import functools
import weakref

import numpy as np
import pandas

_REGISTERED = None


def apply_pandas3_shims() -> None:
    """Make ``import modin`` and its hot path work under pandas 3 (no-ops on pandas 2.x)."""
    import pandas.core.series as pcs
    import pandas.io.parsers.base_parser as bp

    def _stub(*a, **k):
        """Removed from pandas 3; not on the B200 path."""
        raise NotImplementedError

    if not hasattr(pandas, "read_gbq"):
        pandas.read_gbq = _stub
    if not hasattr(pcs, "_coerce_method"):

        def _coerce_method(converter):
            def wrapper(self):
                if len(self) == 1:
                    return converter(self.iloc[0])
                raise TypeError(f"cannot convert the series to {converter}")

            wrapper.__name__ = f"__{converter.__name__}__"
            return wrapper

        pcs._coerce_method = _coerce_method
    if not hasattr(bp.ParserBase, "_validate_usecols_arg"):
        bp.ParserBase._validate_usecols_arg = lambda self, usecols: (usecols, None)
    for cls in (pandas.DataFrame, pandas.Series):
        if getattr(cls.groupby, "_mb200_shim", False):
            continue
        g = cls.groupby

        def _groupby(self, *a, axis=0, _g=g, **k):
            # pandas 3 removed ``axis=``; Modin still passes the default -- anything else must fail, not be ignored
            if axis not in (0, "index"):
                raise TypeError("groupby() got an unexpected keyword argument 'axis' (removed in pandas 3)")
            return _g(self, *a, **k)

        wrapped = functools.wraps(g)(_groupby)
        wrapped._mb200_shim = True
        cls.groupby = wrapped
        f = cls.fillna

        def _fillna(self, *a, method=None, downcast=None, _f=f, **k):
            if method is not None or downcast is not None:
                raise TypeError("fillna() got an unexpected keyword argument 'method' / 'downcast' (removed in pandas 3)")
            return _f(self, *a, **k)

        cls.fillna = functools.wraps(f)(_fillna)


def register(shims: bool | None = None):
    """Register the execution with Modin and return the namespace of generated classes."""
    global _REGISTERED
    if _REGISTERED is not None:
        return _REGISTERED
    if shims is None:
        shims = int(pandas.__version__.split(".")[0]) >= 3
    if shims:
        apply_pandas3_shims()

    import modin.config as cfg
    from modin.config.envvars import Execution
    from modin.core.dataframe import algebra as malg
    from modin.core.dataframe.pandas.dataframe.dataframe import PandasDataframe
    from modin.core.dataframe.pandas.partitioning.partition_manager import PandasDataframePartitionManager
    from modin.core.execution.dispatching.factories import factories
    from modin.core.io.io import BaseIO
    from modin.core.storage_formats.pandas.query_compiler import PandasQueryCompiler

    from . import dist as bdist
    from . import functors as fx
    from . import partitioning as bp
    from .block import DeviceBlock, concat_cols
    from .query_compiler import _reset_row_index, device_operations

    # ---------------------------------------------------------------- partition manager
    class B200OnModinPartitionManager(bp.B200PartitionManager, PandasDataframePartitionManager):
        """Device classmethods first in the MRO; indexing / rebalancing helpers stay Modin's."""

        _partition_class = bp.B200Partition
        _column_partitions_class = bp.B200ColumnPartition
        _row_partition_class = bp.B200RowPartition
        _execution_wrapper = bp.B200Wrapper

        @classmethod
        def from_pandas(cls, df, return_dims=False):
            """The frame (``B200OnModinDataframe.from_pandas``) cuts this rank's row shard itself, together with the
            shard's row labels, so the partition manager must not cut again."""
            return cls.from_pandas_local(df, return_dims)

        # The grid walkers whose bodies are pure protocol (loop over the grid, call ``partition.apply`` /
        # ``add_to_apply_calls`` / ``axis_partition.apply``) are Modin's OWN under the plug-in -- the standalone mirror
        # carries restatements of them only because it must run without Modin.  What stays overridden above are the
        # methods that do something different on a device: groupby_reduce (fused dense table), n_ary_operation (queued
        # for fusion), shuffle_partitions, ingest / egress, combine, finalize / wait.
        map_partitions = classmethod(PandasDataframePartitionManager.map_partitions.__func__)
        lazy_map_partitions = classmethod(PandasDataframePartitionManager.lazy_map_partitions.__func__)
        broadcast_axis_partitions = classmethod(PandasDataframePartitionManager.broadcast_axis_partitions.__func__)
        map_axis_partitions = classmethod(PandasDataframePartitionManager.map_axis_partitions.__func__)
        broadcast_apply = classmethod(PandasDataframePartitionManager.broadcast_apply.__func__)
        base_broadcast_apply = classmethod(PandasDataframePartitionManager.base_broadcast_apply.__func__)
        axis_partition = classmethod(PandasDataframePartitionManager.axis_partition.__func__)
        column_partitions = classmethod(PandasDataframePartitionManager.column_partitions.__func__)
        row_partitions = classmethod(PandasDataframePartitionManager.row_partitions.__func__)

    # ---------------------------------------------------------------- core dataframe
    class B200OnModinDataframe(PandasDataframe):
        _partition_mgr_cls = B200OnModinPartitionManager

        @property
        def engine(self) -> str:  # df.py:137-148
            return "B200"

        @property
        def storage_format(self) -> str:  # df.py:125-135
            return "Arrow"

        # ---- one process per GPU: every rank holds its own row shard (labels included) ----------------------
        @classmethod
        def from_pandas(cls, df):
            """df.py:4592-4620 pairs ``df.index`` with the partitions of ``df``; under torch.distributed the
            partitions hold this rank's contiguous row shard only, so index, dtypes and row lengths are the
            shard's (the same split ``B200Dataframe.from_pandas`` makes)."""
            lo = 0
            if bdist.is_distributed():
                lo, hi = bdist.shard_bounds(len(df))
                df = df.iloc[lo:hi]
            frame = super().from_pandas(df)
            frame._b200_shard_offset = lo  # this rank's first global row position (see merge.row_axis_merge)
            return frame

        @classmethod
        def from_pandas_replicated(cls, df):
            """A small host frame that every rank holds in full (reduction results computed on the host from
            all-reduced numbers): no sharding, and ``to_pandas`` must not gather it again."""
            frame = super().from_pandas(df)
            for p in frame._partitions.flatten():
                p.get().replicated = True
            return frame

        @classmethod
        def from_arrow(cls, at):
            """df.py:4622-4654.  Single process: Modin's own path (the partition manager copies the Arrow buffers
            H2D directly).  Under torch.distributed the rows are sharded like ``from_pandas`` (zero-copy pandas
            view of the table, then this rank's slice of it)."""
            if not bdist.is_distributed():
                return super().from_arrow(at)
            cols = {}
            for name, col in zip(at.column_names, at.columns):
                arr = col.combine_chunks() if hasattr(col, "combine_chunks") else col
                if arr.null_count:
                    arr = arr.fill_null(float("nan"))
                cols[name] = arr.to_numpy(zero_copy_only=False)
            return cls.from_pandas(pandas.DataFrame(cols, copy=False))

        def to_pandas(self):
            """df.py:4691-4722.  Under torch.distributed the partition manager all-gathers the row shards (unless
            the blocks are replicated results), so the host frame carries the JOB-wide rows while ``self.index``
            is this rank's: labels come from the blocks, after the deferred external labels have been pushed
            into them."""
            if not bdist.is_distributed():
                return super().to_pandas()
            self._propagate_index_objs(axis=None)
            df = self._partition_mgr_cls.to_pandas(self._partitions)
            if len(df.columns) == 0 and len(self.columns):
                df = pandas.DataFrame(columns=self.columns, index=df.index)
            return df

        def __dataframe__(self, nan_as_null: bool = False, allow_copy: bool = True):
            """df.py:4803-4824, over the device blocks (``modin_b200.interchange``): buffers stay in HBM and say so
            (``__dlpack_device__`` = CUDA), one chunk per row partition."""
            from .interchange import B200ProtocolDataframe

            self._propagate_index_objs(axis=None)
            blocks = [concat_cols([p.get() for p in row]) if len(row) > 1 else row[0].get() for row in self._partitions]
            return B200ProtocolDataframe(blocks, self.index, nan_as_null, allow_copy)

        @classmethod
        def from_interchange_dataframe(cls, df):
            """df.py:4826-4867 converts through pandas; here CUDA buffers are adopted through DLPack (no copy) and
            host buffers are copied H2D, one row partition per chunk of the producer."""
            if type(df) is cls:
                return df
            from .interchange import blocks_from_dataframe

            blocks = blocks_from_dataframe(df)
            pc = cls._partition_mgr_cls._partition_class
            parts = np.array([[pc.put(b)] for b in blocks], dtype=object).reshape(len(blocks), 1)
            index = None
            if all(b.has_range_index() for b in blocks):
                index = pandas.RangeIndex(blocks[0].range_start, blocks[0].range_start + sum(b.nrows for b in blocks))
            return cls(parts, index, blocks[0].columns, [b.nrows for b in blocks], [len(blocks[0].cols)])

        def map(self, *args, **kwargs):
            """df.py:2253-2322 hands the result this frame's row lengths -- a Map keeps the rows -- so the job-wide
            row count (``get_axis_len``) is handed on with them: Modin's API asks ``.empty`` of every intermediate
            frame, and an expression like ``df * b + c`` must not cost a control-plane collective per operator."""
            out = super().map(*args, **kwargs)
            rows = getattr(self, "_b200_job_rows", None)
            if rows is not None:
                out._b200_job_rows = rows
            return out

        def _build_treereduce_func(self, axis, func):
            """df.py:2081-2123: device reduce functors already return the 1 x W block labelled
            ``__reduced__``; only pandas results need the Series -> frame conversion."""
            pandas_wrapper = super()._build_treereduce_func(axis, func)

            def _tree_reduce_func(df, *args, **kwargs):
                if isinstance(df, DeviceBlock):
                    try:
                        result = func(df, *args, **kwargs)
                    except TypeError as e:
                        # an unbound pandas method (Reduce.register(pandas.DataFrame.median), qc.py:1107) handed a
                        # device block fails inside pandas with "super(type, obj): obj must be an instance ..."
                        if "super(type, obj)" not in str(e):
                            raise
                        raise NotImplementedError(
                            "this reduction has no device implementation in modin_b200 (unsupported operations raise "
                            "instead of falling back to pandas)"
                        ) from e
                    if isinstance(result, DeviceBlock):
                        return result
                    raise NotImplementedError(
                        "this reduction has no device functor in modin_b200 (no pandas fallback on the B200 path)"
                    )
                return pandas_wrapper(df, *args, **kwargs)

            return _tree_reduce_func

        # ---- lazy row / column labels without a reference cycle -----------------------------------------------
        # df.py:517-547: ``index=None`` / ``columns=None`` install ``ModinIndex(self, axis)``, whose default callable is a
        # lambda holding the frame (metadata/index.py:106) -- frame -> ModinIndex -> lambda -> frame.  A frame in such a
        # cycle (every groupby / Fold / merge result: their labels live on the device and stay lazy) is freed by
        # Python's cycle collector only, so its device buffers outlive the last user reference by an arbitrary time.
        # The callable is swapped for one that holds the frame WEAKLY; ``_is_default_callable`` stays set, so a copy
        # handed to another frame is still re-bound to that frame (``maybe_specify_new_frame_ref``) -- and weakened
        # again by that frame's own setter.
        def _weaken_lazy_labels(self, labels, axis):
            if getattr(labels, "_is_default_callable", False) and callable(getattr(labels, "_value", None)):
                ref = weakref.ref(self)

                def labels_and_lengths():
                    frame = ref()
                    if frame is None:
                        raise RuntimeError("the frame these lazy labels belong to has been released")
                    return frame._compute_axis_labels_and_lengths(axis)

                labels._value = labels_and_lengths

        def set_index_cache(self, index):
            super().set_index_cache(index)
            self._weaken_lazy_labels(self._index_cache, 0)

        def set_columns_cache(self, columns):
            super().set_columns_cache(columns)
            self._weaken_lazy_labels(self._columns_cache, 1)

        def set_dtypes_cache(self, dtypes):
            """df.py:415-438.  For ``dtypes=None`` the reference installs a lazy ``DtypesDescriptor(parent_df=self)``: frame
            and descriptor then reference each other, and the frame -- with its partitions, i.e. the device buffers --
            is only released by Python's CYCLE collector, not when the last user reference goes (measured: a 32 GB
            ``df.cumsum()`` result per call stayed allocated until the next generation-2 collection).  Device blocks
            carry their dtypes as host metadata, so whenever every first-row partition already holds its block the
            dtypes are known here and now, and no back-reference is created."""
            if dtypes is None and self.has_materialized_columns and self._partitions.size:
                try:
                    blocks = [p._data for p in self._partitions[0]]
                    if all(isinstance(b, DeviceBlock) and not p.call_queue for b, p in zip(blocks, self._partitions[0])):
                        kinds = [c.dtype for b in blocks for c in b.cols]
                        if len(kinds) == len(self.columns):
                            dtypes = pandas.Series([np.dtype(k) for k in kinds], index=self.columns)
                except Exception:  # whatever is odd about the grid: the reference's lazy path still works
                    dtypes = None
            return super().set_dtypes_cache(dtypes)

        def _compute_dtypes(self, columns=None):
            """df.py:472-520 runs a pandas lambda tree-reduce; device blocks carry their dtypes as host
            metadata, so read them directly."""
            series = [p.get().dtypes for p in self._partitions[0]] if self._partitions.size else []
            dtypes = pandas.concat(series) if series else pandas.Series([], dtype=object)
            dtypes.index = self.columns
            if columns is not None:
                dtypes = dtypes.loc[list(columns)]
            return dtypes

    _LEVEL_KEY = "__b200_index_level__"

    def _labels_as_by(query_compiler, level):
        """(query compiler of ONE key column holding the row labels, the level's name) for ``groupby(level=...)`` on a
        single-level index."""
        from . import ops

        frame = query_compiler._modin_frame
        levels = level if isinstance(level, (list, tuple)) else [level]
        if len(levels) != 1 or frame._partitions.shape[1] < 1:
            raise NotImplementedError("device groupby: one index level")
        frame._propagate_index_objs(axis=0)  # deferred labels go into the blocks first
        pc = frame._partition_mgr_cls._partition_class
        rows, name = [], None
        for row in frame._partitions:
            b = row[0].get()
            if b.index_host is not None or (b.index_cols and len(b.index_cols) != 1):
                raise NotImplementedError("device groupby(level=): numeric single-level row labels")
            if b.index_cols:
                col, name = b.index_cols[0], (b.index_names or [None])[0]
            else:
                col = ops.iota(b.range_start, b.nrows)
            rows.append([pc(DeviceBlock([col], pandas.Index([_LEVEL_KEY]), nrows=b.nrows, range_start=b.range_start))])
        lv = levels[0]
        if isinstance(lv, (int, np.integer)) and not isinstance(lv, bool):
            if lv not in (0, -1):  # pandas' own errors (core/groupby/grouper.py)
                raise ValueError("level > 0 or level < -1 only valid with MultiIndex")
        elif lv != name:
            raise ValueError(f"level name {lv} is not the name of the index")
        by_frame = type(frame)(np.array(rows, dtype=object), frame.copy_index_cache(), pandas.Index([_LEVEL_KEY]),
                               frame.row_lengths, [1])  # fmt: skip
        return query_compiler.__constructor__(by_frame), name

    def _by_level(groupby_agg):
        """A groupby aggregation of ``device_operations`` that also takes ``groupby(level=0)``: the row labels are the
        key (alg/groupby.py:355-390 hands ``level`` to pandas per block).  They already sit on the device (an index
        column) or are a range (materialised with mb200_iota); the frame of one key column built from them goes down
        the ordinary path, and the result's keys take the index level's own name."""

        def caller(query_compiler, by, axis, groupby_kwargs, agg_args, agg_kwargs, drop=False, **kwargs):
            level = groupby_kwargs.get("level")
            key_names = None
            if level is not None:
                if by is not None or axis != 0:
                    raise NotImplementedError("device groupby: `level=` together with `by` is not on the B200 path")
                by, name = _labels_as_by(query_compiler, level)
                key_names = [name]
            return groupby_agg(query_compiler, by, axis, groupby_kwargs, agg_args, agg_kwargs, drop=drop,
                               key_names=key_names, **kwargs)  # fmt: skip

        return caller

    # ---------------------------------------------------------------- query compiler
    def _arith(op, generic):
        """The ``generic`` Binary registration of ``op`` (qc.py:535-566) with one shortcut in front:
        a float64 frame against a real SCALAR keeps its dtypes, so the template's dtype inference (a pandas concat of
        two dtype Series per operator, ~0.5 ms of host time: as much as the kernel needs for 2e7 rows) is skipped and
        the scalar branch of the template (alg/binary.py:444-455: a lazy ``frame.map``) is taken directly."""
        functor = fx.DevBinary(op)

        def caller(query_compiler, other, broadcast=False, *args, dtypes=None, **kwargs):
            frame = query_compiler._modin_frame
            if (dtypes is None and not broadcast and not args and isinstance(other, (float, int, np.floating, np.integer))
                    and not isinstance(other, (bool, np.bool_)) and kwargs.get("level") is None
                    and kwargs.get("fill_value") is None and kwargs.get("axis", 0) in (0, 1, "index", "columns", None)
                    and frame.has_materialized_dtypes and all(dt == np.float64 for dt in frame.dtypes)):  # fmt: skip
                shape_hint = "column" if frame.has_materialized_columns and len(frame.columns) == 1 else None
                new_frame = frame.map(functor, func_args=(other,), func_kwargs=kwargs, dtypes="copy", lazy=True)
                return query_compiler.__constructor__(new_frame, shape_hint=shape_hint)
            return generic(query_compiler, other, broadcast, *args, dtypes=dtypes, **kwargs)

        return caller

    Ops = device_operations(malg)

    class B200OnModinQueryCompiler(Ops, PandasQueryCompiler):
        def get_axis_len(self, axis):
            """qc.py:411-427.  Under torch.distributed ``len(df)`` is the JOB-wide row count, not this rank's shard:
            Modin's API layer decides from it whether a frame is ``empty`` -- and defaults every method call on an
            empty frame to pandas (modin/pandas/base.py:4372) -- so a rank whose shard happens to be empty (a filter that
            only matched rows elsewhere) would leave the device path, skip the collectives the other ranks issue, and
            hang the job.  The count is agreed once per frame over the host-side control group (gloo: no device
            synchronisation) and cached on the frame; results every rank holds in full answer locally."""
            if axis == 0 and bdist.is_distributed():
                frame = self._modin_frame
                n = getattr(frame, "_b200_job_rows", None)
                if n is None:
                    local = len(frame)
                    # the payloads as they are: asking must not run a partition's pending call queue (``get()`` would
                    # launch a queued ``* b`` on its own and cost the fusion with the ``+ c`` that follows)
                    parts = frame._partitions.flatten()
                    replicated = len(parts) > 0 and all(getattr(p._data, "replicated", False) for p in parts)
                    n = local if replicated else bdist.control_sum(local)
                    frame._b200_job_rows = n
                return n
            return super().get_axis_len(axis)

        # Binary (qc.py:535-624)
        add = _arith("add", Ops.add)
        radd = _arith("radd", Ops.radd)
        sub = _arith("sub", Ops.sub)
        rsub = _arith("rsub", Ops.rsub)
        mul = _arith("mul", Ops.mul)
        rmul = _arith("rmul", Ops.rmul)
        truediv = _arith("truediv", Ops.truediv)
        rtruediv = _arith("rtruediv", Ops.rtruediv)
        # Series comparisons are separate registrations in the reference (qc.py:586-604, they take fill_value);
        # on the device a Series is a one-column frame, so the same functors serve
        series_eq = malg.Binary.register(fx.DevBinary("eq"), infer_dtypes="bool")
        series_ne = malg.Binary.register(fx.DevBinary("ne"), infer_dtypes="bool")
        series_lt = malg.Binary.register(fx.DevBinary("lt"), infer_dtypes="bool")
        series_le = malg.Binary.register(fx.DevBinary("le"), infer_dtypes="bool")
        series_gt = malg.Binary.register(fx.DevBinary("gt"), infer_dtypes="bool")
        series_ge = malg.Binary.register(fx.DevBinary("ge"), infer_dtypes="bool")
        # GroupByReduce (qc.py:3741-3748), with groupby(level=)
        groupby_sum = _by_level(Ops.groupby_sum)
        groupby_count = _by_level(Ops.groupby_count)
        groupby_size = _by_level(Ops.groupby_size)
        groupby_mean = _by_level(Ops.groupby_mean)
        groupby_min = _by_level(Ops.groupby_min)
        groupby_max = _by_level(Ops.groupby_max)
        # first / last come from the shared definition as they are; it asks this for the key of groupby(level=)
        _b200_level_key = _labels_as_by

        def unique(self, keep="first", ignore_index=True, subset=None):
            """qc.py:2231-2270 -- what ``drop_duplicates`` (modin/pandas/base.py:1600-1623) and ``Series.unique``
            ask for.  One full-axis application of the device functor instead of duplicated() + row selection."""
            pos = fx.DevDropDuplicates.resolve(self.columns, subset, keep)
            frame = self._modin_frame  # under torch.distributed the functor exchanges the per-rank survivors itself
            if frame._partitions.shape[1] != 1:
                raise NotImplementedError("device drop_duplicates: frames of one column partition (up to 32 columns)")
            fn = fx.DevDropDuplicates()
            new_frame = frame.apply_full_axis(
                0, lambda blk: fn(blk, pos, keep=keep, ignore_index=bool(ignore_index)), new_columns=self.columns,
                dtypes="copy", keep_partitioning=True, num_splits=1, sync_labels=False,
            )  # fmt: skip
            return self.__constructor__(new_frame, shape_hint=self._shape_hint)

        def sort_rows_by_column_values(self, columns, ascending=True, **kwargs):
            """qc.py ``sort_rows_by_column_values`` -> PandasDataframe.sort_by (df.py:2741-2791), a range-partitioning
            shuffle whose sampling / pivot / split callbacks run pandas code on the blocks.  Here the same shuffle
            with device callbacks (``B200PartitionManager.shuffle_partitions`` + ``shuffle.DevShuffleFunctions``):
            stable, NaN last, one float64 / int64 key column; across GPUs one key range per rank."""
            from .dataframe import B200Dataframe

            pos, asc = fx.DevSortRows.resolve(self.columns, columns, ascending, **kwargs)
            frame = self._modin_frame
            frame._propagate_index_objs(axis=0)  # deferred external row labels go into the blocks first
            mirror = B200Dataframe(frame._partitions, None, self.columns, None, None, None)
            done = mirror.sort_by(pos, asc, bool(kwargs.get("ignore_index", False)))
            new_frame = type(frame)(done._partitions, None, self.columns, done.row_lengths, done.column_widths,
                                    dtypes=frame.copy_dtypes_cache())  # fmt: skip
            return self.__constructor__(new_frame)

        def nunique(self, axis=0, dropna=True):
            """qc.py:1109-1113 is a full-axis ``pandas.DataFrame.nunique``; here one group table per int64 column,
            the answer is its number of groups.  The W counts go back as a 1 x W frame like the other reductions."""
            if axis != 0:
                raise NotImplementedError("nunique(axis=1) is not on the B200 path")
            bad = [c for c, dt in zip(self.columns, self.dtypes) if np.dtype(dt) != np.int64]
            if bad:
                raise NotImplementedError(f"nunique on the B200 path counts int64 columns only (got {bad!r})")
            counts = []
            for label in self.columns:
                key = self.getitem_column_array([label])
                sizes = key.groupby_size(by=key, axis=0, groupby_kwargs={}, agg_args=(), agg_kwargs={})
                counts.append(sum(sizes._modin_frame.row_lengths))  # across GPUs: this rank's key range of the table
            if bdist.is_distributed():
                import torch

                t = torch.tensor(counts, dtype=torch.int64, device=self._modin_frame._partitions[0, 0].get().cols[0].data.device)
                bdist.all_reduce_values([t], ["sum"])
                counts = [int(v) for v in t.tolist()]
            from modin.utils import MODIN_UNNAMED_SERIES_LABEL

            host = pandas.DataFrame([counts], columns=self.columns, index=[MODIN_UNNAMED_SERIES_LABEL], dtype=np.int64)
            return self.__constructor__(type(self._modin_frame).from_pandas_replicated(host))

        def getitem_array(self, key):
            """qc.py:3072-3103.  A one-column bool query compiler is boolean row selection: the reference registers
            ``lambda df, r: df[r]`` as a Binary template (``__getitem_bool``, qc.py:3021-3025) and calls it with
            ``broadcast=True`` -- ``broadcast_apply(axis=0, ..., join_type="left", labels="drop")``.  Same call here
            with the device row filter as the block function (the template itself cannot be reused: its broadcast
            branch calls ``right.squeeze()`` on the block, binary.py:396-402).  Lists of labels go to Modin's code."""
            if isinstance(key, type(self)) and len(key.dtypes) == 1 and pandas.api.types.is_bool_dtype(key.dtypes.iloc[0]):
                if len(key.index) != len(self.index):
                    raise ValueError(f"Item wrong length {len(key.index)} instead of {len(self.index)}.")
                fn = fx.DevRowFilter()
                new_frame = self._modin_frame.broadcast_apply(
                    0, lambda left, right: fn(left, right), key._modin_frame, join_type="left", labels="drop",
                    dtypes="copy",
                )  # fmt: skip
                return self.__constructor__(new_frame)
            return super().getitem_array(key)

        def isin(self, values, ignore_indices=False):
            """qc.py ``isin`` (a Map over ``pandas.DataFrame.isin``): a list of integers against int64 columns."""
            if isinstance(values, (type(self), dict, pandas.Series, pandas.DataFrame)) or ignore_indices:
                raise NotImplementedError("isin on the B200 path takes a list / array of integers")
            fn = fx.DevIsin(values)
            return self.__constructor__(self._modin_frame.map(lambda blk: fn(blk), dtypes=np.bool_))

        def dropna(self, **kwargs):
            """qc.py:3249-3333.  Rows only: ``notna`` of the (subset) columns -> row-wise all / any -> the boolean
            row selection above, all on the device."""
            from pandas._libs import lib as pandas_lib

            how = kwargs.get("how", "any")
            how = "any" if how is pandas_lib.no_default or how is None else how
            if kwargs.get("axis", 0) not in (0, "index") or kwargs.get("thresh", pandas_lib.no_default) not in (pandas_lib.no_default, None):
                raise NotImplementedError("dropna on the B200 path drops rows, without thresh=")
            if how not in ("any", "all"):
                raise ValueError(f"invalid how option: {how}")
            subset = kwargs.get("subset")
            src = self if subset is None else self.getitem_column_array(list(subset) if pandas.api.types.is_list_like(subset) else [subset])
            flags = src.notna()._modin_frame
            from modin.utils import MODIN_UNNAMED_SERIES_LABEL

            fn = fx.DevRowLogical("all" if how == "any" else "any", label=MODIN_UNNAMED_SERIES_LABEL)
            mask = flags.apply_full_axis(
                1, lambda blk: fn(blk), new_index=flags.copy_index_cache(), new_columns=pandas.Index([MODIN_UNNAMED_SERIES_LABEL]),
                dtypes=np.bool_, keep_partitioning=True, num_splits=1, sync_labels=False,
            )  # fmt: skip
            return self.getitem_array(self.__constructor__(mask, shape_hint="column"))

        def cumprod(self, *args, **kwargs):
            raise NotImplementedError("cumprod is not on the B200 path")

        def reset_index(self, **kwargs):
            """qc.py ``reset_index``: only ``drop=True`` over all levels -- a renumbering of the blocks' range starts
            (metadata).  Turning row labels into columns would need the labels on the device first."""
            if not kwargs.get("drop", False) or kwargs.get("level") is not None:
                raise NotImplementedError("reset_index on the B200 path: drop=True, no level=")
            return self.__constructor__(_reset_row_index(self._modin_frame))

    # ---------------------------------------------------------------- IO + factory
    class B200IO(BaseIO):
        frame_cls = B200OnModinDataframe
        query_compiler_cls = B200OnModinQueryCompiler

        @classmethod
        def read_parquet(cls, **kwargs):
            """io.py:218-220 defaults to ``pandas.read_parquet`` + ``from_pandas``; here the file is decoded to an
            Arrow table on the host (pyarrow) and its column buffers are copied to the device as they are
            (``from_arrow``: no pandas frame in between).  ``path`` and ``columns`` only; filters, partitioned
            datasets and storage options are the reference's ``parquet_dispatcher`` (962 lines), out of scope."""
            import pyarrow.parquet as pq

            path = kwargs.pop("path")
            columns = kwargs.pop("columns", None)
            from pandas._libs import lib as pandas_lib

            extra = {k: v for k, v in kwargs.items() if v is not pandas_lib.no_default and v not in (None, False, "auto")
                     and k not in ("engine", "dtype_backend", "filesystem")}  # fmt: skip
            if extra:
                raise NotImplementedError(f"read_parquet({', '.join(sorted(extra))}=...) is not on the B200 path")
            return cls.from_arrow(pq.read_table(path, columns=columns))

    class ArrowOnB200Factory(factories.BaseFactory):
        @classmethod
        def prepare(cls):
            cls.io_cls = B200IO

    cfg.StorageFormat.add_option("Arrow")
    cfg.Engine.add_option("B200")
    if "B200" not in cfg.Backend.get_active_backends() if hasattr(cfg.Backend, "get_active_backends") else True:
        try:
            cfg.Backend.register_backend("B200", Execution(storage_format="Arrow", engine="B200"))
        except ValueError:
            pass  # already registered in this interpreter
    setattr(factories, "ArrowOnB200Factory", ArrowOnB200Factory)

    class _NS:
        pass

    ns = _NS()
    ns.PartitionManager = B200OnModinPartitionManager
    ns.Dataframe = B200OnModinDataframe
    ns.QueryCompiler = B200OnModinQueryCompiler
    ns.IO = B200IO
    ns.Factory = ArrowOnB200Factory
    _REGISTERED = ns
    return ns


def from_device_blocks(blocks):
    """``modin.pandas.DataFrame`` over device blocks that already sit in this rank's HBM, one row partition per block
    -- the from_map-style ingest (modin/core/io/io.py:184-209; what
    ``modin.distributed.dataframe.pandas.from_partitions`` does for Ray object refs, partitions.py:154-264): no host
    frame is built and nothing is copied.  Blocks must share their column labels and carry RangeIndex labels that
    run on from each other (``synth.device_blocks``)."""
    ns = register()
    import modin.pandas as mpd

    blocks = list(blocks)
    if not blocks:
        raise ValueError("from_device_blocks needs at least one block")
    for b in blocks:
        if not b.has_range_index() or list(b.columns) != list(blocks[0].columns):
            raise NotImplementedError("from_device_blocks: range-indexed blocks with identical columns")
    pc = ns.PartitionManager._partition_class
    parts = np.array([[pc.put(b)] for b in blocks], dtype=object).reshape(len(blocks), 1)
    start = blocks[0].range_start
    index = pandas.RangeIndex(start, start + sum(b.nrows for b in blocks))
    frame = ns.Dataframe(parts, index, blocks[0].columns, [b.nrows for b in blocks], [len(blocks[0].cols)],
                         dtypes=blocks[0].dtypes)  # fmt: skip
    frame._b200_shard_offset = start  # this rank's first global row position (see merge.row_axis_merge)
    return mpd.DataFrame(query_compiler=ns.QueryCompiler(frame))


def activate():
    """``register()`` + ``modin.set_execution(engine="B200", storage_format="Arrow")``."""
    ns = register()
    import modin

    modin.set_execution(engine="B200", storage_format="Arrow")
    return ns
