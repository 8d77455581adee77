"""B200Dataframe: the core dataframe over a 2-D grid of device partitions.

Mirror of ``PandasDataframe`` (modin/core/dataframe/pandas/dataframe/dataframe.py) for the
methods on the hot path: ``map`` (:2253-2319), ``tree_reduce`` (:2208-2250) with
``_build_treereduce_func`` (:2081-2123) and ``_compute_tree_reduce_metadata`` (:2125-2168),
``n_ary_op`` (:3851-3950) with the ``_check_if_axes_identical`` fast path (:3678-3707),
``broadcast_apply`` (:3233-3335), ``broadcast_apply_full_axis`` (:3483-3676),
``groupby_reduce`` (:4530-4589), ``from_pandas`` / ``from_arrow`` / ``to_pandas``
(:4592-4722), ``combine``, ``finalize`` / ``wait_computations`` (:4780-4791).

Metadata (index, columns, dtypes, row lengths, column widths) lives on the host and is O(W) or
a ``RangeIndex``; a 1e9-row index is never materialised.  Under torch.distributed every rank
holds the row shard it owns: ``_partitions`` is the LOCAL grid, ``index`` the local labels, and
``global_nrows`` the job-wide row count.
"""

from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np
import pandas

from . import dist
from .block import DeviceBlock
from .functors import MODIN_UNNAMED_SERIES_LABEL
from .partitioning import B200PartitionManager


class B200Dataframe:
    _partition_mgr_cls = B200PartitionManager
    engine = "B200"
    storage_format = "Arrow"

    def __init__(self, partitions, index=None, columns=None, row_lengths=None, column_widths=None, dtypes=None,
                 pandas_backend=None):  # fmt: skip
        self._partitions = np.asarray(partitions, dtype=object)
        if self._partitions.ndim != 2:
            raise ValueError("partitions must be a 2-D grid")
        self._index_cache = index
        self._columns_cache = columns
        self._row_lengths_cache = list(row_lengths) if row_lengths is not None else None
        self._column_widths_cache = list(column_widths) if column_widths is not None else None
        self._dtypes = dtypes
        self._pandas_backend = pandas_backend
        self._filter_empties()

    @property
    def __constructor__(self):
        return type(self)

    # ---- metadata ----------------------------------------------------------------------------
    def _filter_empties(self):
        """Drop zero-length row / column partitions (df.py:582-640), keeping at least a 1x1 grid."""
        if self._partitions.size == 0:
            return
        rl = self.row_lengths
        cw = self.column_widths
        keep_r = [i for i, n in enumerate(rl) if n > 0] or [0]
        keep_c = [j for j, n in enumerate(cw) if n > 0] or [0]
        if len(keep_r) != len(rl) or len(keep_c) != len(cw):
            self._partitions = self._partitions[np.ix_(keep_r, keep_c)]
            self._row_lengths_cache = [rl[i] for i in keep_r]
            self._column_widths_cache = [cw[j] for j in keep_c]

    @property
    def row_lengths(self) -> List[int]:
        if self._row_lengths_cache is None:
            self._row_lengths_cache = [row[0].length() for row in self._partitions] if self._partitions.size else []
        return self._row_lengths_cache

    @property
    def column_widths(self) -> List[int]:
        if self._column_widths_cache is None:
            self._column_widths_cache = [p.width() for p in self._partitions[0]] if self._partitions.size else []
        return self._column_widths_cache

    @property
    def index(self) -> pandas.Index:
        if self._index_cache is None:
            self._index_cache, _ = self._partition_mgr_cls.get_indices(0, self._partitions)
        return self._index_cache

    @property
    def columns(self) -> pandas.Index:
        if self._columns_cache is None:
            self._columns_cache, _ = self._partition_mgr_cls.get_indices(1, self._partitions)
        return self._columns_cache

    @property
    def dtypes(self) -> pandas.Series:
        if self._dtypes is None:
            series = [p.get().dtypes for p in self._partitions[0]]
            self._dtypes = pandas.concat(series) if series else pandas.Series(dtype=object)
        return self._dtypes

    @property
    def has_materialized_dtypes(self):
        return self._dtypes is not None

    @property
    def has_materialized_index(self):
        return self._index_cache is not None

    @property
    def has_materialized_columns(self):
        return self._columns_cache is not None

    def __len__(self):
        return sum(self.row_lengths)

    @property
    def global_nrows(self) -> int:
        """Job-wide row count (sum over ranks of the local shard lengths)."""
        n = len(self)
        if dist.is_distributed() and not self._is_replicated():
            import torch

            t = torch.tensor([n], dtype=torch.int64, device=self._any_device())
            dist.all_reduce_values([t], ["sum"])
            n = int(t.item())
        return n

    def _any_device(self):
        for p in self._partitions.flatten():
            b = p.get()
            if b.cols:
                return b.cols[0].data.device
        from .block import current_device

        return current_device()

    def _is_replicated(self) -> bool:
        return all(p.get().replicated for p in self._partitions.flatten())

    def copy_index_cache(self, copy_lengths=False):
        return self._index_cache

    def copy_columns_cache(self, copy_lengths=False):
        return self._columns_cache

    def copy_dtypes_cache(self):
        return self._dtypes

    def copy(self):
        return self.__constructor__(self._partitions, self._index_cache, self._columns_cache,
                                    self._row_lengths_cache, self._column_widths_cache, self._dtypes)  # fmt: skip

    # ---- Map ------------------------------------------------------------------------------------
    def map(self, func: Callable, dtypes=None, new_columns=None, func_args=None, func_kwargs=None, lazy=False):
        """df.py:2253-2319."""
        map_fn = self._partition_mgr_cls.lazy_map_partitions if lazy else self._partition_mgr_cls.map_partitions
        new_partitions = map_fn(self._partitions, func, func_args, func_kwargs)
        if new_columns is not None and self.has_materialized_columns:
            assert len(new_columns) == len(self.columns), \
                "New column's length must be identical to the previous columns"  # fmt: skip
        elif new_columns is None:
            new_columns = self.copy_columns_cache(copy_lengths=True)
        if isinstance(dtypes, str) and dtypes == "copy":
            dtypes = self.copy_dtypes_cache()
        elif dtypes is not None and not isinstance(dtypes, pandas.Series):
            dtypes = pandas.Series([pandas.api.types.pandas_dtype(dtypes)] * len(self.columns), index=new_columns)
        return self.__constructor__(new_partitions, self.copy_index_cache(copy_lengths=True), new_columns,
                                    self._row_lengths_cache, self._column_widths_cache, dtypes=dtypes)  # fmt: skip

    # ---- TreeReduce -------------------------------------------------------------------------------
    def _build_treereduce_func(self, axis, func):
        """df.py:2081-2123.  Device reduce functors already return the 1 x W block labelled
        ``__reduced__`` that the reference builds from the pandas Series, so this is the identity
        for them; anything else is rejected (no pandas on this path)."""
        return func

    def _compute_tree_reduce_metadata(self, axis, new_parts, dtypes=None):
        """df.py:2125-2168."""
        new_axes, new_axes_lengths = [0, 0], [0, 0]
        new_axes[axis] = pandas.Index([MODIN_UNNAMED_SERIES_LABEL])
        new_axes[axis ^ 1] = self.columns if axis == 0 else self.index
        new_axes_lengths[axis] = [1]
        new_axes_lengths[axis ^ 1] = self.column_widths if axis == 0 else self.row_lengths
        if dtypes == "copy":
            dtypes = self.copy_dtypes_cache()
        elif dtypes is not None:
            dtypes = pandas.Series([pandas.api.types.pandas_dtype(dtypes)] * len(new_axes[1]), index=new_axes[1])
        return self.__constructor__(new_parts, *new_axes, *new_axes_lengths, dtypes)

    def tree_reduce(self, axis, map_func: Callable, reduce_func: Optional[Callable] = None, dtypes=None):
        """df.py:2208-2250: map every block to a 1 x W partial, then reduce each column partition's
        partials (plus an all_reduce across GPUs, issued by the reduce-phase functor itself)."""
        if axis != 0:
            raise NotImplementedError("tree_reduce along axis=1 is not on the B200 path")
        map_func = self._build_treereduce_func(axis, map_func)
        reduce_func = map_func if reduce_func is None else self._build_treereduce_func(axis, reduce_func)
        map_parts = self._partition_mgr_cls.map_partitions(self._partitions, map_func)
        reduce_parts = self._partition_mgr_cls.map_axis_partitions(axis, map_parts, reduce_func, num_splits=1)
        return self._compute_tree_reduce_metadata(axis, reduce_parts, dtypes=dtypes)

    def reduce(self, axis, function: Callable, dtypes=None):
        """df.py:2171-2205: ``function`` over every FULL column partition -> 1 x W (the Reduce template).  The
        device functor sees this rank's blocks of the axis and finishes with its own collective."""
        if axis != 0:
            raise NotImplementedError("reduce along axis=1 is not on the B200 path")
        function = self._build_treereduce_func(axis, function)
        new_parts = self._partition_mgr_cls.map_axis_partitions(axis, self._partitions, function, num_splits=1)
        return self._compute_tree_reduce_metadata(axis, new_parts, dtypes=dtypes)

    def fold(self, axis, func: Callable, new_index=None, new_columns=None, shape_preserved=False):
        """df.py:2357-2400: ``func`` over every FULL column partition, partitioning kept (the Fold template)."""
        if axis != 0:
            raise NotImplementedError("fold along axis=1 is not on the B200 path")
        row_lengths = column_widths = None
        if shape_preserved:
            new_index = self.copy_index_cache(copy_lengths=True) if new_index is None else new_index
            new_columns = self.copy_columns_cache(copy_lengths=True) if new_columns is None else new_columns
            row_lengths, column_widths = self._row_lengths_cache, self._column_widths_cache
        new_parts = self._partition_mgr_cls.map_axis_partitions(axis, self._partitions, func, keep_partitioning=True)
        return self.__constructor__(new_parts, new_index, new_columns, row_lengths, column_widths)

    # ---- Binary -----------------------------------------------------------------------------------
    def hstack(self, other: "B200Dataframe") -> "B200Dataframe":
        """Columns of ``self`` followed by the columns of ``other`` (same rows, same row labels): the column half of
        ``PandasDataframe.concat(axis=1)`` (df.py:3952-4096) for operands that only need their row cuts aligned.
        Buffers are shared; up to 32 columns stay one column partition."""
        from .block import concat_cols

        other = self._align_rows_like(other, "column assignment")  # pandas aligns on the frame's row labels
        if len(set(self.columns) & set(other.columns)):
            raise ValueError("hstack needs distinct column labels")
        pc = self._partition_mgr_cls._partition_class
        total = len(self.columns) + len(other.columns)
        new_rows = []
        for row, orow in zip(self._partitions, other._partitions):
            if total <= 32:
                new_rows.append([pc(concat_cols([p.get() for p in row] + [p.get() for p in orow]))])
            else:
                new_rows.append(list(row) + list(orow))
        parts = np.array(new_rows, dtype=object).reshape(len(new_rows), -1)
        widths = [total] if total <= 32 else list(self.column_widths) + list(other.column_widths)
        return self.__constructor__(parts, self._index_cache, self.columns.append(other.columns), self._row_lengths_cache,
                                    widths, None)  # fmt: skip

    def head_rows(self, n: int) -> "B200Dataframe":
        """First ``n`` rows of the job-wide frame (views of the first partitions' buffers)."""
        n = max(int(n), 0)
        lo = dist.exclusive_row_offset(len(self)) if dist.is_distributed() else 0
        take = max(0, min(len(self), n - lo))
        return self._slice_local(0, take)

    def tail_rows(self, n: int) -> "B200Dataframe":
        n = max(int(n), 0)
        total = self.global_nrows
        lo = dist.exclusive_row_offset(len(self)) if dist.is_distributed() else 0
        start = max(0, (total - n) - lo)
        return self._slice_local(min(start, len(self)), len(self))

    def _slice_local(self, start: int, stop: int) -> "B200Dataframe":
        cut = self._repartition_rows([start, stop - start, len(self) - stop])
        bounds = np.cumsum([0] + list(cut.row_lengths))
        keep = [i for i in range(len(cut.row_lengths)) if bounds[i] >= start and bounds[i + 1] <= stop and cut.row_lengths[i]]
        if not keep:  # empty selection: a zero-row view of the first partition
            pc = self._partition_mgr_cls._partition_class
            parts = np.array([[pc(p.get().slice_rows(0, 0)) for p in self._partitions[0]]], dtype=object)
            return self.__constructor__(parts, None, self._columns_cache, None, self._column_widths_cache, self._dtypes)
        return self.__constructor__(cut._partitions[keep, :], None, self._columns_cache, [cut.row_lengths[i] for i in keep],
                                    self._column_widths_cache, self._dtypes)  # fmt: skip

    def relabel_columns(self, new_labels: pandas.Index) -> "B200Dataframe":
        """New column labels over the same column buffers (no kernel, no copy)."""
        bounds = np.cumsum([0] + list(self.column_widths))
        pc = self._partition_mgr_cls._partition_class
        new_rows = []
        for row in self._partitions:
            new_row = []
            for j, p in enumerate(row):
                blk = p.get()
                new_row.append(pc(blk.with_cols(blk.cols, new_labels[bounds[j] : bounds[j + 1]])))
            new_rows.append(new_row)
        parts = np.array(new_rows, dtype=object).reshape(self._partitions.shape)
        dtypes = None
        if self._dtypes is not None:
            dtypes = self._dtypes.copy()
            dtypes.index = new_labels
        return self.__constructor__(parts, self._index_cache, new_labels, self._row_lengths_cache,
                                    self._column_widths_cache, dtypes)  # fmt: skip

    def rowwise_to_column(self, func) -> "B200Dataframe":
        """``func(whole row block) -> one-column block`` per row partition (a row-wise reduction such as
        ``all(axis=1)``): same row partitioning and row labels, one column partition."""
        from .block import concat_cols

        pc = self._partition_mgr_cls._partition_class
        new_rows = []
        for row in self._partitions:
            blk = concat_cols([p.get() for p in row]) if len(row) > 1 else row[0].get()
            new_rows.append([pc(func(blk))])
        parts = np.array(new_rows, dtype=object).reshape(len(new_rows), 1)
        return self.__constructor__(parts, self._index_cache, None, self._row_lengths_cache, [1], None)

    def filter_rows(self, mask: "B200Dataframe") -> "B200Dataframe":
        """Rows where the one-column bool frame ``mask`` is True (boolean indexing; no cross-partition movement:
        every row partition is compacted on its own, so the result keeps the partitioning and the row order)."""
        from .functors import DevRowFilter

        if len(mask.columns) != 1:
            raise NotImplementedError("row selection takes a one-column bool mask")
        if not self.index.equals(mask.index):
            # pandas (check_bool_indexer): the mask is re-indexed on the frame's labels and must cover all of them
            if not mask.index.is_unique or not self.index.isin(mask.index).all():
                raise pandas.errors.IndexingError(
                    "Unalignable boolean Series provided as indexer (index of the boolean Series and of the indexed "
                    "object do not match)."
                )
        mask = self._align_rows_like(mask, "boolean mask")
        from .block import concat_cols

        pc = self._partition_mgr_cls._partition_class
        fn = DevRowFilter()
        new_rows = []
        for row, mrow in zip(self._partitions, mask._partitions):
            blk = concat_cols([p.get() for p in row]) if len(row) > 1 else row[0].get()
            new_rows.append([pc(fn(blk, mrow[0].get()))])
        parts = np.array(new_rows, dtype=object).reshape(len(new_rows), 1)
        return self.__constructor__(parts, None, self._columns_cache, None, None, self._dtypes)

    def sort_by(self, col_position: int, ascending: bool = True, ignore_index: bool = False) -> "B200Dataframe":
        """Stable sort of the rows by one float64 / int64 column (NaN last) -- the device form of
        ``PandasDataframe.sort_by`` (df.py:2741-2791), which range-partitions the rows by sampled pivots
        (``_apply_func_to_range_partitioning`` df.py:2565-2739) and sorts every range with pandas.

        Here the same shuffle on the device (``partition manager.shuffle_partitions`` with ``DevShuffleFunctions``):
        sample the key's order-preserving int64 image, pivots from the pooled samples, every row partition split by
        ``digitize`` + stable radix sort + one gather, and each key range sorted by ``DevSortBlock`` (stable LSD radix
        sort of (image, row id), one gather per column).  Across GPUs there is one range per rank and the transpose
        is ONE all_to_all of raw rows over NVLink; rank r ends up with the r-th key range, ties in original row
        order.  Row labels travel as a device index column."""
        from .block import DeviceBlock, concat_cols
        from .config import NPartitions
        from .shuffle import DevShuffleFunctions, DevSortBlock

        # one column partition per row (a row block spans every column partition on the device path: zero-copy)
        pc = self._partition_mgr_cls._partition_class
        parts = self._partitions
        if parts.shape[1] > 1:
            parts = np.array([[pc(concat_cols([p.get() for p in row]))] for row in parts], dtype=object)
        first = parts[0, 0].get()
        if first.cols[col_position].dtype not in (np.float64, np.int64):
            raise NotImplementedError("device sort_values needs a float64 or int64 key column")
        if any(row[0].get().index_host is not None for row in parts) and not ignore_index:
            raise NotImplementedError("sort_values keeps host-resident (non-numeric) row labels only with ignore_index=True")
        if ignore_index:  # labels are dropped anyway: give every block a throw-away range so that none is host-resident
            parts = np.array([[pc(DeviceBlock(row[0].get().cols, row[0].get().columns, nrows=row[0].get().nrows))]
                              for row in parts], dtype=object)  # fmt: skip
        nbins = 1 if dist.is_distributed() else min(NPartitions.get(), max(1, len(self) // (1 << 16)))
        if nbins == 1 and len(parts) > 1 and not dist.is_distributed():
            # one new partition wanted, several held: gather the rows and apply the function once
            # (``combine_and_apply``, df.py:2565-2739 ``_apply_func_to_range_partitioning``)
            from .block import concat_rows
            from .shuffle import _with_label_column

            parts = np.array([[pc(concat_rows([_with_label_column(row[0].get()) for row in parts]))]], dtype=object)
        shuffle = DevShuffleFunctions(col_position, ascending, ideal_num_new_partitions=max(1, nbins))
        new_parts = self._partition_mgr_cls.shuffle_partitions(parts, 0, shuffle, DevSortBlock(col_position, ascending))
        if len(new_parts) > 1 and all(len(row) == 1 for row in new_parts):
            pass
        lengths = [row[0].get().nrows for row in new_parts]
        if ignore_index:
            offset = dist.exclusive_row_offset(sum(lengths)) if dist.is_distributed() else 0
            rows = []
            for row, n in zip(new_parts, lengths):
                b = row[0].get()
                rows.append([pc(DeviceBlock(b.cols, b.columns, nrows=n, range_start=offset))])
                offset += n
            new_parts = np.array(rows, dtype=object)
        return self.__constructor__(new_parts, None, self._columns_cache, lengths, [len(first.cols)], self._dtypes)

    def drop_duplicate_rows(self, col_position: int, keep: str = "first", ignore_index: bool = False) -> "B200Dataframe":
        """Rows holding the first / last occurrence of every value of one int64 column, in row order
        (``DevDropDuplicates``).  Across GPUs the keys of every rank's own survivors are all-gathered in rank order,
        the same pass names the job-wide winners and every rank keeps its own: the result stays row-sharded."""
        from .block import concat_cols, concat_rows
        from .functors import DevDropDuplicates

        rows = [concat_cols([p.get() for p in row]) if len(row) > 1 else row[0].get() for row in self._partitions]
        block = concat_rows(rows) if len(rows) > 1 else rows[0]
        out = DevDropDuplicates()(block, col_position, keep=keep, ignore_index=ignore_index)
        pc = self._partition_mgr_cls._partition_class
        return self.__constructor__(np.array([[pc(out)]], dtype=object), None, self._columns_cache, [out.nrows],
                                    [len(out.cols)], self._dtypes)  # fmt: skip

    def _repartition_rows(self, lengths: List[int]) -> "B200Dataframe":
        """Same rows, cut at ``lengths`` instead of ``self.row_lengths`` (the row half of ``_copartition``,
        df.py:3799-3840, without a reindex): target partitions inside one source partition are views of its
        buffers; a target partition that spans several sources is a device-to-device concatenation."""
        from .block import concat_rows

        src_bounds = np.cumsum([0] + list(self.row_lengths))
        ncolparts = self._partitions.shape[1] if self._partitions.size else 0
        pc = self._partition_mgr_cls._partition_class
        new_rows, pos = [], 0
        for L in lengths:
            lo, hi = pos, pos + int(L)
            row = []
            for j in range(ncolparts):
                pieces = []
                for i in range(len(self.row_lengths)):
                    a, b = max(lo, int(src_bounds[i])), min(hi, int(src_bounds[i + 1]))
                    if b > a:
                        pieces.append(self._partitions[i, j].get().slice_rows(a - int(src_bounds[i]), b - int(src_bounds[i])))
                if not pieces:  # empty target partition
                    pieces = [self._partitions[0, j].get().slice_rows(0, 0)]
                row.append(pc(concat_rows(pieces) if len(pieces) > 1 else pieces[0]))
            new_rows.append(row)
            pos = hi
        parts = np.array(new_rows, dtype=object).reshape(len(lengths), ncolparts)
        return self.__constructor__(parts, self._index_cache, self._columns_cache, list(lengths), self._column_widths_cache,
                                    self._dtypes)  # fmt: skip

    def _reindex_rows(self, labels: pandas.Index, lengths: List[int]) -> "B200Dataframe":
        """This frame's rows re-labelled to ``labels`` (missing labels -> NaN rows) and cut at ``lengths``: the
        ``map_axis_partitions(0, parts, make_reindexer(...), lengths=base_lengths)`` step of
        ``PandasDataframe._copartition`` (df.py:3799-3840) -- every column partition is gathered along the rows,
        re-indexed on the device (``DevReindex``) and split again."""
        from .functors import DevReindex
        from .partitioning import Bound

        if dist.is_distributed() and not self._is_replicated():
            # the labels to align against live on the other ranks too; every rank refuses together
            raise NotImplementedError("label alignment between row-sharded frames is not on the B200 path")
        parts = self._partition_mgr_cls.map_axis_partitions(
            0, self._partitions, Bound(DevReindex(), (labels,), {"axis": 0}), lengths=list(lengths))
        return self.__constructor__(parts, labels, self._columns_cache, list(lengths), self._column_widths_cache, None)

    def _copartition_rows(self, others: list, how: str = "outer", sort=None):
        """``_copartition(axis=0, ...)`` (df.py:3709-3848): join the row labels of ``self`` and ``others``
        (``how`` = "outer" for binary operators, "left" for assignments / masks / group keys; pandas sorts the joined
        index when the labels differ, df.py:3759-3760) and bring every frame to the joined labels and to the same
        row cuts.  Returns ``(self', others')``; frames whose labels already equal the joined index are only re-cut."""
        if all(self._check_if_axes_identical(o, 0) for o in others):
            return self, list(others)
        if sort is None:
            sort = not all(self.index.equals(o.index) for o in others)
        joined = self.index
        for o in others:
            if not joined.equals(o.index):
                joined = joined.join(o.index, how=how, sort=sort)
        base = self if self.index.equals(joined) else None
        lengths = self.row_lengths if base is not None else None
        if lengths is None:
            from .partitioning import get_length_list
            from .config import MinRowPartitionSize, NPartitions

            lengths = [n for n in get_length_list(len(joined), NPartitions.get(), MinRowPartitionSize.get()) if n] or [0]
        new_self = self if base is not None else self._reindex_rows(joined, lengths)
        out = []
        for o in others:
            if o.index.equals(joined):
                out.append(o if o.row_lengths == list(lengths) else o._repartition_rows(list(lengths)))
            else:
                out.append(o._reindex_rows(joined, lengths))
        return new_self, out

    def _align_rows_like(self, other: "B200Dataframe", what: str) -> "B200Dataframe":
        """``other`` brought to THIS frame's row labels and cuts (pandas aligns an assigned Series, a boolean mask or
        a group-key Series on the frame's index -- a left join of the labels)."""
        if self.index.equals(other.index):
            return other if other.row_lengths == self.row_lengths else other._repartition_rows(self.row_lengths)
        if not other.index.is_unique:
            raise ValueError("cannot reindex on an axis with duplicate labels")
        return other._reindex_rows(self.index, self.row_lengths)

    def _check_if_axes_identical(self, other: "B200Dataframe", axis: int = 0) -> bool:
        """df.py:3678-3707."""
        if axis == 0:
            return self.index.equals(other.index) and self.row_lengths == other.row_lengths
        return self.columns.equals(other.columns) and self.column_widths == other.column_widths

    def n_ary_op(self, op, right_frames: list, join_type="outer", copartition_along_columns=True, labels="replace",
                 dtypes=None, sort=None):  # fmt: skip
        """df.py:3851-3950.  Row labels go through ``_copartition`` (df.py:3709-3848): identical labels and cuts are
        the no-op fast path (df.py:3750-3758), equal labels with other cuts are re-cut (views), different labels are
        joined (outer, sorted -- pandas' alignment of binary operators) and every frame is re-indexed on the device
        (``DevReindex``).  Column labels must already agree."""
        left = self
        for other in right_frames:
            if not (self.columns.equals(other.columns) and self.column_widths == other.column_widths):
                raise NotImplementedError(
                    "binary op between frames with different COLUMN labels is not on the B200 path "
                    "(row labels are aligned; select / rename the columns first)"
                )
        # row labels: identical -> no-op; same labels, other cuts -> re-cut; different labels -> the join + reindex
        # of _copartition (df.py:3709-3848)
        left, aligned = self._copartition_rows(list(right_frames), how=join_type if join_type in ("outer", "left", "inner") else "outer",
                                               sort=sort)  # fmt: skip
        if left is not self:
            new_frame = left._partition_mgr_cls.n_ary_operation(left._partitions, op, [o._partitions for o in aligned])
            return self.__constructor__(new_frame, left._index_cache, left._columns_cache, left._row_lengths_cache,
                                        left._column_widths_cache, None)  # fmt: skip
        new_frame = self._partition_mgr_cls.n_ary_operation(
            self._partitions, op, [other._partitions for other in aligned]
        )
        return self.__constructor__(new_frame, self._index_cache, self._columns_cache, self._row_lengths_cache,
                                    self._column_widths_cache, dtypes)  # fmt: skip

    def broadcast_apply(self, axis, func, other, join_type="left", copartition=True, labels="keep", dtypes=None):
        """df.py:3233-3335: every block gets the matching slice of ``other`` along ``axis``."""
        if not self._check_if_axes_identical(other, axis):
            raise NotImplementedError("broadcast_apply needs co-partitioned operands on the B200 path")
        new_frame = self._partition_mgr_cls.broadcast_apply(axis, func, self._partitions, other._partitions)
        return self.__constructor__(new_frame, self._index_cache, self._columns_cache, self._row_lengths_cache,
                                    self._column_widths_cache, dtypes)  # fmt: skip

    def broadcast_apply_full_axis(self, axis, func, other, new_index=None, new_columns=None, apply_indices=None,
                                  enumerate_partitions=False, dtypes=None, keep_partitioning=True, num_splits=None,
                                  sync_labels=True, pass_axis_lengths_to_partitions=False):  # fmt: skip
        """df.py:3483-3676: apply ``func(full_axis_block, other_frame_block)`` to every row (axis=1) or
        column (axis=0) of the grid with ``other`` broadcast whole."""
        if other is not None:
            others = other if isinstance(other, list) else [other]
            other_parts = [o._partitions for o in others]
        else:
            other_parts = None
        new_partitions = self._partition_mgr_cls.broadcast_axis_partitions(
            axis=axis, left=self._partitions, right=other_parts[0] if other_parts else None, apply_func=func,
            apply_indices=apply_indices, enumerate_partitions=enumerate_partitions, keep_partitioning=keep_partitioning,
            num_splits=1 if num_splits is None else num_splits,
        )  # fmt: skip
        return self.__constructor__(new_partitions, new_index, new_columns, None, None, dtypes)

    # ---- GroupByReduce ----------------------------------------------------------------------------
    def groupby_reduce(self, axis, by, map_func, reduce_func, new_index=None, new_columns=None, apply_indices=None):
        """df.py:4530-4589."""
        if by is not None and not (self.index.equals(by.index) and self.row_lengths == by.row_lengths):
            if not self.index.equals(by.index) and not self.index.isin(by.index).all():
                # pandas would group the uncovered rows under NaN keys and drop them: float keys are not on the path
                raise NotImplementedError("group keys that do not cover every row label are not on the B200 path")
            by = self._align_rows_like(by, "group keys")
        by_parts = by if by is None else by._partitions
        new_partitions = self._partition_mgr_cls.groupby_reduce(axis, self._partitions, by_parts, map_func, reduce_func,
                                                                apply_indices)  # fmt: skip
        return self.__constructor__(new_partitions, new_index, new_columns)

    # ---- structure ---------------------------------------------------------------------------------
    def combine(self):
        """pm.combine (pm.py:1328-1373): one partition holding the whole frame (all ranks' rows)."""
        parts = self._partition_mgr_cls.combine(self._partitions)
        return self.__constructor__(parts, None, self._columns_cache, None, None, self._dtypes)

    def take_2d_labels_or_positional(self, row_positions=None, col_positions=None):
        """Column selection by position (subset of df.py:1188-1389): buffers are shared."""
        if row_positions is not None:
            raise NotImplementedError("row selection is not on the B200 path")
        cols = list(col_positions)
        widths = self.column_widths
        bounds = np.cumsum([0] + widths)
        new_rows = []
        for row in self._partitions:
            blocks = [p.get() for p in row]
            picked = []
            for c in cols:
                j = int(np.searchsorted(bounds, c, side="right") - 1)
                picked.append(blocks[j].select_columns([c - bounds[j]]))
            from .block import concat_cols

            blk = concat_cols(picked) if len(picked) > 1 else picked[0]
            new_rows.append([self._partition_mgr_cls._partition_class(blk)])
        new_cols = self.columns[cols]
        dt = self._dtypes.iloc[cols] if self._dtypes is not None else None
        return self.__constructor__(np.array(new_rows), self._index_cache, new_cols, self._row_lengths_cache,
                                    [len(cols)], dt)  # fmt: skip

    # ---- ingest / egress ----------------------------------------------------------------------------
    @classmethod
    def from_pandas(cls, df: pandas.DataFrame):
        """df.py:4592-4620."""
        new_index = df.index
        new_columns = df.columns
        new_dtypes = df.dtypes
        parts, _, row_lengths, col_widths = cls._partition_mgr_cls.from_pandas(df, return_dims=True)
        lo = 0
        if dist.is_distributed():
            lo, hi = dist.shard_bounds(len(df))
            new_index = new_index[lo:hi]
        frame = cls(parts, new_index, new_columns, row_lengths, col_widths, dtypes=new_dtypes)
        frame._b200_shard_offset = lo  # this rank's first global row position (a fresh ingest: rows are in job order)
        return frame

    @classmethod
    def from_arrow(cls, at):
        """df.py:4622-4654."""
        parts, _, row_lengths, col_widths = cls._partition_mgr_cls.from_arrow(at, return_dims=True)
        return cls(parts, None, pandas.Index(at.column_names), row_lengths, col_widths)

    @classmethod
    def from_blocks(cls, blocks: List[DeviceBlock]):
        """Frame from device blocks already resident on this rank (from_map-style ingest,
        modin/core/io/io.py:184-209): one row partition per block."""
        pc = cls._partition_mgr_cls._partition_class
        parts = np.array([[pc.put(b)] for b in blocks], dtype=object)
        first = blocks[0]
        index = None
        if all(b.has_range_index() for b in blocks):
            index = pandas.RangeIndex(first.range_start, first.range_start + sum(b.nrows for b in blocks))
        return cls(parts, index, first.columns, [b.nrows for b in blocks], [len(first.cols)], dtypes=first.dtypes)

    def __dataframe__(self, nan_as_null: bool = False, allow_copy: bool = True):
        """df.py:4803-4824: the interchange-protocol view of this frame -- device buffers, one chunk per row
        partition (``modin_b200.interchange``)."""
        from .block import concat_cols
        from .interchange import B200ProtocolDataframe

        blocks = [concat_cols([p.get() for p in row]) if len(row) > 1 else row[0].get() for row in self._partitions]
        return B200ProtocolDataframe(blocks, self.index, nan_as_null, allow_copy)

    @classmethod
    def from_interchange_dataframe(cls, df):
        """df.py:4826-4867 -- without the detour through pandas: CUDA buffers are adopted through DLPack, host
        buffers are copied H2D."""
        if type(df) is cls:
            return df
        from .interchange import blocks_from_dataframe

        return cls.from_blocks(blocks_from_dataframe(df))

    def to_pandas(self) -> pandas.DataFrame:
        """df.py:4691-4722."""
        df = self._partition_mgr_cls.to_pandas(self._partitions)
        if len(df.columns) == 0 and self._columns_cache is not None and len(self._columns_cache):
            df = pandas.DataFrame(columns=self._columns_cache, index=df.index)
        return df

    def to_numpy(self, **kwargs):
        return self._partition_mgr_cls.to_numpy(self._partitions, **kwargs)

    def finalize(self):
        self._partition_mgr_cls.finalize(self._partitions)

    def wait_computations(self):
        self._partition_mgr_cls.wait_partitions(self._partitions.flatten())
