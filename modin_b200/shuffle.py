"""Range-partitioning shuffle on the device (SURVEY.md §8 a13 / f2).

Reference: ``PandasDataframePartitionManager.shuffle_partitions`` (partition_manager.py:1937-2052) driven by a
``ShuffleFunctions`` object (modin/core/dataframe/pandas/dataframe/utils.py:111-475): sample the key column of every
row partition, pick pivots from the pooled samples (TeraSort), split every row partition into one piece per key
range (``np.digitize`` against the pivots), transpose, and run ``final_shuffle_func`` over the pieces of each range --
after which every key lives in exactly one partition and the partitions are in key order.

Here the same three callbacks work on device blocks:

* ``sample_fn``  strided sample of the key column's ORDER-PRESERVING int64 image (MB200_OP_ORDERED_S: float64 and
  int64 keys, NaN last, descending = bitwise NOT) -- a few thousand values, the only data that reaches the host;
* ``pivot_fn``   pools the samples (all-gathered across GPUs so that every rank picks the same pivots), sorts them
  and takes evenly spaced quantiles;
* ``split_fn``   bin id per row (``mb200_digitize_i64``), stable radix sort of (bin, row id), ONE gather of every
  column, pieces = row slices (views) at the bin boundaries.  Row labels travel as a device column.

Across GPUs there is one key range per rank and the transpose is one ``all_to_all`` of raw rows
(``dist.exchange_rows``): the NVLink shuffle of the north-star, used where pre-aggregation is impossible (sort).
"""

from __future__ import annotations

from typing import List

import numpy as np

from . import dist, ops
from .block import DeviceBlock, DeviceColumn, concat_rows
from .functors import DevFn, _check_block
from .groupkeys import fold_zero_sign


def _with_label_column(block: DeviceBlock) -> DeviceBlock:
    """Row labels as ONE device column (a RangeIndex block gets its labels materialised: they stop being a range
    the moment rows move)."""
    if block.index_host is not None:
        raise NotImplementedError("the device shuffle moves numeric row labels only (host-resident labels: use ignore_index)")
    if block.index_cols:
        if len(block.index_cols) != 1:
            raise NotImplementedError("the device shuffle does not move MultiIndex labels")
        return block
    return DeviceBlock(block.cols, block.columns, nrows=block.nrows, index_cols=[ops.iota(block.range_start, block.nrows)],
                       index_names=[None])  # fmt: skip


def key_image(block: DeviceBlock, key_position: int, ascending: bool) -> DeviceColumn:
    key = block.cols[key_position]
    if key.dtype not in (np.float64, np.int64):
        raise NotImplementedError("device range partitioning needs a float64 or int64 key column")
    if block.nrows == 0:
        return DeviceColumn.empty(0, np.int64)
    if key.dtype == np.float64:  # -0.0 and 0.0 tie: rows keep their order, as in pandas' stable sort
        return ops.map_columns("ordered_s", [fold_zero_sign(key)], s0=[0.0 if ascending else 1.0])[0]
    return ops.map_columns("ordered_s", [key], s0=[0 if ascending else 1])[0]


class DevShuffleFunctions:
    """``ShuffleSortFunctions`` (dfutils.py:111-475) for device blocks: ``sample_fn`` / ``pivot_fn`` / ``split_fn``."""

    SAMPLES_PER_PARTITION = 2048

    def __init__(self, key_position: int, ascending: bool = True, ideal_num_new_partitions: int = 1):
        self.key_position, self.ascending = int(key_position), bool(ascending)
        self.ideal = max(1, int(ideal_num_new_partitions))
        self.pivots: List[int] = []

    # -- 1. sample (dfutils.py:163-237)
    def sample_fn(self, block: DeviceBlock):
        _check_block(block, "DevShuffleFunctions.sample_fn")
        img = key_image(block, self.key_position, self.ascending)
        n = len(img)
        step = max(1, n // self.SAMPLES_PER_PARTITION)
        return img.data[::step].contiguous() if n else img.data

    # -- 2. pivots (dfutils.py:238-332)
    def pivot_fn(self, samples) -> int:
        t = ops.torch_mod()
        pool = t.cat([s.reshape(-1) for s in samples]) if samples else None
        if dist.is_distributed():
            dev = ops.current_device() if pool is None else pool.device
            pool = t.empty(0, dtype=t.int64, device=dev) if pool is None else pool
            pool = dist.all_gather_rows([pool])[0]
            nbins = dist.world_size()  # one key range per GPU
        else:
            nbins = self.ideal
        if pool is None or pool.numel() == 0 or nbins <= 1:
            self.pivots = [] if nbins <= 1 else [0] * (nbins - 1)
            return max(1, nbins)
        pool, _ = t.sort(pool)
        m = pool.numel()
        q = [min(m - 1, (i * m) // nbins) for i in range(1, nbins)]
        self.pivots = [int(v) for v in pool[t.as_tensor(q, device=pool.device)].tolist()]
        return nbins

    # -- 3. split (dfutils.py:355-475)
    def split_fn(self, block: DeviceBlock) -> List[DeviceBlock]:
        _check_block(block, "DevShuffleFunctions.split_fn")
        nbins = len(self.pivots) + 1
        block = _with_label_column(block)
        if nbins == 1:
            return [block]
        n = block.nrows
        labels = block.index_cols[0]
        if n == 0:
            return [block.slice_rows(0, 0) for _ in range(nbins)]
        bins = ops.digitize(key_image(block, self.key_position, self.ascending), self.pivots)
        perm = ops.iota(0, n)
        ops.sort_pairs(bins, perm)  # stable: rows of one bin keep their order
        moved = ops.take_columns(list(block.cols) + [labels], perm)
        # bin boundaries: heads of the runs of equal bin ids (<= nbins of them) -> host
        starts_np, present = ops.run_starts(bins)
        bounds = np.full(nbins + 1, n, dtype=np.int64)
        for b_id, s in zip(present, starts_np):
            bounds[int(b_id)] = int(s)
        have = {int(x) for x in present}
        for b_id in range(nbins - 1, -1, -1):  # bins that own no rows start where the next one does
            if b_id not in have:
                bounds[b_id] = bounds[b_id + 1]
        whole = DeviceBlock(moved[:-1], block.columns, nrows=n, index_cols=[moved[-1]], index_names=block.index_names or [None])
        return [whole.slice_rows(int(bounds[i]), int(bounds[i + 1])) for i in range(nbins)]


class DevSortBlock(DevFn):
    """``final_shuffle_func`` of a sort: stable sort of the rows of ONE key range by the key column (radix sort of
    (order-preserving image, row id), one gather per column); labels ride along as a device column."""

    op = "sort_block"

    def __init__(self, key_position: int, ascending: bool = True):
        self.key_position, self.ascending = int(key_position), bool(ascending)

    def __call__(self, block, *args, **kwargs):
        _check_block(block, "DevSortBlock")
        block = _with_label_column(block)
        n = block.nrows
        if n <= 1:
            return block
        img = key_image(block, self.key_position, self.ascending)
        perm = ops.iota(0, n)
        ops.sort_pairs(img, perm)
        moved = ops.take_columns(list(block.cols) + [block.index_cols[0]], perm)
        return DeviceBlock(moved[:-1], block.columns, nrows=n, index_cols=[moved[-1]], index_names=block.index_names or [None])


def exchange_pieces(pieces: List[DeviceBlock]) -> DeviceBlock:
    """The transpose step across GPUs: ``pieces[r]`` goes to rank r; what arrives (one piece per rank, in rank order,
    i.e. in original row order) is concatenated.  One ``all_to_all`` of the packed 8-byte columns + labels."""
    first = pieces[0]
    if any(c.dtype == np.bool_ for c in first.cols):
        raise NotImplementedError("the multi-GPU row shuffle moves 8-byte columns only (bool columns are not packed)")
    send_counts = [p.nrows for p in pieces]
    whole = concat_rows(pieces) if len(pieces) > 1 else first
    tensors = [c.data for c in whole.cols] + [whole.index_cols[0].data]
    received = dist.exchange_rows(tensors, send_counts)
    cols = [DeviceColumn(x, c.dtype) for x, c in zip(received[:-1], whole.cols)]
    lab = DeviceColumn(received[-1], whole.index_cols[0].dtype)
    return DeviceBlock(cols, first.columns, nrows=len(lab), index_cols=[lab], index_names=first.index_names or [None])
