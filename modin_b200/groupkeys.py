"""Group keys of a device groupby, for both front doors: how the keys become the ONE int64 key column the single-key
device groupby runs on (``key_image``), how the result's keys are restored (``restore_keys``), and how a dictionary
aggregation is split per function and zipped back (``split_aggregations`` / ``zip_aggregations``).  Everything here
works on lists of device blocks, one per row partition; each front door wraps them into its own frame type.

Several int64 keys are packed.  The reference hands ``df.groupby([...])`` to pandas per block (alg/groupby.py:124-208),
which builds a combined group index with ``get_group_index``.  Here the key tuples are packed into one int64 on the
device, ``sum_i (k_i - min_i) * stride_i`` with ``stride_i = prod_{j>i} (max_j - min_j + 1)``, the single-key device
groupby (dense or hashed table) runs on the image, and the G result keys are unpacked afterwards -- per row one
subtract + multiply per key column and k - 1 adds; per GROUP one divmod on the host (result-sized, not row-sized).  The
key ranges come from the columns' cached statistics (``ops.key_stats``), agreed across ranks once.
"""

from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np
import pandas

from . import dist, ops
from .block import DeviceBlock, DeviceColumn

PACKED_KEY = "__packed_key__"
FLOAT_KEY = "float64 image"  # the restore description of one float64 key (``key_image``)


def packing_plan(key_blocks: Sequence[DeviceBlock]):
    """(mins, ranges, strides) for the key columns of ``key_blocks`` (one block per row partition, identical columns),
    identical on every rank."""
    k = len(key_blocks[0].cols)
    for b in key_blocks:
        for c in b.cols:
            if c.dtype != np.int64:
                raise NotImplementedError("multi-column groupby on the B200 path needs int64 key columns")
    mins, maxs = [], []
    for p in range(k):
        lo, hi = ops.key_stats([b.cols[p] for b in key_blocks])[:2]
        if dist.is_distributed():
            t = ops.torch_mod()
            per_rank = dist.all_gather_small(t.tensor([lo, hi], dtype=t.int64, device=ops.current_device()))
            lo, hi = min(r[0] for r in per_rank), max(r[1] for r in per_rank)
        if lo > hi:
            lo = hi = 0  # no rows anywhere
        mins.append(lo)
        maxs.append(hi)
    ranges = [hi - lo + 1 for lo, hi in zip(mins, maxs)]
    strides = [1] * k
    for i in range(k - 2, -1, -1):
        strides[i] = strides[i + 1] * ranges[i + 1]
    if strides[0] * ranges[0] >= 1 << 62:
        raise NotImplementedError("the key ranges of this multi-column groupby do not pack into 62 bits")
    return mins, ranges, strides


def pack(block: DeviceBlock, plan) -> DeviceColumn:
    """Packed key column of one block of key columns."""
    mins, _ranges, strides = plan
    packed = None
    for c, lo, s in zip(block.cols, mins, strides):
        if not block.nrows:
            return DeviceColumn.empty(0, np.int64)
        # (key - lo) * stride, in that order: -lo * stride alone need not fit int64, the difference always does
        term = ops.map_columns("mul_s", ops.map_columns("sub_s", [c], s0=[lo]), s0=[s])[0]
        packed = term if packed is None else ops.map_columns("add", [packed], [term])[0]
    return packed


def unpack(packed: DeviceColumn, plan) -> List[DeviceColumn]:
    """The original key columns of G packed result keys (host divmod on G values)."""
    mins, ranges, strides = plan
    host = packed.to_numpy().astype(np.int64)
    return [DeviceColumn.from_numpy(((host // s) % r + lo).astype(np.int64)) for lo, r, s in zip(mins, ranges, strides)]


# ---- float64 group keys ------------------------------------------------------------------------------------------
_I64_MAX = np.iinfo(np.int64).max
_MAG = np.int64(0x7FFFFFFFFFFFFFFF)


def float_image(key: DeviceColumn) -> DeviceColumn:
    """Order-preserving int64 image of a float64 key column: ``-0.0`` folded into ``0.0`` first (pandas groups them
    together), then the total order of IEEE doubles as a signed integer (``MB200_OP_ORDERED_S``, the map the device
    sort uses); every NaN becomes INT64_MAX, i.e. ONE group that sorts last -- where ``dropna`` finds it."""
    if key.dtype != np.float64:
        raise TypeError("float_image takes a float64 column")
    if not len(key):
        return DeviceColumn.empty(0, np.int64)
    return ops.map_columns("ordered_s", [fold_zero_sign(key)], s0=[0])[0]


def fold_zero_sign(key: DeviceColumn) -> DeviceColumn:
    """``key + 0.0``: ``-0.0`` becomes ``0.0``, every other value is unchanged (NaN stays NaN).  pandas treats the
    two zeros as one key when it groups, sorts (ties, kept in row order) and matches labels, so every order-preserving
    image of a float64 key is taken from this column, never from the raw bits."""
    return ops.map_columns("add_s", [key], s0=[0.0])[0]


def float_keys(image: DeviceColumn) -> np.ndarray:
    """The float64 keys behind G image values (host arithmetic on G numbers: the image map is its own inverse)."""
    img = image.to_numpy().astype(np.int64)
    bits = img ^ ((img >> np.int64(63)) & _MAG)
    keys = bits.view(np.float64).copy()
    keys[img == _I64_MAX] = np.nan
    return keys


# ---- the key image and the restore -------------------------------------------------------------------------------
def key_image(key_blocks: List[DeviceBlock]):
    """(image blocks, restore description) for the key columns of a groupby, one block per row partition.

    One int64 key: the blocks themselves and ``None`` -- nothing is launched or allocated.  One float64 key: its
    order-preserving image under the key's own label (``float_image``) and ``FLOAT_KEY``.  Several int64 keys: their
    packed image labelled ``PACKED_KEY`` and ``(packing plan, key labels)``."""
    first = key_blocks[0]
    if len(first.cols) > 1:
        plan = packing_plan(key_blocks)
        label = pandas.Index([PACKED_KEY])
        images = [DeviceBlock([pack(b, plan)], label, nrows=b.nrows, range_start=b.range_start) for b in key_blocks]
        return images, (plan, list(first.columns))
    if first.cols[0].dtype == np.float64:
        return [DeviceBlock([float_image(b.cols[0])], b.columns, nrows=b.nrows, range_start=b.range_start)
                for b in key_blocks], FLOAT_KEY  # fmt: skip
    return key_blocks, None


def restore_keys(blocks: List[DeviceBlock], image, dropna: bool = True, names=None) -> List[DeviceBlock]:
    """Result blocks of a groupby on ``key_image``'s image, with the original keys as index columns: unpacked
    several keys, or the float64 keys -- whose NaN group (the last row, if any) is dropped under ``dropna``.  ``names``
    replaces the index names (``groupby(level=)``: the level's name)."""
    out = []
    for b in blocks:
        keys, key_names = b.index_cols, b.index_names
        if image == FLOAT_KEY:
            host = float_keys(keys[0]) if b.nrows else np.zeros(0, dtype=np.float64)
            if dropna and b.nrows and np.isnan(host[-1]):
                b, host = b.slice_rows(0, b.nrows - 1), host[:-1]
            keys = [DeviceColumn.from_numpy(host)]
        elif image is not None:
            plan, key_names = image
            keys = unpack(keys[0], plan)
        nb = DeviceBlock(b.cols, b.columns, nrows=b.nrows, index_cols=keys, index_names=names or key_names)
        nb.keys_sorted_unique = True
        out.append(nb)
    return out


# ---- dictionary aggregation --------------------------------------------------------------------------------------
_DICT_AGGS = ("sum", "count", "mean", "min", "max")


def split_aggregations(spec: dict, columns, keys=()) -> Dict[str, list]:
    """``{column: function}`` -> ``{function: [columns]}``, in first-seen order.  ``groupby.agg`` with a dictionary
    runs one device aggregation per DISTINCT function over the columns that ask for it (the reference's
    ``_groupby_dict_reduce``, qc.py:3876-3970, builds one map / reduce table per function the same way)."""
    by_func = {}
    for col, fn in spec.items():
        if not isinstance(fn, str) or fn not in _DICT_AGGS:
            raise NotImplementedError(f"groupby.agg({{{col!r}: {fn!r}}}) is not on the B200 path")
        if col not in columns or col in keys:
            raise KeyError(col)
        by_func.setdefault(fn, []).append(col)
    return by_func


def zip_aggregations(spec: dict, by_func: Dict[str, list], results: List[List[list]]) -> List[DeviceBlock]:
    """One block per row partition holding ``spec``'s columns in its order, taken from the per-function results
    (``results[i]``: the rows of ``by_func``'s i-th aggregation, each row the list of its column partitions' blocks).
    Every result carries the same ascending group keys, so the columns are zipped as they are: buffers shared."""
    where = {c: (i, j) for i, cols in enumerate(by_func.values()) for j, c in enumerate(cols)}
    if any(len(row) != 1 for rows in results for row in rows):
        raise NotImplementedError("dictionary aggregation over more than 32 columns per function")
    if len({len(rows) for rows in results}) != 1:
        raise NotImplementedError("per-function results are partitioned differently")
    out = []
    for row in zip(*results):
        blks = [r[0] for r in row]
        if len({b.nrows for b in blks}) != 1:
            raise NotImplementedError("per-function results are partitioned differently")
        nb = DeviceBlock([blks[i].cols[j] for i, j in (where[c] for c in spec)], pandas.Index(list(spec)),
                         nrows=blks[0].nrows, index_cols=blks[0].index_cols, index_names=blks[0].index_names)  # fmt: skip
        nb.keys_sorted_unique = True
        nb.replicated = blks[0].replicated
        out.append(nb)
    return out

