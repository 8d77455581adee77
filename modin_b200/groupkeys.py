"""Several int64 group keys as ONE: the order-preserving packing behind ``df.groupby([k1, k2, ...])``.

The reference hands ``df.groupby([...])`` to pandas per block (alg/groupby.py:124-208), which builds a combined group
index with ``get_group_index``.  Here the key tuples are packed into one int64 on the device,
``sum_i (k_i - min_i) * stride_i`` with ``stride_i = prod_{j>i} (max_j - min_j + 1)``, the single-key device groupby
(dense or hashed table) runs on the image, and the G result keys are unpacked afterwards -- per row one subtract +
multiply per key column and k - 1 adds; per GROUP one divmod on the host (result-sized, not row-sized).  The key
ranges come from the columns' cached statistics (``ops.key_stats``), agreed across ranks once.
"""

from __future__ import annotations

from typing import List, Sequence

import numpy as np

from . import dist, ops
from .block import DeviceBlock, DeviceColumn

PACKED_KEY = "__packed_key__"


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

