"""Partitions and the partition manager of the B200 execution.

Mirrors, name for name, the classes of the reference's partition layer:

* ``B200Wrapper``           <- PythonWrapper            (modin/core/execution/python/common/engine_wrapper.py:17-97)
* ``B200Partition``         <- PandasDataframePartition (partitioning/partition.py:33-453) /
                               PandasOnPythonDataframePartition (pandas_on_python/partitioning/partition.py:22-176)
* ``B200ColumnPartition`` / ``B200RowPartition`` <- PandasDataframeAxisPartition (axis_partition.py:29-744)
* ``B200PartitionManager``  <- PandasDataframePartitionManager (partition_manager.py:95-2052)

Differences that are the point of the exercise: the payload is a ``DeviceBlock``; functions are
device functors (functors.py); "execution" is a kernel launch on the rank's CUDA stream (host
returns immediately, ``wait`` = stream sync); the call queue is a *fusion window*; full-axis
functions that the reference runs in one gathered task become local kernels + a collective
when the job spans several GPUs (dist.py).
"""

from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np
import pandas

from . import dist
from .block import DeviceBlock, HostBlock, concat_cols, concat_rows, torch_mod
from .config import BenchmarkMode, HostStreamMinBytes, MinColumnPartitionSize, MinRowPartitionSize, NPartitions
from .functors import DevAffine, DevBinary, DevFma3, DevFn, DevGroupbyMap, DevGroupbyReduce, fused_dense_groupby


# ------------------------------------------------------------------ small utilities (sfutils.py)
def compute_chunksize(axis_len: int, num_splits: int, min_block_size: int) -> int:
    """Reference: modin/core/storage_formats/pandas/utils.py:28-58."""
    if not isinstance(min_block_size, int) or min_block_size <= 0:
        raise ValueError(f"'min_block_size' should be int > 0, passed: {min_block_size=}")
    chunksize = axis_len // num_splits
    if axis_len % num_splits:
        chunksize += 1
    return max(chunksize, min_block_size)


def get_length_list(axis_len: int, num_splits: int, min_block_size: int) -> List[int]:
    """Reference: modin/core/storage_formats/pandas/utils.py:156-182."""
    chunksize = compute_chunksize(axis_len, num_splits, min_block_size)
    return [
        (chunksize if (i + 1) * chunksize <= axis_len else max(0, axis_len - i * chunksize))
        for i in range(num_splits)
    ]


class Bound:
    """``func`` with trailing positional/keyword arguments bound -- the inspectable equivalent of
    the reference's ``lambda x: function(x, *args, **kwargs)`` closures (alg/map.py:64-66), so the
    call queue can see which device functor it is about to run."""

    __slots__ = ("fn", "args", "kwargs")

    def __init__(self, fn, args=(), kwargs=None):
        self.fn, self.args, self.kwargs = fn, tuple(args), dict(kwargs or {})

    def __call__(self, *lead, **kw):
        return self.fn(*lead, *self.args, **{**self.kwargs, **kw})


def unwrap(func):
    """(functor, bound_args, bound_kwargs) of a possibly Bound callable.

    Modin's own templates hand the partition manager closures, not functors: the Binary template wraps the
    registered function as ``lambda x, y: func(x, y, *args, **kwargs)`` (alg/binary.py:421).  When such a closure's
    free variables are exactly a device functor plus its ``args`` / ``kwargs``, it is read back into the same
    (functor, args, kwargs) triple, so that the call queue can still fuse ``a * b`` with the ``+ c`` that follows
    under the real ``modin.pandas``."""
    if isinstance(func, Bound):
        return func.fn, func.args, func.kwargs
    code, cells = getattr(func, "__code__", None), getattr(func, "__closure__", None)
    if code is not None and cells and code.co_name == "<lambda>" and set(code.co_freevars) == {"func", "args", "kwargs"}:
        free = {name: cell.cell_contents for name, cell in zip(code.co_freevars, cells)}
        if isinstance(free["func"], DevFn) and code.co_argcount == 2 and isinstance(free["args"], tuple):
            return free["func"], free["args"], dict(free["kwargs"])
    return func, (), {}


# ------------------------------------------------------------------ engine wrapper
class B200Wrapper:
    """Synchronous-host / asynchronous-device engine wrapper (``deploy`` launches kernels on the
    current CUDA stream and returns; ``wait``/``materialize`` need no futures)."""

    @classmethod
    def deploy(cls, func, f_args=None, f_kwargs=None, num_returns=1):
        return func(*(f_args or ()), **(f_kwargs or {}))

    @classmethod
    def is_future(cls, item):
        return False

    @classmethod
    def materialize(cls, obj_id):
        return obj_id

    @classmethod
    def put(cls, data, **kwargs):
        return data

    @classmethod
    def wait(cls, obj_ids=None, num_returns=None):
        t = torch_mod()
        if t.cuda.is_available():
            t.cuda.current_stream().synchronize()


# ------------------------------------------------------------------ call-queue fusion
def _scalar_operand(entry):
    """(op, operand) if the queue entry is DevBinary against a scalar / row vector, else None."""
    func, args, kwargs = entry
    fn, bargs, bkw = unwrap(func)
    if not isinstance(fn, DevBinary):
        return None
    allargs = tuple(bargs) + tuple(args)
    if not allargs:
        return None
    other = allargs[0]
    extra = {**bkw, **kwargs}
    if extra.get("level") is not None or extra.get("fill_value") is not None:
        return None
    if isinstance(other, (B200Partition, DeviceBlock)):
        return None
    if isinstance(other, (int, float, np.integer, np.floating)) and not isinstance(other, bool):
        return fn.op, other
    if isinstance(other, (list, tuple, np.ndarray)):
        return fn.op, list(other)
    return None


def _block_operand(entry):
    func, args, kwargs = entry
    fn, bargs, bkw = unwrap(func)
    if not isinstance(fn, DevBinary):
        return None
    allargs = tuple(bargs) + tuple(args)
    if not allargs or not isinstance(allargs[0], (B200Partition, DeviceBlock)):
        return None
    extra = {**bkw, **kwargs}
    if extra.get("level") is not None or extra.get("fill_value") is not None:
        return None
    return fn.op, allargs[0]


def _entry_kwargs(entry):
    func, _args, kwargs = entry
    return {**unwrap(func)[2], **kwargs}


def fuse_call_queue(queue: list) -> list:
    """Peephole fusion over adjacent queue entries:
    ``x * s`` ; ``+ t``   -> AFFINE(s, t)   (one sweep, two roundings)
    ``a * b`` ; ``+ c``   -> FMA3(a, b, c)  (one sweep instead of two + a temporary)."""
    out = []
    i = 0
    while i < len(queue):
        cur = queue[i]
        nxt = queue[i + 1] if i + 1 < len(queue) else None
        if nxt is not None:
            a, b = _scalar_operand(cur), _scalar_operand(nxt)
            if a and b and a[0] in ("mul", "rmul") and b[0] in ("add", "radd"):
                out.append([DevAffine(a[1], b[1]), (), {}])
                i += 2
                continue
            fa, fb = _block_operand(cur), _block_operand(nxt)
            if fa and fb and fa[0] in ("mul", "rmul") and fb[0] in ("add", "radd"):
                out.append([_Fma3Entry(fa[1], fb[1], _entry_kwargs(cur), _entry_kwargs(nxt)), (), {}])
                i += 2
                continue
        out.append(cur)
        i += 1
    return out


class _Fma3Entry(DevFn):
    """``a * b`` then ``+ c`` between blocks, met next to each other in a call queue.  One FMA3 sweep (two roundings)
    when the three operands are float64 throughout, non-empty, identically shaped and labelled; anything else (int64
    or mixed columns, empty blocks, a one-column operand to broadcast) runs the two ``DevBinary`` steps one after the
    other, with their dtype promotion, label checks and empty-frame handling."""

    op = "fma3"

    def __init__(self, b, c, kw_mul=None, kw_add=None):
        self.b, self.c = b, c
        self.kw_mul, self.kw_add = dict(kw_mul or {}), dict(kw_add or {})

    def __call__(self, a):
        b, c = _payload(self.b), _payload(self.c)
        fusable = (
            a.nrows > 0 and a.nrows == b.nrows == c.nrows and len(a.cols) == len(b.cols) == len(c.cols)
            and a.columns.equals(b.columns) and a.columns.equals(c.columns)
            and all(x.dtype == np.float64 for blk in (a, b, c) for x in blk.cols)
        )  # fmt: skip
        if fusable:
            return DevFma3()(a, b, c)
        return DevBinary("add")(DevBinary("mul")(a, b, **self.kw_mul), c, **self.kw_add)


def _payload(x):
    return x.get() if isinstance(x, B200Partition) else x


def _inherit_replicated(result, inputs):
    """A function of blocks that EVERY rank holds in full (results of collectives: reductions, gathered frames)
    gives every rank the same block again -- the flag that keeps later reduce phases from combining it across ranks
    once more is handed on, whatever functor built the result."""
    blocks = [b for b in inputs if isinstance(b, DeviceBlock)]
    if isinstance(result, DeviceBlock) and not result.replicated and blocks and all(b.replicated for b in blocks):
        result.replicated = True
    return result


def _run_queue(data, queue):
    for func, args, kwargs in fuse_call_queue(queue):
        args = tuple(_payload(a) for a in args)
        fn, bargs, bkw = unwrap(func)
        bargs = tuple(_payload(a) for a in bargs)
        data = _inherit_replicated(fn(data, *bargs, *args, **{**bkw, **kwargs}), (data, *bargs, *args))
    return data


# ------------------------------------------------------------------ host-resident blocks: streamed execution
def _streamable_step(queue):
    """``(op, s0, s1)`` when the (fused) call queue of a host-resident partition is ONE elementwise sweep that
    ``mb200_map_host`` can stream -- ``x * s + t`` (AFFINE), ``abs`` / ``neg``, or one arithmetic op against a scalar
    or row vector -- over float64 columns; else None.  ``s0`` / ``s1`` are scalars or per-column lists."""
    from .functors import DevMap

    fused = fuse_call_queue(queue)
    if len(fused) != 1:
        return None
    func, args, kwargs = fused[0]
    fn, bargs, bkw = unwrap(func)
    if isinstance(fn, DevAffine) and not args and not bargs:
        return "affine", fn.mul, fn.add
    if isinstance(fn, DevMap) and fn.op in ("abs", "neg") and not args and not bargs:
        return fn.op, None, None
    sc = _scalar_operand(fused[0])
    if sc is not None:
        op = {"add": "add_s", "radd": "add_s", "mul": "mul_s", "rmul": "mul_s", "sub": "sub_s", "rsub": "rsub_s",
              "truediv": "div_s", "rtruediv": "rdiv_s"}.get(sc[0])  # fmt: skip
        if op is not None:
            return op, sc[1], None
    return None


def stream_to_pandas(row_partitions):
    """``to_pandas`` of row partitions that still live on the host (``HostBlock``) and carry a streamable call queue:
    every block is pushed through the device in chunks (H2D copy, one fused sweep, D2H copy, overlapped on three
    streams by ``mb200_map_host``) straight into the columns of the result frame -- pinned buffers from the pool, so
    both copies run as plain DMA.  Returns None when the partitions do not qualify (the caller then takes the
    device-resident path).  This is what ``pd.DataFrame(host) * b + c -> to_pandas()`` costs end to end."""
    from . import _lib, hostpath

    if not row_partitions or dist.is_distributed():
        return None
    steps = []
    for p in row_partitions:
        if not isinstance(p._data, HostBlock) or not p.call_queue:
            return None
        st = _streamable_step(p.call_queue)
        if st is None:
            return None
        steps.append(st)
    first = row_partitions[0]._data
    W = first.ncols
    if any(p._data.ncols != W or list(p._data.frame.columns) != list(first.frame.columns) for p in row_partitions):
        return None
    if any(dt != np.dtype("float64") for p in row_partitions for dt in p._data.frame.dtypes):
        return None  # int64 columns would need pandas' promotion rules per op: device-resident path
    total = sum(p._data.nrows for p in row_partitions)
    out = [hostpath.pinned_array(total, np.float64) for _ in range(W)]
    pos = 0
    for p, (op, s0, s1) in zip(row_partitions, steps):
        n = p._data.nrows
        vec = lambda v: None if v is None else ([float(x) for x in v] if isinstance(v, (list, tuple, np.ndarray)) else [float(v)] * W)  # noqa: E731
        a, b = vec(s0), vec(s1)
        if (a is not None and len(a) != W) or (b is not None and len(b) != W):
            return None
        if n:
            hostpath.stream_map(op, _lib.F64, p._data.columns_numpy(), [o[pos : pos + n] for o in out], s0=a, s1=b)
        pos += n
    index = row_partitions[0]._data.frame.index
    for p in row_partitions[1:]:
        index = index.append(p._data.frame.index)
    return pandas.DataFrame(dict(zip(range(W), out)), index=index, copy=False).set_axis(first.frame.columns, axis=1)


# ------------------------------------------------------------------ block partition
class B200Partition:
    """One block partition holding a DeviceBlock (immutable value semantics)."""

    execution_wrapper = B200Wrapper

    def __init__(self, data, length=None, width=None, call_queue=None):
        self._data = data
        self.call_queue = list(call_queue) if call_queue else []
        self._length_cache = length
        self._width_cache = width

    @property
    def __constructor__(self):
        return type(self)

    # -- execution -------------------------------------------------------------------------------
    def _on_device(self):
        """The payload as a DeviceBlock: a block left on the host at ingest (HostBlock) is copied H2D now."""
        if isinstance(self._data, HostBlock):
            self._data = self._data.materialize()
        return self._data

    def get(self):
        self.drain_call_queue()
        block = self._on_device()
        if getattr(block, "_pending", None) is not None:
            block.nrows  # a block sized on the device learns its row count (and trims its buffers) before anyone reads it
        return block

    @property
    def list_of_blocks(self):
        self.drain_call_queue()
        return [self._on_device()]

    def apply(self, func: Callable, *args, **kwargs):
        """Run the call queue, then ``func`` (pandas_on_python/partitioning/partition.py:76-123);
        no defensive copies: blocks are immutable and device functors never write in place."""
        queue = self.call_queue + [[func, args, kwargs]]
        try:
            data = _run_queue(self._on_device(), queue)
        except Exception:
            raise
        return self.__constructor__(data)

    def add_to_apply_calls(self, func, *args, length=None, width=None, **kwargs):
        return self.__constructor__(
            self._data, call_queue=self.call_queue + [[func, args, kwargs]], length=length, width=width
        )

    def drain_call_queue(self):
        if not self.call_queue:
            return
        queue, self.call_queue = self.call_queue, []
        try:
            self._data = _run_queue(self._on_device(), queue)
        except Exception:
            self.call_queue = []  # reference clears the queue on failure (partition.py:111-116)
            raise
        self._length_cache = self._width_cache = None

    def wait(self):
        self.drain_call_queue()
        self.execution_wrapper.wait()

    # -- construction ----------------------------------------------------------------------------
    @classmethod
    def put(cls, obj):
        """pandas.DataFrame -> device partition (H2D); a DeviceBlock is wrapped as is."""
        if isinstance(obj, DeviceBlock):
            return cls(obj, length=obj.nrows, width=len(obj.cols))
        if HostBlock.eligible(obj, HostStreamMinBytes.get()) and not dist.is_distributed():
            from .block import current_device

            current_device()  # no device, no ingest: fail here like the eager H2D path would
            return cls(HostBlock(obj), length=len(obj), width=obj.shape[1])
        block = DeviceBlock.from_pandas(obj)
        return cls(block, length=block.nrows, width=len(block.cols))

    @classmethod
    def preprocess_func(cls, func):
        return func

    @classmethod
    def empty(cls):
        return cls.put(pandas.DataFrame())

    # -- metadata --------------------------------------------------------------------------------
    def length(self, materialize=True):
        if self._length_cache is None:
            self._length_cache = self._data.nrows if isinstance(self._data, HostBlock) and not self.call_queue \
                else self.get().nrows  # fmt: skip
        return self._length_cache

    def width(self, materialize=True):
        if self._width_cache is None:
            self._width_cache = self._data.ncols if isinstance(self._data, HostBlock) and not self.call_queue \
                else len(self.get().cols)  # fmt: skip
        return self._width_cache

    # -- egress / structure ----------------------------------------------------------------------
    def to_pandas(self):
        streamed = stream_to_pandas([self])
        return streamed if streamed is not None else self.get().to_pandas()

    def to_numpy(self, **kwargs):
        return self.get().to_numpy()

    def mask(self, row_labels, col_labels):
        """Positional sub-block (part.py:219-300): slices share buffers; arbitrary row lists gather."""
        block = self.get()
        if not (isinstance(col_labels, slice) and col_labels == slice(None)):
            pos = list(range(len(block.cols))[col_labels]) if isinstance(col_labels, slice) else list(col_labels)
            block = block.select_columns(pos)
        if isinstance(row_labels, slice):
            if row_labels != slice(None):
                start, stop, step = row_labels.indices(block.nrows)
                if step != 1:
                    raise NotImplementedError("strided row masks are not on the B200 path")
                block = block.slice_rows(start, stop)
        else:
            rows = np.asarray(list(row_labels), dtype=np.int64)
            if len(rows) and np.array_equal(rows, np.arange(rows[0], rows[0] + len(rows))):
                block = block.slice_rows(int(rows[0]), int(rows[0]) + len(rows))
            else:
                from . import ops
                from .block import DeviceColumn

                idx = DeviceColumn.from_numpy(rows)
                cols = ops.take_columns(block.cols, idx)
                ih = block.index[rows]
                block = DeviceBlock(cols, block.columns, nrows=len(rows), index_host=ih)
        return self.__constructor__(block)

    def split(self, split_func, num_splits, *args):
        outs = split_func(self.get(), *args)
        return [self.__constructor__(o) for o in outs]


# ------------------------------------------------------------------ axis partitions
def split_block(axis: int, block: DeviceBlock, num_splits: int, lengths=None, min_block_size=None):
    """split_result_of_axis_func_pandas (sfutils.py:61-153) for device blocks: views, no copies."""
    if num_splits == 1 and lengths is None:
        return [block]
    total = block.nrows if axis == 0 else len(block.cols)
    if lengths is None:
        mbs = min_block_size or (MinRowPartitionSize.get() if axis == 0 else MinColumnPartitionSize.get())
        lengths = get_length_list(total, num_splits, mbs)
    outs, pos = [], 0
    for ln in lengths:
        if axis == 0:
            outs.append(block.slice_rows(pos, pos + ln))
        else:
            outs.append(block.select_columns(list(range(pos, min(pos + ln, total)))))
        pos += ln
    return outs


class B200AxisPartition:
    """Virtual partition spanning a full row or column of the grid."""

    axis: Optional[int] = None
    partition_type = B200Partition
    instance_type = DeviceBlock

    def __init__(self, list_of_partitions, get_ip=False, full_axis=True, call_queue=None, length=None, width=None):
        if isinstance(list_of_partitions, B200Partition):
            list_of_partitions = [list_of_partitions]
        self._list_of_block_partitions = list(list_of_partitions)
        self.full_axis = full_axis
        self.call_queue = call_queue or []

    @property
    def list_of_block_partitions(self):
        return self._list_of_block_partitions

    @property
    def list_of_blocks(self):
        return [p.get() for p in self._list_of_block_partitions]

    def _gathered(self) -> DeviceBlock:
        blocks = self.list_of_blocks
        return concat_rows(blocks) if self.axis == 0 else concat_cols(blocks)

    @classmethod
    def deploy_axis_func(cls, axis, func, f_args, f_kwargs, num_splits, maintain_partitioning, blocks,
                         lengths=None, manual_partition=False, min_block_size=None):  # fmt: skip
        """axpart.py:396-499: concat the blocks along ``axis``, run ``func`` once, split the result.
        When the job spans several ranks (the other ranks hold the remaining blocks of this axis), a reduce-phase
        device functor finishes with its own collective (``functors._spans_ranks``)."""
        gathered = concat_rows(blocks) if axis == 0 else concat_cols(blocks)
        fn, bargs, bkw = unwrap(func)
        args = tuple(bargs) + tuple(f_args or ())
        kwargs = {**bkw, **(f_kwargs or {})}
        result = _inherit_replicated(fn(gathered, *args, **kwargs), (gathered, *args))
        if manual_partition:
            lengths_ = lengths
        elif num_splits == 1:
            return [result]
        elif maintain_partitioning and lengths is None:
            lengths_ = [b.nrows if axis == 0 else len(b.cols) for b in blocks]
            if sum(lengths_) != (result.nrows if axis == 0 else len(result.cols)):
                lengths_ = None
        else:
            lengths_ = lengths
        return split_block(axis, result, num_splits, lengths_, min_block_size)

    @classmethod
    def deploy_func_between_two_axis_partitions(cls, axis, func, f_args, f_kwargs, num_splits, len_of_left,
                                                other_shape, blocks, min_block_size=None):  # fmt: skip
        """axpart.py:502-593: gather the left axis partition and the (broadcast) right frame, apply
        ``func(left, right)``, split."""
        left_blocks, right_blocks = blocks[:len_of_left], blocks[len_of_left:]
        lt = concat_rows(left_blocks) if axis == 0 else concat_cols(left_blocks)
        # rebuild the right frame from its 2-D grid described by `other_shape` (cumulative offsets)
        rows = []
        for i in range(1, len(other_shape)):
            rows.append(concat_cols(right_blocks[other_shape[i - 1] : other_shape[i]]))
        rt = concat_rows(rows) if len(rows) > 1 else rows[0]
        fn, bargs, bkw = unwrap(func)
        result = _inherit_replicated(fn(lt, rt, *bargs, *(f_args or ()), **{**bkw, **(f_kwargs or {})}), (lt, rt))
        if num_splits == 1:
            return [result]
        return split_block(axis, result, num_splits, None, min_block_size)

    def apply(self, func, *args, num_splits=None, other_axis_partition=None, maintain_partitioning=True,
              lengths=None, manual_partition=False, **kwargs):  # fmt: skip
        """axpart.py:199-309."""
        if num_splits is None:
            num_splits = len(self._list_of_block_partitions)
        if other_axis_partition is not None:
            if not isinstance(other_axis_partition, list):
                other_axis_partition = [other_axis_partition]
            other_shape = np.cumsum([0] + [len(o.list_of_block_partitions) for o in other_axis_partition])
            blocks = self.list_of_blocks + [b for o in other_axis_partition for b in o.list_of_blocks]
            outs = self.deploy_func_between_two_axis_partitions(
                self.axis, func, args, kwargs, num_splits, len(self._list_of_block_partitions), other_shape, blocks
            )
        else:
            outs = self.deploy_axis_func(
                self.axis, func, args, kwargs, num_splits, maintain_partitioning, self.list_of_blocks,
                lengths=lengths, manual_partition=manual_partition,
            )  # fmt: skip
        return [self.partition_type(o) for o in outs]

    def split(self, split_func, num_splits, *args, extract_metadata=False):
        """axpart.py:321-366: gather the blocks of this axis partition, split them with ``split_func`` into
        ``num_splits`` pieces (the range-partitioning split step), one new block partition per piece."""
        fn, bargs, bkw = unwrap(split_func)
        pieces = fn(self._gathered(), *bargs, *args, **bkw)
        if len(pieces) != num_splits:
            raise ValueError(f"split function returned {len(pieces)} pieces, expected {num_splits}")
        return [self.partition_type(b) for b in pieces]

    def wait(self):
        for p in self._list_of_block_partitions:
            p.wait()


class B200ColumnPartition(B200AxisPartition):
    axis = 0


class B200RowPartition(B200AxisPartition):
    axis = 1


# ------------------------------------------------------------------ partition manager
def wait_computations_if_benchmark_mode(func):
    """pm.py:52-92: under BenchmarkMode block until the device finished the produced partitions."""

    def wrapper(cls, *args, **kwargs):
        result = func(cls, *args, **kwargs)
        if BenchmarkMode.get():
            parts = result[0] if isinstance(result, tuple) else result
            if isinstance(parts, np.ndarray):
                cls.finalize(parts)
                cls.wait_partitions(parts.flatten())
        return result

    wrapper.__name__ = func.__name__
    wrapper.__doc__ = func.__doc__
    return wrapper


class B200PartitionManager:
    """Classmethods over the 2-D grid of ``B200Partition`` objects (np.ndarray[object])."""

    _partition_class = B200Partition
    _column_partitions_class = B200ColumnPartition
    _row_partition_class = B200RowPartition
    _execution_wrapper = B200Wrapper

    @classmethod
    def preprocess_func(cls, map_func):
        return cls._partition_class.preprocess_func(map_func)

    # -- axis views ------------------------------------------------------------------------------
    @classmethod
    def column_partitions(cls, partitions, full_axis=True):
        if not isinstance(partitions, list):
            partitions = [partitions]
        return [cls._column_partitions_class(col, full_axis=full_axis)
                for frame in partitions for col in frame.T]  # fmt: skip

    @classmethod
    def row_partitions(cls, partitions):
        if not isinstance(partitions, list):
            partitions = [partitions]
        return [cls._row_partition_class(row) for frame in partitions for row in frame]

    @classmethod
    def axis_partition(cls, partitions, axis, full_axis: bool = True):
        return cls.column_partitions(partitions, full_axis) if not axis else cls.row_partitions(partitions)

    # -- Map -------------------------------------------------------------------------------------
    @classmethod
    @wait_computations_if_benchmark_mode
    def map_partitions(cls, partitions, map_func, func_args=None, func_kwargs=None):
        """pm.py:708-769 / base_map_partitions pm.py:615-654."""
        preprocessed = cls.preprocess_func(map_func)
        return np.array(
            [[part.apply(preprocessed, *(func_args or ()), **(func_kwargs or {})) for part in row]
             for row in partitions]
        ).reshape(np.asarray(partitions).shape)  # fmt: skip

    @classmethod
    @wait_computations_if_benchmark_mode
    def lazy_map_partitions(cls, partitions, map_func, func_args=None, func_kwargs=None, enumerate_partitions=False):
        """pm.py:773-815: queue the function; it runs (possibly fused) at the next apply/get."""
        preprocessed = cls.preprocess_func(map_func)
        return np.array(
            [[part.add_to_apply_calls(preprocessed, *(tuple() if func_args is None else func_args),
                                      **(func_kwargs or {}), **({"partition_idx": i} if enumerate_partitions else {}))
              for part in row] for i, row in enumerate(partitions)]
        ).reshape(np.asarray(partitions).shape)  # fmt: skip

    # -- full-axis -------------------------------------------------------------------------------
    @classmethod
    @wait_computations_if_benchmark_mode
    def broadcast_axis_partitions(cls, axis, apply_func, left, right, keep_partitioning=False, num_splits=None,
                                  apply_indices=None, broadcast_all=True, enumerate_partitions=False, lengths=None,
                                  apply_func_args=None, **kwargs):  # fmt: skip
        """pm.py:498-611."""
        if keep_partitioning and num_splits is None:
            num_splits = len(left) if axis == 0 else len(left.T)
        elif lengths:
            num_splits = len(lengths)
        elif num_splits is None:
            num_splits = NPartitions.get()
        preprocessed = cls.preprocess_func(apply_func)
        left_partitions = cls.axis_partition(left, axis)
        right_partitions = None if right is None else cls.axis_partition(right, axis)
        kw = {"num_splits": num_splits, "maintain_partitioning": keep_partitioning, **kwargs}
        if lengths:
            kw["lengths"] = lengths
            kw["manual_partition"] = True
        if apply_indices is None:
            apply_indices = np.arange(len(left_partitions))
        result_blocks = np.array(
            [
                left_partitions[i].apply(
                    preprocessed,
                    *(apply_func_args if apply_func_args else []),
                    other_axis_partition=(right_partitions if broadcast_all else right_partitions[i])
                    if right_partitions is not None else None,
                    **kw,
                    **({"partition_idx": idx} if enumerate_partitions else {}),
                )
                for idx, i in enumerate(apply_indices)
            ],
            dtype=object,
        )  # fmt: skip
        return result_blocks.T if not axis else result_blocks

    @classmethod
    @wait_computations_if_benchmark_mode
    def map_axis_partitions(cls, axis, partitions, map_func, keep_partitioning=False, num_splits=None, lengths=None,
                            enumerate_partitions=False, **kwargs):  # fmt: skip
        """pm.py:818-879."""
        return cls.broadcast_axis_partitions(
            axis=axis, left=partitions, apply_func=map_func, keep_partitioning=keep_partitioning,
            num_splits=num_splits, right=None, lengths=lengths, enumerate_partitions=enumerate_partitions, **kwargs,
        )  # fmt: skip

    # -- broadcast -------------------------------------------------------------------------------
    @classmethod
    @wait_computations_if_benchmark_mode
    def base_broadcast_apply(cls, axis, apply_func, left, right):
        """pm.py:443-494: every left block gets the matching slice of ``right`` (all its blocks
        along axis^1 concatenated -- zero-copy for device blocks)."""
        preprocessed = cls.preprocess_func(apply_func)

        def map_func(df, *others):
            other = (concat_cols(others) if axis == 0 else concat_rows(others)) if len(others) > 1 else others[0]
            return preprocessed(df, other)

        rt_axis_parts = cls.axis_partition(right, axis ^ 1)
        return np.array(
            [[part.apply(map_func, *(rt_axis_parts[col_idx].list_of_blocks if axis
                                     else rt_axis_parts[row_idx].list_of_blocks))
              for col_idx, part in enumerate(left[row_idx])] for row_idx in range(len(left))]
        )  # fmt: skip

    @classmethod
    @wait_computations_if_benchmark_mode
    def broadcast_apply(cls, axis, apply_func, left, right):
        """pm.py:658-704."""
        return cls.base_broadcast_apply(axis, apply_func, left, right)

    # -- GroupByReduce ---------------------------------------------------------------------------
    @classmethod
    @wait_computations_if_benchmark_mode
    def groupby_reduce(cls, axis, partitions, by, map_func, reduce_func, apply_indices=None):
        """pm.py:303-357."""
        if apply_indices is not None:
            partitions = partitions[apply_indices] if axis else partitions[:, apply_indices]
        if by is not None:
            assert partitions.shape[axis] == by.shape[axis], (
                f"the number of partitions along {axis=} is not equal: "
                + f"{partitions.shape[axis]} != {by.shape[axis]}"
            )
            # a row block spans every column partition on the device path (zero-copy concat)
            if partitions.shape[1] > 1:
                partitions = np.array([[cls._partition_class(concat_cols([p.get() for p in row]))]
                                       for row in partitions])  # fmt: skip
            # keys in a narrow range: map + reduce fused into one direct-addressed table per GPU, merged
            # across GPUs by element-wise collectives (functors.fused_dense_groupby); else the general path
            fn_map, fn_red = unwrap(cls.preprocess_func(map_func))[0], unwrap(cls.preprocess_func(reduce_func))[0]
            if axis == 0 and isinstance(fn_map, DevGroupbyMap) and isinstance(fn_red, DevGroupbyReduce) and by.shape[1] == 1:
                fused = fused_dense_groupby(fn_map, fn_red, [row[0].get() for row in partitions],
                                            [row[0].get() for row in by])  # fmt: skip
                if fused is not None:
                    return np.array([[cls._partition_class(fused)]])
            mapped_partitions = cls.broadcast_apply(axis, map_func, left=partitions, right=by)
        else:
            mapped_partitions = cls.map_partitions(partitions, map_func)
        num_splits = min(len(partitions), NPartitions.get())
        return cls.map_axis_partitions(axis, mapped_partitions, reduce_func, enumerate_partitions=True,
                                       num_splits=num_splits)  # fmt: skip

    # -- range-partitioning shuffle -------------------------------------------------------------
    @classmethod
    @wait_computations_if_benchmark_mode
    def shuffle_partitions(cls, partitions, index, shuffle_functions, final_shuffle_func, right_partitions=None):
        """pm.py:1937-2052: sample the key column of every row partition, let ``shuffle_functions`` pick the pivots,
        split every row partition into one piece per key range, transpose, and run ``final_shuffle_func`` over the
        pieces of each range.  Returns ``num_bins`` row partitions in key order (one column partition each).

        Across GPUs (``shuffle_functions.pivot_fn`` then answers one range per rank) the transpose is an
        ``all_to_all`` of raw rows over NVLink (``shuffle.exchange_pieces``): rank r ends up with range r."""
        from .shuffle import exchange_pieces

        if right_partitions is not None:
            raise NotImplementedError("range-partition shuffle with a broadcast right side is not on the B200 path")
        masked = partitions[:, index]
        sample_func = cls.preprocess_func(shuffle_functions.sample_fn)
        if masked.ndim == 1:
            samples = [part.apply(sample_func) for part in masked]
        else:
            samples = [cls._row_partition_class(row, full_axis=False).apply(sample_func)[0] for row in masked]
        samples = [s._data for s in samples]  # small device tensors, not blocks
        num_bins = shuffle_functions.pivot_fn(samples)
        row_partitions = cls.row_partitions(partitions)
        if num_bins <= 1:
            return np.array([[row_part.apply(final_shuffle_func, num_splits=1)[0]] for row_part in row_partitions])
        split_row_partitions = np.array(
            [part.split(shuffle_functions.split_fn, num_splits=num_bins) for part in row_partitions], dtype=object
        ).reshape(len(row_partitions), num_bins).T  # [bin][source row partition]
        if dist.is_distributed():
            # pieces of bin r from all local row partitions -> rank r
            send = [concat_rows([p.get() for p in pieces]) if len(pieces) > 1 else pieces[0].get() for pieces in split_row_partitions]
            mine = exchange_pieces(send)
            fn, bargs, bkw = unwrap(cls.preprocess_func(final_shuffle_func))
            return np.array([[cls._partition_class(fn(mine, *bargs, **bkw))]])
        return np.array(
            [[cls._column_partitions_class(list(pieces), full_axis=False).apply(final_shuffle_func, num_splits=1)[0]]
             for pieces in split_row_partitions]
        )  # fmt: skip

    # -- n-ary -----------------------------------------------------------------------------------
    @classmethod
    @wait_computations_if_benchmark_mode
    def n_ary_operation(cls, left, func, right: list):
        """pm.py:1725-1788: ``out[i,j] = func(left[i,j], *right_k[i,j])``.  Fusable device binary
        functors are queued instead of launched, so ``a*b`` followed by ``+c`` becomes one sweep."""
        func = cls.preprocess_func(func)
        fn, _, _ = unwrap(func)
        lazy = isinstance(fn, DevFn) and fn.fusable and len(right) == 1

        def get_right_block(right_partitions, row_idx, col_idx):
            return right_partitions[row_idx][col_idx]

        def one(part, row_idx, col_idx):
            others = [get_right_block(r, row_idx, col_idx) for r in right]
            if lazy:
                return part.add_to_apply_calls(func, *others)
            return part.apply(func, *others)

        return np.array([[one(part, i, j) for j, part in enumerate(row)] for i, row in enumerate(left)])

    # -- ingest / egress -------------------------------------------------------------------------
    @classmethod
    def split_pandas_df_into_partitions(cls, df, row_chunksize, col_chunksize, update_bar=None):
        """pm.py:1029-1066."""
        put = cls._partition_class.put
        parts = []
        for i in range(0, max(len(df), 1), row_chunksize):
            row = []
            for j in range(0, max(len(df.columns), 1), col_chunksize):
                row.append(put(df.iloc[i : i + row_chunksize, j : j + col_chunksize]))
            parts.append(row)
        return np.array(parts)

    @classmethod
    def from_pandas(cls, df, return_dims=False):
        """pm.py:1070-1149: split the host frame into the grid and H2D every block.  Under
        torch.distributed each rank ingests only its own row shard."""
        if dist.is_distributed():
            lo, hi = dist.shard_bounds(len(df))
            df = df.iloc[lo:hi]
        return cls.from_pandas_local(df, return_dims)

    @classmethod
    def from_pandas_local(cls, df, return_dims=False):
        """The grid split + H2D of ``from_pandas`` for a frame that is already this rank's own (a shard cut by the
        caller, or a small frame every rank holds in full)."""
        num_splits = NPartitions.get()
        row_chunksize = compute_chunksize(df.shape[0], num_splits, MinRowPartitionSize.get())
        col_chunksize = compute_chunksize(df.shape[1], num_splits, MinColumnPartitionSize.get())
        # on the device path column partitions only exist above 32 columns (one launch sweeps <= 32)
        col_chunksize = max(col_chunksize, MinColumnPartitionSize.get())
        parts = cls.split_pandas_df_into_partitions(df, row_chunksize, col_chunksize)
        backend = None
        if not return_dims:
            return parts, backend
        row_lengths = [row_chunksize if i + row_chunksize < len(df) else len(df) % row_chunksize or row_chunksize
                       for i in range(0, len(df), row_chunksize)]  # fmt: skip
        col_widths = [col_chunksize if i + col_chunksize < len(df.columns) else len(df.columns) % col_chunksize
                      or col_chunksize for i in range(0, len(df.columns), col_chunksize)]  # fmt: skip
        if len(df) == 0:
            row_lengths = [0]
        if len(df.columns) == 0:
            col_widths = [0]
        return parts, backend, row_lengths, col_widths

    @classmethod
    def from_arrow(cls, at, return_dims=False):
        """pm.py:1152-1169 goes through ``at.to_pandas()``; here each Arrow column's data buffer is
        viewed zero-copy on the host and copied H2D directly."""
        import pyarrow as pa  # noqa: F401

        cols = {}
        for name, col in zip(at.column_names, at.columns):
            arr = col.combine_chunks() if hasattr(col, "combine_chunks") else col
            if arr.null_count:
                if not pa.types.is_floating(arr.type):
                    raise NotImplementedError("nullable non-float Arrow columns are not on the B200 path")
                arr = arr.fill_null(float("nan"))
            cols[name] = arr.to_numpy(zero_copy_only=False)
        return cls.from_pandas(pandas.DataFrame(cols, copy=False), return_dims=return_dims)

    @classmethod
    def get_objects_from_partitions(cls, partitions):
        return [p.get() for p in partitions]

    @classmethod
    def to_pandas(cls, partitions):
        """pm.py:989-1005: D2H every block and assemble the host frame (all ranks' shards when
        distributed)."""
        if len(partitions) and np.asarray(partitions).shape[1] == 1:
            streamed = stream_to_pandas([row[0] for row in partitions])
            if streamed is not None:
                return streamed
        rows = []
        for row in partitions:
            blocks = [p.get() for p in row]
            rows.append(concat_cols(blocks) if len(blocks) > 1 else blocks[0])
        if not rows:
            return pandas.DataFrame()
        block = concat_rows(rows) if len(rows) > 1 else rows[0]
        if dist.is_distributed() and not block.replicated:
            block = gather_block(block)
        return block.to_pandas()

    @classmethod
    def to_numpy(cls, partitions, **kwargs):
        return cls.to_pandas(partitions).to_numpy(**kwargs)

    @classmethod
    def get_indices(cls, axis, partitions, index_func=None):
        """pm.py:1220-1267."""
        if index_func is None:
            index_func = (lambda b: b.index) if axis == 0 else (lambda b: b.columns)
        target = partitions.T if axis == 0 else partitions
        if len(target) == 0:
            return pandas.Index([]), []
        new_idx = [index_func(p.get()) for p in target[0]]
        total = new_idx[0]
        for ix in new_idx[1:]:
            total = total.append(ix)
        return total, new_idx

    @classmethod
    def concat(cls, axis, left_parts, right_parts):
        """pm.py:943-986."""
        if type(right_parts) is list:
            right_parts = [o for o in right_parts if o.size != 0]
            to_concat = [left_parts] + right_parts if left_parts.size != 0 else right_parts
            result = np.concatenate(to_concat, axis=axis) if len(to_concat) else left_parts
        else:
            result = np.append(left_parts, right_parts, axis=axis)
        return result, None

    @classmethod
    def combine(cls, partitions, new_index=None, new_columns=None):
        """pm.py:1328-1373: collapse the grid into ONE partition (used to broadcast the dim table).
        Across ranks the dim shards are all-gathered so every GPU holds the whole table."""
        rows = []
        for row in partitions:
            blocks = [p.get() for p in row]
            rows.append(concat_cols(blocks) if len(blocks) > 1 else blocks[0])
        block = concat_rows(rows) if len(rows) > 1 else rows[0]
        if dist.is_distributed() and not block.replicated:
            block = gather_block(block)
        return np.array([[cls._partition_class(block)]])

    @classmethod
    def finalize(cls, partitions):
        for p in np.asarray(partitions).flatten():
            p.drain_call_queue()

    @classmethod
    def wait_partitions(cls, partitions):
        """pm.py:1200-1217: one stream synchronisation covers every partition of this rank."""
        for p in partitions:
            p.drain_call_queue()
        cls._execution_wrapper.wait()

    @classmethod
    def create_partition_from_metadata(cls, dtypes=None, **metadata):
        metadata_dataframe = pandas.DataFrame(**metadata)
        if dtypes is not None:
            metadata_dataframe = metadata_dataframe.astype(dtypes)
        return cls._partition_class.put(metadata_dataframe)


def gather_block(block: DeviceBlock) -> DeviceBlock:
    """All-gather the row shards of a block so that every rank holds all rows."""
    from .block import DeviceColumn

    t = torch_mod()
    tensors = [c.data for c in block.cols]
    icols = list(block.index_cols or [])
    dev = tensors[0].device if tensors else ("cuda" if dist._dist().get_backend() == "nccl" else "cpu")
    # The ranks first agree on the label layout, in ONE small collective that every rank issues whatever its shard
    # looks like: the layouts can differ (a row filter gives the ranks that had rows a device label column while a
    # rank whose shard was already empty keeps its range), and ranks that then gathered different tensor lists -- or
    # one rank raising while the others wait -- would deadlock.
    label_is_float = int(bool(icols) and icols[0].dtype == np.float64)
    meta = dist.all_gather_small(t.tensor([len(icols), int(block.index_host is not None), block.range_start, block.nrows,
                                           label_is_float], dtype=t.int64, device=dev))  # fmt: skip
    if any(m[1] for m in meta):  # on every rank, not just the one that holds them
        raise NotImplementedError("gathering row shards with host-resident (non-numeric) row labels is not on the B200 path")
    nlabel = max(int(m[0]) for m in meta)
    if nlabel > 1 and len(icols) != nlabel:
        raise NotImplementedError("gathering row shards whose label levels differ between ranks is not on the B200 path")
    if nlabel == 1 and not icols:  # explicit labels elsewhere: this rank's range becomes explicit too, in their dtype
        as_float = any(m[0] and m[4] for m in meta)
        ldt, ndt = (t.float64, np.float64) if as_float else (t.int64, np.int64)
        if as_float:
            icols = [DeviceColumn(t.arange(block.range_start, block.range_start + block.nrows, dtype=ldt, device=dev), ndt)]
        else:
            from . import ops

            icols = [ops.iota(block.range_start, block.nrows)]
    tensors += [c.data for c in icols]
    gathered = dist.all_gather_rows(tensors)
    ncol = len(block.cols)
    cols = [DeviceColumn(g, c.dtype) for g, c in zip(gathered[:ncol], block.cols)]
    nrows = int(gathered[0].shape[0]) if gathered else 0
    if icols:
        ic = [DeviceColumn(g, c.dtype) for g, c in zip(gathered[ncol:], icols)]
        out = DeviceBlock(cols, block.columns, nrows=nrows, index_cols=ic, index_names=block.index_names or [None] * len(ic))
    else:
        # every shard is a run of a RangeIndex, but not necessarily of 0..N: tail() / a shifted RangeIndex start
        # later, and slices taken shard by shard need not run on from each other
        spans = [(int(m[2]), int(m[3])) for m in meta if m[3] > 0]
        if all(b[0] == a[0] + a[1] for a, b in zip(spans, spans[1:])):  # one job-wide range: labels stay O(1)
            out = DeviceBlock(cols, block.columns, nrows=nrows, range_start=spans[0][0] if spans else 0)
        else:
            labels = t.cat([t.arange(s, s + n, dtype=t.int64, device=dev) for s, n in spans])
            out = DeviceBlock(cols, block.columns, nrows=nrows, index_cols=[DeviceColumn(labels, np.int64)], index_names=[None])
    out.replicated = True
    return out
