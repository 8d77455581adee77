"""Operator templates: Map, TreeReduce, Reduce, Fold, Binary.

Same contract as modin/core/dataframe/algebra/: ``Template.register(func, ...)`` returns a
``caller(query_compiler, *args, **kwargs) -> query_compiler`` closure that calls the matching
core-dataframe method (``map`` / ``tree_reduce`` / ``n_ary_op`` / ``broadcast_apply`` /
``reduce`` / ``fold``).  The registered ``func`` is a device functor (functors.py) with the pandas
method's calling convention; arguments are bound with ``Bound`` (the inspectable twin of the
reference's ``lambda x: function(x, *args, **kwargs)``) so the partition call queue can fuse.

Reference: operator.py:21-64, map.py:32-70, tree_reduce.py:33-82, reduce.py:32-71, fold.py:32-95,
binary.py:296-460.  The groupby aggregations are not a template here: ``query_compiler.device_operations`` calls
``groupby_reduce`` with the device functors directly, under both front doors.
"""

from __future__ import annotations

from typing import Callable, Optional

import numpy as np
import pandas

from .partitioning import Bound


class Operator:
    """alg/operator.py:21-64."""

    def __init__(self):
        raise ValueError(f"Please use {type(self).__name__}.register instead of the constructor")

    @classmethod
    def register(cls, func: Callable, **kwargs):
        raise NotImplementedError("Please implement in child class")

    @classmethod
    def validate_axis(cls, axis: Optional[int]) -> int:
        return 0 if axis is None else axis

    @classmethod
    def apply(cls, df, func, func_args=None, func_kwargs=None, **kwargs):
        operator = cls.register(func, **kwargs)
        qc_result = operator(df._query_compiler, *(func_args or ()), **(func_kwargs or {}))
        return type(df)(query_compiler=qc_result)


class Map(Operator):
    """alg/map.py:32-70."""

    @classmethod
    def register(cls, function, *call_args, **call_kwds):
        def caller(query_compiler, *args, **kwargs):
            kwds = dict(call_kwds)
            shape_hint = kwds.pop("shape_hint", None) or query_compiler._shape_hint
            return query_compiler.__constructor__(
                query_compiler._modin_frame.map(Bound(function, args, kwargs), *call_args, **kwds),
                shape_hint=shape_hint,
            )

        return caller


class TreeReduce(Operator):
    """alg/tree_reduce.py:33-82."""

    @classmethod
    def register(cls, map_function, reduce_function=None, axis=None, compute_dtypes=None):
        if reduce_function is None:
            reduce_function = map_function

        def caller(query_compiler, *args, **kwargs):
            _axis = kwargs.get("axis") if axis is None else axis
            new_dtypes = None
            if compute_dtypes and query_compiler.frame_has_materialized_dtypes:
                new_dtypes = str(compute_dtypes(query_compiler.dtypes, *args, **kwargs))
            return query_compiler.__constructor__(
                query_compiler._modin_frame.tree_reduce(
                    cls.validate_axis(_axis),
                    Bound(map_function, args, kwargs),
                    Bound(reduce_function, args, kwargs),
                    dtypes=new_dtypes,
                )
            )

        return caller


class Reduce(Operator):
    """alg/reduce.py:32-71: one function over FULL column partitions (``PandasDataframe.reduce``, df.py:2171-2205) --
    for reductions that have no map / combine split (var, std: two dependent sweeps)."""

    @classmethod
    def register(cls, reduce_function, axis=None, shape_hint=None):
        def caller(query_compiler, *args, **kwargs):
            _axis = kwargs.get("axis") if axis is None else axis
            return query_compiler.__constructor__(
                query_compiler._modin_frame.reduce(cls.validate_axis(_axis), Bound(reduce_function, args, kwargs))
            )

        return caller


class Fold(Operator):
    """alg/fold.py:32-95: one shape-preserving function over FULL column partitions (``PandasDataframe.fold``,
    df.py:2357-2400) -- cumulative functions and forward fill."""

    @classmethod
    def register(cls, fold_function, shape_preserved=False):
        def caller(query_compiler, fold_axis=None, *args, new_index=None, new_columns=None, **kwargs):
            return query_compiler.__constructor__(
                query_compiler._modin_frame.fold(
                    cls.validate_axis(fold_axis), Bound(fold_function, args, kwargs), new_index=new_index,
                    new_columns=new_columns, shape_preserved=shape_preserved,
                )  # fmt: skip
            )

        return caller


class Binary(Operator):
    """alg/binary.py:296-460 (dtype inference is per device block, so `infer_dtypes` hints are
    accepted for signature parity and the result dtypes are read off the produced blocks)."""

    @classmethod
    def register(cls, func, join_type="outer", sort=None, labels="replace", infer_dtypes=None):
        def caller(query_compiler, other, broadcast=False, *args, dtypes=None, **kwargs):
            axis = kwargs.get("axis", 0)
            if isinstance(other, type(query_compiler)) and broadcast:
                assert len(other.columns) == 1, (
                    "Invalid broadcast argument for `broadcast_apply`, too many columns: {}".format(len(other.columns))
                )
            shape_hint = None
            if isinstance(other, type(query_compiler)):
                if len(query_compiler.columns) == 1 and len(other.columns) == 1 and \
                        query_compiler.columns.equals(other.columns):  # fmt: skip
                    shape_hint = "column"
                if broadcast:
                    return query_compiler.__constructor__(
                        query_compiler._modin_frame.broadcast_apply(
                            axis, Bound(func, args, kwargs), other._modin_frame, join_type=join_type, labels=labels,
                            dtypes=dtypes,
                        ),
                        shape_hint=shape_hint,
                    )  # fmt: skip
                return query_compiler.__constructor__(
                    query_compiler._modin_frame.n_ary_op(
                        Bound(func, args, kwargs), [other._modin_frame], join_type=join_type, sort=sort,
                        labels=labels, dtypes=dtypes,
                    ),
                    shape_hint=shape_hint,
                )  # fmt: skip
            if isinstance(other, dict):
                other = pandas.Series(other)
            if len(query_compiler.columns) == 1 and np.isscalar(other):
                shape_hint = "column"
            if (isinstance(other, (list, tuple, np.ndarray)) and axis not in (0, "index")
                    and query_compiler._modin_frame._partitions.shape[1] > 1):  # fmt: skip
                # a positional row vector over SEVERAL column partitions: the reference applies it full-axis so that
                # every call sees whole rows (binary.py:431-442, whose TODO proposes chunking `other` instead); here it
                # is labelled with the frame's columns and each block takes its slice by label, as for a Series.  One
                # column partition keeps the list (fusable).
                W = len(query_compiler.columns)
                if len(other) != W:
                    raise ValueError(f"Unable to coerce to Series, length must be {W}: given {len(other)}")
                other = pandas.Series(list(other), index=query_compiler.columns)
            # scalar / list / Series operand: lazy map (binary.py:449-455) -> lands in the call queue
            new_modin_frame = query_compiler._modin_frame.map(
                func, func_args=(other, *args), func_kwargs=kwargs, dtypes=dtypes, lazy=True
            )
            return query_compiler.__constructor__(new_modin_frame, shape_hint=shape_hint)

        return caller

