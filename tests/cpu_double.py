"""TEST DOUBLE for the device: lets the host-side stack (templates -> frame -> partition manager ->
partitions -> functors) run in a container without a GPU by swapping the kernel wrappers of
``modin_b200.ops`` for numpy/pandas stand-ins that work on CPU torch tensors.

This is test infrastructure in the same sense as ``oracle/``: it exists so that the HOST LOGIC
(partition grid, call-queue fusion, functor argument handling, template wiring, the real-Modin
plug-in glue) can be exercised by ``pytest -m "not gpu"``.  It is installed by the ``cpu_device``
fixture only; nothing in ``modin_b200/`` imports it and the product has no CPU path.
"""

from __future__ import annotations

import contextlib

import numpy as np
import pandas
import torch

from modin_b200 import _lib, block, ops
from modin_b200.block import DeviceColumn


def _np(col: DeviceColumn) -> np.ndarray:
    a = col.data.numpy()
    return a.view(np.bool_) if col.dtype == np.bool_ else a


def _col(arr: np.ndarray) -> DeviceColumn:
    arr = np.ascontiguousarray(arr)
    host = arr.view(np.uint8) if arr.dtype == np.bool_ else arr
    return DeviceColumn(torch.from_numpy(host.copy()), arr.dtype)


def map_columns(op, in0, in1=None, in2=None, s0=None, s1=None):
    out = []
    for j, a in enumerate(in0):
        x = _np(a)
        y = _np(in1[j]) if in1 is not None else None
        z = _np(in2[j]) if in2 is not None else None
        p = s0[j] if s0 is not None else None
        q = s1[j] if s1 is not None else None
        if a.dtype == np.bool_ and op not in ("copy", "not", "and", "or", "xor"):
            raise TypeError("bool columns")
        with np.errstate(all="ignore"):
            r = {
                "abs": lambda: np.abs(x), "neg": lambda: -x, "isna": lambda: np.isnan(x), "notna": lambda: ~np.isnan(x),
                "fillna_s": lambda: np.where(np.isnan(x), p, x), "affine": lambda: x * p + q,
                "add_s": lambda: x + p, "sub_s": lambda: x - p, "rsub_s": lambda: p - x, "mul_s": lambda: x * p,
                "div_s": lambda: x / np.float64(p), "rdiv_s": lambda: np.float64(p) / x,
                "eq_s": lambda: x == p, "ne_s": lambda: x != p, "lt_s": lambda: x < p, "le_s": lambda: x <= p,
                "gt_s": lambda: x > p, "ge_s": lambda: x >= p,
                "copy": lambda: x.astype(np.int64) if x.dtype == np.bool_ else x.copy(),
                "clip_s": lambda: np.where(x < p, p, np.where(x > q, q, x)).astype(x.dtype),
                "ordered_s": lambda: _ordered_image(x, p),
                "not": lambda: ~x, "and": lambda: x & y, "or": lambda: x | y, "xor": lambda: x ^ y,
                "round_s": lambda: (np.rint(x * p) / p if q >= 0 else np.rint(x / p) * p) if x.dtype == np.float64 else x,
                "add": lambda: x + y, "sub": lambda: x - y, "mul": lambda: x * y, "div": lambda: x / y,
                "eq": lambda: x == y, "ne": lambda: x != y, "lt": lambda: x < y, "le": lambda: x <= y,
                "gt": lambda: x > y, "ge": lambda: x >= y, "fillna": lambda: np.where(np.isnan(x), y, x),
                "fma3": lambda: x * y + z,
            }[op]()  # fmt: skip
        if op in ("div", "div_s", "rdiv_s"):
            r = r.astype(np.float64)
        out.append(_col(np.asarray(r)))
    return out


def _ordered_image(x, desc):
    """numpy restatement of MB200_OP_ORDERED_S (csrc/elementwise.cu)."""
    if x.dtype == np.float64:
        b = x.view(np.int64)
        o = b ^ ((b >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))
        o = np.where(desc, ~o, o)
        return np.where(np.isnan(x), np.iinfo(np.int64).max, o).astype(np.int64)
    o = x.astype(np.int64)
    return (~o if desc else o).astype(np.int64)


def sort_pairs(keys, payload):
    """In-place stable sort of (keys, payload) by key."""
    k, p = _np(keys), _np(payload)
    order = np.argsort(k, kind="stable")
    k[:], p[:] = k[order], p[order]


def reduce_columns(op, cols, skipna=True, variant=0, centers=None):
    vals, cnts = [], []
    for j, c in enumerate(cols):
        x = _np(c)
        if op == "ssd":
            ok = ~np.isnan(x)
            with np.errstate(all="ignore"):
                d = float(centers[j]) - (x[ok] if skipna else x)
                vals.append(torch.tensor([np.sum(d * d)], dtype=torch.float64))
            cnts.append(torch.tensor([int(ok.sum())], dtype=torch.int64))
            continue
        if c.dtype == np.int64:
            n = len(x)
            v = {"sum": x.sum() if n else 0, "min": x.min() if n else np.iinfo(np.int64).max,
                 "max": x.max() if n else np.iinfo(np.int64).min, "count": 0, "prod": x.prod() if n else 1}[op]  # fmt: skip
            vals.append(torch.tensor([v], dtype=torch.int64))
            cnts.append(torch.tensor([n], dtype=torch.int64))
            continue
        ok = ~np.isnan(x)
        n = int(ok.sum())
        with np.errstate(all="ignore"):
            if op == "sum":
                v = x[ok].sum() if skipna else x.sum()
            elif op == "prod":
                v = x[ok].prod() if skipna else x.prod()
            elif op == "count":
                v = 0.0
            elif n == 0 or (not skipna and n < len(x)):
                v = np.nan
            else:
                v = x[ok].min() if op == "min" else x[ok].max()
        vals.append(torch.tensor([v], dtype=torch.float64))
        cnts.append(torch.tensor([n], dtype=torch.int64))
    return vals, cnts


def hash_aggregate(items, flags, capacity_hint, partial=False, sort=True):
    keys = np.concatenate([_np(it[0]) for it in items])
    nv = len(items[0][1]) if items[0][1] else 0
    df = pandas.DataFrame({"k": keys})
    uniq = np.sort(np.unique(keys))
    g = df.groupby("k", sort=True)
    sums = cnts = sizes = None
    if flags & _lib.GB_SUM:
        sums = []
        for v in range(nv):
            x = np.concatenate([_np(it[1][v]) for it in items])
            sums.append(_col(pandas.Series(np.where(np.isnan(x), 0.0, x)).groupby(keys, sort=True).sum().to_numpy()))
    for flag, fn in ((_lib.GB_MIN, "min"), (_lib.GB_MAX, "max")):
        if flags & flag:
            sums = []
            for v in range(nv):
                x = np.concatenate([_np(it[1][v]) for it in items])
                sums.append(_col(getattr(pandas.Series(x).groupby(keys, sort=True), fn)().to_numpy().astype(np.float64)))
    if flags & _lib.GB_COUNT:
        cnts = []
        for v in range(nv):
            if partial:
                c = np.concatenate([_np(it[2][v]) for it in items])
            else:
                c = (~np.isnan(np.concatenate([_np(it[1][v]) for it in items]))).astype(np.int64)
            cnts.append(_col(pandas.Series(c).groupby(keys, sort=True).sum().to_numpy().astype(np.int64)))
    if flags & _lib.GB_SIZE:
        z = np.concatenate([_np(it[3]) for it in items]) if partial else np.ones(len(keys), dtype=np.int64)
        sizes = _col(pandas.Series(z).groupby(keys, sort=True).sum().to_numpy().astype(np.int64))
    del g
    return _col(uniq.astype(np.int64)), sums, cnts, sizes


def key_range_device(key_cols):
    ks = [_np(k) for k in key_cols if len(k)]
    if not ks:
        return torch.tensor([np.iinfo(np.int64).max, np.iinfo(np.int64).min, 0, 0], dtype=torch.int64)
    return torch.tensor([min(int(k.min()) for k in ks), max(int(k.max()) for k in ks), 0, 0], dtype=torch.int64)


class GroupTable:
    """numpy stand-in for the DENSE device table (same array layout as include/modin_b200.h), so that the
    fused map+reduce path and its cross-rank merge by collectives run under gloo."""

    @classmethod
    def dense(cls, key_min, key_max, nvals, flags):
        self = cls()
        self.kbase, self.R, self.nvals, self.flags = int(key_min), int(key_max) - int(key_min) + 1, nvals, flags
        self.vs = max(4, (nvals + 3) & ~3)
        R, vs = self.R, self.vs
        self.acc = self.cnt = self.size = None
        if flags & _lib.GB_SUM:
            self.acc = torch.zeros(R * vs, dtype=torch.float64)
        elif flags & _lib.GB_MIN:
            self.acc = torch.full((R * vs,), np.iinfo(np.int64).max, dtype=torch.int64)
        elif flags & _lib.GB_MAX:
            self.acc = torch.full((R * vs,), np.iinfo(np.int64).min, dtype=torch.int64)
        if flags & _lib.GB_COUNT:
            self.cnt = torch.zeros(R * vs, dtype=torch.int64)
        if flags & _lib.GB_SIZE:
            self.size = torch.zeros(R, dtype=torch.int64)
        self.present = torch.zeros(4 * ((R + 3) // 4), dtype=torch.uint8)
        self.win = (0, R)
        return self

    @staticmethod
    def _ordered(x):  # order-preserving int64 image of float64 (csrc/groupby.cu f64_to_ordered)
        b = x.view(np.int64)
        return b ^ ((b >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))

    def accumulate(self, keys, vals):
        g = _np(keys) - self.kbase
        assert len(g) == 0 or (g.min() >= 0 and g.max() < self.R)
        self.present.numpy()[g] = 1
        if self.size is not None:
            np.add.at(self.size.numpy(), g, 1)
        for v, col in enumerate(vals):
            x = _np(col)
            ok = ~np.isnan(x)
            o = g[ok] * self.vs + v
            if self.flags & _lib.GB_SUM:
                np.add.at(self.acc.numpy(), o, x[ok])
            elif self.flags & _lib.GB_MIN:
                np.minimum.at(self.acc.numpy(), o, self._ordered(x[ok]))
            elif self.flags & _lib.GB_MAX:
                np.maximum.at(self.acc.numpy(), o, self._ordered(x[ok]))
            if self.cnt is not None:
                np.add.at(self.cnt.numpy(), o, 1)

    def collective_arrays(self):
        acc_op = "sum" if self.flags & _lib.GB_SUM else ("min" if self.flags & _lib.GB_MIN else "max")
        out = [(self.acc, acc_op, self.vs), (self.cnt, "sum", self.vs), (self.size, "sum", 1), (self.present, "max", 1)]
        return [(x, op, per) for x, op, per in out if x is not None]

    def reduce_scatter(self, chunk, reduce_scatter_fn, r):
        assert self.R % chunk == 0 and chunk % 4 == 0
        sl = GroupTable()
        sl.kbase, sl.R, sl.nvals, sl.flags, sl.vs = self.kbase + r * chunk, chunk, self.nvals, self.flags, self.vs
        sl.acc = sl.cnt = sl.size = None
        sl.win = (0, chunk)
        names = [n for n in ("acc", "cnt", "size", "present") if getattr(self, n) is not None]
        for name, (x, op, per) in zip(names, self.collective_arrays()):
            out = torch.empty(chunk * per, dtype=x.dtype)
            reduce_scatter_fn(out, x[: self.R * per], op)
            setattr(sl, name, out)
        return sl

    def hint_skew(self, skewed):
        pass

    def window(self, lo, hi):
        assert lo % 4 == 0 and (hi % 4 == 0 or hi == self.R) and 0 <= lo <= hi <= self.R
        self.win = (int(lo), int(hi))

    def _gids(self):
        lo, hi = self.win
        return lo + np.nonzero(self.present.numpy()[lo:hi])[0]

    def ngroups(self):
        return len(self._gids()), False

    def emit(self, ngroups, sort=True):
        g = self._gids()
        assert len(g) == ngroups
        sums = cnts = sizes = None
        if self.acc is not None:
            a = self.acc.numpy().reshape(self.R, self.vs)[g]
            if not self.flags & _lib.GB_SUM:
                empty = a == (np.iinfo(np.int64).max if self.flags & _lib.GB_MIN else np.iinfo(np.int64).min)
                a = np.where(empty, np.nan, (a ^ ((a >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))).view(np.float64))
            sums = [_col(np.ascontiguousarray(a[:, v])) for v in range(self.nvals)]
        if self.cnt is not None:
            c = self.cnt.numpy().reshape(self.R, self.vs)[g]
            cnts = [_col(np.ascontiguousarray(c[:, v])) for v in range(self.nvals)]
        if self.size is not None:
            sizes = _col(self.size.numpy()[g])
        return _col((g + self.kbase).astype(np.int64)), sums, cnts, sizes

    def emit_async(self):
        ng, _ = self.ngroups()
        keys, sums, cnts, sizes = self.emit(ng, sort=False)
        lo, hi = self.win
        cap = hi - lo

        def pad(col):
            if col is None:
                return None
            a = _np(col)
            return _col(np.concatenate([a, np.zeros(cap - len(a), dtype=a.dtype)]))

        return (pad(keys), [pad(c) for c in sums] if sums else None, [pad(c) for c in cnts] if cnts else None, pad(sizes),
                torch.tensor([ng, 0], dtype=torch.int64))

    def close(self):
        pass


class JoinTable:
    def __init__(self, dim_keys):
        self.keys = _np(dim_keys)
        self.index = pandas.Index(self.keys)

    def is_unique(self):
        return bool(self.index.is_unique)

    def _idx(self, fact_keys):
        if self.index.is_unique:
            return self.index.get_indexer(_np(fact_keys)).astype(np.int64)
        # repeated dim keys: the device table keeps ONE row per key (hit / miss is what callers use it for)
        uniq, first = np.unique(self.keys, return_index=True)
        fk = _np(fact_keys)
        pos = np.searchsorted(uniq, fk)
        pos_c = np.minimum(pos, len(uniq) - 1)
        return np.where(uniq[pos_c] == fk, first[pos_c], -1).astype(np.int64)

    def probe(self, fact_keys):
        idx = self._idx(fact_keys)
        return _col(idx), torch.tensor([int((idx >= 0).sum())])

    def probe_gather(self, fact_keys, dim_cols):
        idx = self._idx(fact_keys)
        outs = []
        for c in dim_cols:
            x = _np(c)
            null = np.nan if c.dtype == np.float64 else 0
            if len(x) == 0:  # empty dim table: every row misses (the kernel never dereferences a dim row on a miss)
                outs.append(_col(np.full(len(idx), null).astype(c.dtype)))
                continue
            outs.append(_col(np.where(idx >= 0, x[np.maximum(idx, 0)], null).astype(c.dtype)))
        return outs, torch.tensor([int((idx >= 0).sum())])

    def close(self):
        pass


def take_columns(cols, idx):
    i = _np(idx)
    outs = []
    for c in cols:
        x = _np(c)
        null = np.nan if c.dtype == np.float64 else 0
        if len(x) == 0:  # empty source: only negative (null) positions are legal, nothing is dereferenced
            assert not (i >= 0).any(), "take from an empty column with a non-negative position"
            outs.append(_col(np.full(len(i), null).astype(c.dtype)))
            continue
        outs.append(_col(np.where(i >= 0, x[np.maximum(i, 0)], null).astype(c.dtype)))
    return outs


def compact_hits(idx):
    pos = np.nonzero(_np(idx) >= 0)[0].astype(np.int64)
    return _col(pos), len(pos)


def cast_columns_f64(cols):
    return [c if c.dtype == np.float64 else _col(_np(c).astype(np.float64)) for c in cols]


def cast_columns_i64(cols):
    return [_col(_np(c).astype(np.int64)) if c.dtype == np.bool_ else c for c in cols]


def expand_matches(fact_keys, dim_keys, keep_misses):
    fk, dk = _np(fact_keys), _np(dim_keys)
    order = np.argsort(dk, kind="stable")
    ks = dk[order]
    lo, hi = np.searchsorted(ks, fk, side="left"), np.searchsorted(ks, fk, side="right")
    cnt = hi - lo
    out_cnt = np.where(cnt > 0, cnt, 1 if keep_misses else 0)
    left = np.repeat(np.arange(len(fk), dtype=np.int64), out_cnt)
    offs = np.concatenate([[0], np.cumsum(out_cnt)[:-1]]) if len(fk) else np.zeros(0, dtype=np.int64)
    within = np.arange(len(left), dtype=np.int64) - np.repeat(offs, out_cnt)
    src = np.repeat(lo, out_cnt) + within
    hit = np.repeat(cnt > 0, out_cnt)
    right = np.where(hit, order[np.minimum(src, max(len(order) - 1, 0))] if len(order) else -1, -1).astype(np.int64)
    return _col(left), _col(right), int((cnt == 0).sum())


def concat_columns(pieces):
    pieces = list(pieces)
    return pieces[0] if len(pieces) == 1 else _col(np.concatenate([_np(p) for p in pieces]))


_CUM_ID = {"sum": -0.0, "max": -np.inf, "min": np.inf, "ffill": np.nan}  # -0.0: x + -0.0 = x (csrc/cum.cu)


def _cum_comb(op, a, b):
    if op == "sum":
        return a + b
    if op == "max":  # ties go to the later operand, b
        return np.where(b >= a, b, a)
    if op == "min":
        return np.where(b <= a, b, a)
    return np.where(np.isnan(b), a, b)


def _cum_ident(op, dtype):
    if dtype == np.float64:
        return np.float64(_CUM_ID[op])
    return np.int64({"sum": 0, "max": np.iinfo(np.int64).min, "min": np.iinfo(np.int64).max}[op])


def cum_partials(op, cols):
    n = len(cols[0]) if cols else 0
    st = ops.CumState(op, n)
    by_code = {}
    for j, c in enumerate(cols):
        if c.dtype == np.bool_ or (op == "ffill" and c.dtype != np.float64):
            raise TypeError(f"cumulative {op} over {c.dtype} columns is not on the B200 path")
        by_code.setdefault(c.code, []).append(j)
    for code, idxs in by_code.items():
        tot = []
        for j in idxs:
            x = _np(cols[j])
            v = x[~np.isnan(x)] if x.dtype == np.float64 else x
            if op == "sum" and x.dtype == np.float64:
                v = np.where(np.isnan(x), 0.0, x)  # NaN rows add +0.0
            ident = _cum_ident(op, x.dtype)
            with np.errstate(all="ignore"):
                tot.append(ident if len(v) == 0 else {"sum": lambda: np.cumsum(v)[-1], "max": v.max, "min": v.min,
                                                     "ffill": lambda: v[-1]}[op]())  # cumsum: -0.0 + -0.0 stays -0.0
        st.groups.append((code, idxs, None, torch.from_numpy(np.asarray(tot, dtype=_np(cols[idxs[0]]).dtype))))
    return st


def cum_carry(state, gathered, rank):
    out = []
    for (code, idxs, _s, totals), g in zip(state.groups, gathered):
        g = g.numpy().reshape(-1, len(idxs))
        run = np.full(len(idxs), _cum_ident(state.op, g.dtype), dtype=g.dtype)
        with np.errstate(all="ignore"):
            for r in range(rank):
                run = _cum_comb(state.op, run, g[r]).astype(g.dtype)
        out.append(torch.from_numpy(run))
    return out


def cum_apply(state, cols, carries=None):
    outs = [None] * len(cols)
    op = state.op
    for k, (code, idxs, _s, _t) in enumerate(state.groups):
        for pos, j in enumerate(idxs):
            x = _np(cols[j])
            ident = _cum_ident(op, x.dtype)
            carry = carries[k].numpy()[pos] if carries is not None else ident
            nan = np.isnan(x) if x.dtype == np.float64 else np.zeros(len(x), dtype=bool)
            with np.errstate(all="ignore"):
                if op == "ffill":
                    r = pandas.Series(x).ffill().to_numpy()
                    r = np.where(np.isnan(r), carry, r)
                else:
                    v = np.where(nan, x.dtype.type(0) if op == "sum" else ident, x)  # int64 stays int64 (and wraps)
                    acc = {"sum": np.cumsum, "max": np.maximum.accumulate, "min": np.minimum.accumulate}[op](v)
                    r = _cum_comb(op, np.full(len(x), carry, dtype=x.dtype), acc).astype(x.dtype)
                    if x.dtype == np.float64:
                        r = np.where(nan, np.nan, r)
            outs[j] = _col(r)
    return outs


def run_starts(sorted_keys):
    b = _np(sorted_keys)
    if len(b) == 0:
        return np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64)
    starts = np.nonzero(np.concatenate([[True], b[1:] != b[:-1]]))[0].astype(np.int64)
    return starts, b[starts]


def digitize(values, pivots):
    return _col(np.searchsorted(np.asarray(list(pivots), dtype=np.int64), _np(values), side="right").astype(np.int64))


def iota(start, nrows):
    return _col(np.arange(start, start + nrows, dtype=np.int64))


def full_column(nrows, dtype, value):
    return _col(np.full(nrows, value, dtype=np.dtype(dtype)))


@contextlib.contextmanager
def installed():
    """Swap the device for the double (context manager used by the ``cpu_device`` fixture)."""
    from modin_b200 import synth

    saved = {
        "current_device": block.current_device,
        **{n: getattr(ops, n) for n in ("map_columns", "reduce_columns", "hash_aggregate", "JoinTable", "take_columns",
                                        "compact_hits", "cast_columns_f64", "cast_columns_i64", "gen_f64", "gen_i64", "GroupTable",
                                        "key_range_device", "sort_pairs", "iota", "full_column", "expand_matches", "digitize", "run_starts", "concat_columns", "cum_partials", "cum_carry", "cum_apply")},
    }  # fmt: skip
    ops.GroupTable, ops.key_range_device, ops.sort_pairs = GroupTable, key_range_device, sort_pairs
    ops.iota, ops.full_column, ops.expand_matches, ops.digitize = iota, full_column, expand_matches, digitize
    ops.run_starts, ops.concat_columns = run_starts, concat_columns
    ops.cum_partials, ops.cum_carry, ops.cum_apply = cum_partials, cum_carry, cum_apply
    ops.cast_columns_i64 = cast_columns_i64
    block.current_device = lambda: torch.device("cpu")
    ops.current_device = block.current_device
    ops.map_columns, ops.reduce_columns, ops.hash_aggregate = map_columns, reduce_columns, hash_aggregate
    ops.JoinTable, ops.take_columns, ops.compact_hits, ops.cast_columns_f64 = JoinTable, take_columns, compact_hits, \
        cast_columns_f64  # fmt: skip
    ops.gen_f64 = lambda n, seed, col, row_offset=0, nan_per_64k=0: _col(synth.gen_f64(n, seed, col, row_offset, nan_per_64k))
    ops.gen_i64 = lambda n, seed, col, modulus, row_offset=0, skew=False: _col(
        (synth.gen_i64_skew if skew else synth.gen_i64)(n, seed, col, modulus, row_offset))
    try:
        yield
    finally:
        block.current_device = saved.pop("current_device")
        ops.current_device = block.current_device
        for n, v in saved.items():
            setattr(ops, n, v)
