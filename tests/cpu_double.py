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


def key_range_device(key_cols):
    ks = [_np(k) for k in key_cols if len(k)]
    if not ks:
        return torch.tensor([np.iinfo(np.int64).max, np.iinfo(np.int64).min, 0, 0], dtype=torch.int64)
    return torch.tensor([min(int(k.min()) for k in ks), max(int(k.max()) for k in ks), 0, 0], dtype=torch.int64)


class GroupTable(ops.GroupTable):
    """numpy stand-in for the device group table, hashed or dense (dense arrays in the layout of include/modin_b200.h,
    so that the fused path's cross-rank merge by collectives runs under gloo).  Only the calls into the library are
    replaced: filling, the counted emit, the dense-or-hashed choice and the reduce-scatter are the real code.

    ``created`` lists the kind of every table made ("hashed", "dense", or "slice" for a reduce-scattered part);
    ``round_trips`` counts ``ngroups()`` calls, the host round trip of a counted emit."""

    created: list = []
    round_trips = 0

    def __init__(self, group_capacity, nvals, flags):
        R, vs = int(group_capacity), ops.value_stride(nvals)
        arrays = {"acc": torch.empty(R * vs, dtype=torch.float64 if flags & _lib.GB_SUM else torch.int64),
                  "cnt": torch.empty(R * vs, dtype=torch.int64), "size": torch.empty(R, dtype=torch.int64)}  # fmt: skip
        self._setup(None, R, nvals, flags, arrays, "hashed")
        self.keys = np.zeros(0, dtype=np.int64)  # distinct keys, by group id

    @classmethod
    def _dense_table(cls, kbase, nkeys, nvals, flags, arrays, parent=None):
        self = cls.__new__(cls)
        self._setup(kbase, nkeys, nvals, flags, arrays, "dense" if parent is None else "slice")
        if parent is not None:  # the reduce-scattered arrays hold merged values
            self.overflow = parent.overflow
        return self

    def _setup(self, kbase, capacity, nvals, flags, arrays, kind):
        self.kbase, self.capacity, self.nvals, self.flags = kbase, int(capacity), int(nvals), int(flags)
        self.vs = ops.value_stride(nvals)
        self.acc, self.cnt, self.size, self.present = (arrays.get(n) for n in ("acc", "cnt", "size", "present"))
        if not flags & (_lib.GB_SUM | _lib.GB_MIN | _lib.GB_MAX):
            self.acc = None
        if not flags & _lib.GB_COUNT:
            self.cnt = None
        if not flags & _lib.GB_SIZE:
            self.size = None
        if kind != "slice":  # what mb200_gb_create / _create_dense clear the arrays to
            if self.acc is not None:
                ident = 0 if flags & _lib.GB_SUM else np.iinfo(np.int64).max if flags & _lib.GB_MIN else np.iinfo(np.int64).min
                self.acc.fill_(ident)
            for x in (self.cnt, self.size, self.present):
                if x is not None:
                    x.zero_()
        self.overflow = False
        self.win = (0, self.capacity)
        GroupTable.created.append(kind)

    @staticmethod
    def _ordered(x):  # order-preserving int64 image of float64 (csrc/groupby.cu f64_to_ordered)
        b = x.view(np.int64)
        return b ^ ((b >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))

    def _gids(self, keys):
        """Group id of every row; ``capacity`` for a row whose key found no room (the table then overflows)."""
        k = _np(keys)
        if self.kbase is not None:
            g = k - self.kbase
            outside = (g < 0) | (g >= self.capacity)
            self.overflow |= bool(outside.any())
            return np.where(outside, self.capacity, g)
        new = np.setdiff1d(k, self.keys)
        room = self.capacity - len(self.keys)
        if len(new) > room:
            self.overflow = True
        self.keys = np.concatenate([self.keys, new[:room]])
        order = np.argsort(self.keys, kind="stable")
        pos = np.minimum(np.searchsorted(self.keys[order], k), max(len(order) - 1, 0))
        found = self.keys[order][pos] == k if len(order) else np.zeros(len(k), dtype=bool)
        return np.where(found, order[pos] if len(order) else 0, self.capacity)

    def _add(self, keys, vals, cnts=None, sizes=None):
        """Rows into the table: raw values (count the non-NaN ones, one row each), or with ``cnts`` / ``sizes`` the
        columns of partial tables.  NaN values are skipped either way, as the kernel does."""
        g = self._gids(keys)
        live = g < self.capacity
        g = g[live]
        if self.present is not None:
            self.present.numpy()[g] = 1
        if self.size is not None:
            np.add.at(self.size.numpy(), g, _np(sizes)[live] if sizes is not None else 1)
        for v, col in enumerate(vals or []):
            x = _np(col)[live]
            ok = ~np.isnan(x)
            o = g[ok] * self.vs + v
            if self.flags & _lib.GB_SUM:
                np.add.at(self.acc.numpy(), o, x[ok])
            elif self.flags & _lib.GB_MIN:
                np.minimum.at(self.acc.numpy(), o, self._ordered(x[ok]))
            elif self.flags & _lib.GB_MAX:
                np.maximum.at(self.acc.numpy(), o, self._ordered(x[ok]))
            if self.cnt is not None:
                np.add.at(self.cnt.numpy(), g * self.vs + v, _np(cnts[v])[live] if cnts is not None else ok.astype(np.int64))

    def accumulate(self, keys, vals):
        self._add(keys, vals)

    def merge_partial(self, keys, sums, cnts=None, sizes=None):
        self._add(keys, sums, cnts, sizes)

    def hint_skew(self, skewed):
        pass

    def window(self, lo, hi):
        assert lo % 4 == 0 and (hi % 4 == 0 or hi == self.capacity) and 0 <= lo <= hi <= self.capacity
        self.win = (int(lo), int(hi))

    def _rows(self, sort):
        """Group ids in emit order: a dense table's present keys of the window, ascending; a hashed table's groups,
        ascending by key when ``sort``."""
        if self.kbase is not None:
            lo, hi = self.win
            return lo + np.nonzero(self.present.numpy()[lo:hi])[0]
        g = np.arange(min(len(self.keys), self.capacity))
        return g[np.argsort(self.keys[g], kind="stable")] if sort else g

    def ngroups(self):
        GroupTable.round_trips += 1
        return len(self._rows(False)), self.overflow

    def _emit(self, g):
        sums = cnts = sizes = None
        if self.acc is not None:
            a = self.acc.numpy().reshape(self.capacity, self.vs)[g]
            if not self.flags & _lib.GB_SUM:
                empty = a == (np.iinfo(np.int64).max if self.flags & _lib.GB_MIN else np.iinfo(np.int64).min)
                a = np.where(empty, np.nan, (a ^ ((a >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))).view(np.float64))
            sums = [_col(np.ascontiguousarray(a[:, v])) for v in range(self.nvals)]
        if self.cnt is not None:
            c = self.cnt.numpy().reshape(self.capacity, self.vs)[g]
            cnts = [_col(np.ascontiguousarray(c[:, v])) for v in range(self.nvals)]
        if self.size is not None:
            sizes = _col(self.size.numpy()[g])
        keys = g + self.kbase if self.kbase is not None else self.keys[g]
        return _col(keys.astype(np.int64)), sums, cnts, sizes

    def emit(self, ngroups, sort=True):
        if self.overflow and self.kbase is None:
            raise _lib.B200Error("mb200_gb_emit: table overflowed: recreate with a larger group capacity")
        g = self._rows(sort)
        assert len(g) == ngroups
        return self._emit(g)

    def emit_async(self):
        g = self._rows(False)
        keys, sums, cnts, sizes = self._emit(g)
        lo, hi = self.win
        cap = hi - lo

        def pad(col):
            if col is None:
                return None
            a = _np(col)
            return _col(np.concatenate([a, np.zeros(cap - len(a), dtype=a.dtype)]))

        return (pad(keys), [pad(c) for c in sums] if sums else None, [pad(c) for c in cnts] if cnts else None, pad(sizes),
                torch.tensor([len(g), int(self.overflow)], dtype=torch.int64))

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
        **{n: getattr(ops, n) for n in ("map_columns", "reduce_columns", "JoinTable", "take_columns",
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
    ops.map_columns, ops.reduce_columns = map_columns, reduce_columns
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
