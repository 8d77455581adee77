"""``groupby.first`` / ``last`` through both front doors, with the device replaced by the numpy test double: the
functors (one position table per partition, one gather per column, the reduce over concatenated partial values),
the shared groupby caller (``skipna`` / ``min_count``, several keys, float keys, ``level=0``, ``as_index=False``,
dictionaries) and the rank-order combine under 2 and 3 gloo ranks.  Results are compared with pandas for values
(bit for bit), index and dtypes.  ``PositionTable`` below is the numpy twin of a FIRST / LAST group table
(csrc/groupby.cu): min / max of row positions, NULL value columns, positions running on across accumulate calls, and
-1 for a group without a value on emit."""

import contextlib
import os
import sys

import numpy as np
import pandas
import pytest

from modin_b200 import _lib, config, ops

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref")
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
POS = _lib.GB_FIRST | _lib.GB_LAST


@contextlib.contextmanager
def double_installed():
    sys.path.insert(0, HERE)
    import cpu_double

    class PositionTable(cpu_double.GroupTable):
        """The double's group table, playing FIRST / LAST tables as well."""

        def _setup(self, kbase, capacity, nvals, flags, arrays, kind):
            super()._setup(kbase, capacity, nvals, flags, arrays, kind)
            self.rows = 0
            if flags & POS:
                self.acc = arrays["acc"]
                if kind != "slice":
                    self.acc.fill_(I64_MAX if flags & _lib.GB_FIRST else I64_MIN)

        def accumulate(self, keys, vals):
            if any(v is None for v in vals) and not self.flags & POS or any(v is not None and v.dtype != np.float64 for v in vals):
                raise TypeError("device groupby aggregates float64 value columns")  # as GroupTable.accumulate
            if not self.flags & POS:
                return super().accumulate(keys, vals)
            g = self._gids(keys)
            live = g < self.capacity
            pos = self.rows + np.arange(len(g), dtype=np.int64)
            self.rows += len(g)
            if self.present is not None:
                self.present.numpy()[g[live]] = 1
            if self.size is not None:
                np.add.at(self.size.numpy(), g[live], 1)
            red = np.minimum.at if self.flags & _lib.GB_FIRST else np.maximum.at
            for v, col in enumerate(vals):
                ok = live if col is None else live & ~np.isnan(col.data.numpy())
                red(self.acc.numpy(), g[ok] * self.vs + v, pos[ok])

        def merge_partial(self, keys, sums, cnts=None, sizes=None):
            if self.flags & POS:
                raise _lib.B200Error("groupby: FIRST / LAST tables do not merge partial tables")
            return super().merge_partial(keys, sums, cnts, sizes)

        def _emit(self, g):
            if not self.flags & POS:
                return super()._emit(g)
            acc, self.acc = self.acc, None
            try:
                keys, _, cnts, sizes = super()._emit(g)
            finally:
                self.acc = acc
            a = acc.numpy().reshape(self.capacity, self.vs)[g]
            a = np.where(a == (I64_MAX if self.flags & _lib.GB_FIRST else I64_MIN), -1, a)
            return keys, [cpu_double._col(np.ascontiguousarray(a[:, v])) for v in range(self.nvals)], cnts, sizes

    with cpu_double.installed():
        ops.GroupTable = PositionTable
        yield PositionTable


@pytest.fixture
def dev():
    old = config.NPartitions.get()
    with double_installed():
        yield
    config.NPartitions.put(old)


def _frame(n=41, seed=5, groups=6):
    """Keys 0..groups-1 plus a group (99) whose float values are all NaN; float columns with NaN at a group's first and
    last rows, signed zeros and infinities; int64 with its limits; bool."""
    rng = np.random.default_rng(seed)
    key = rng.integers(0, groups, n)
    key[[3, 17, 30]] = 99
    f = rng.standard_normal(n)
    f[rng.random(n) < 0.3] = np.nan
    for k in range(groups):  # NaN at every group's first and last row
        rows = np.flatnonzero(key == k)
        if len(rows) > 2:
            f[rows[0]] = f[rows[-1]] = np.nan
    f[key == 99] = np.nan
    z = np.where(np.arange(n) % 2 == 0, -0.0, 0.0)
    z[rng.random(n) < 0.2] = np.nan
    inf = np.where(np.arange(n) % 3 == 0, np.inf, -np.inf)
    inf[key == 99] = np.nan
    lim = np.where(np.arange(n) % 4 == 0, I64_MIN, np.where(np.arange(n) % 4 == 1, I64_MAX, np.arange(n)))
    return pandas.DataFrame({"key": key.astype(np.int64), "f": f, "i": lim.astype(np.int64), "b": rng.random(n) < 0.5,
                             "z": z, "inf": inf})  # fmt: skip


def _same(got, want):
    """Values bit for bit (NaN == NaN, -0.0 != 0.0), index and dtypes."""
    pandas.testing.assert_index_equal(got.index, want.index, exact=False)
    assert list(got.columns) == list(want.columns), (list(got.columns), list(want.columns))
    assert list(got.dtypes) == list(want.dtypes), (list(got.dtypes), list(want.dtypes))
    for j in range(want.shape[1]):
        a, b = got.iloc[:, j].to_numpy(), want.iloc[:, j].to_numpy()
        if a.dtype == np.float64:
            nan = np.isnan(b)
            assert np.array_equal(np.isnan(a), nan) and np.array_equal(a[~nan].view(np.int64), b[~nan].view(np.int64)), j
        else:
            assert np.array_equal(a, b), j


def _cases(mk, pdf):
    df = mk(pdf)
    for fn in ("first", "last"):
        for kw in ({}, {"skipna": False}, {"min_count": -1}, {"min_count": 0}, {"min_count": 1}):
            _same(getattr(df.groupby("key"), fn)(**kw)._to_pandas(), getattr(pdf.groupby("key"), fn)(**kw))
        _same(getattr(df[["key", "i", "b"]].groupby("key"), fn)()._to_pandas(), getattr(pdf[["key", "i", "b"]].groupby("key"), fn)())
        _same(df.groupby("key").agg(fn)._to_pandas(), pdf.groupby("key").agg(fn))
        _same(getattr(df.groupby("key", as_index=False), fn)()._to_pandas(), getattr(pdf.groupby("key", as_index=False), fn)())
    spec = {"f": "first", "i": "last", "z": "sum", "b": "last", "inf": "first"}
    _same(df.groupby("key").agg(spec)._to_pandas(), pdf.groupby("key").agg(spec))


# ------------------------------------------------------------------ the Modin-free mirror (modin_b200.pandas)
@pytest.mark.parametrize("nparts", [1, 3])
def test_mirror_first_last_match_pandas(dev, nparts):
    import modin_b200.pandas as bpd

    config.NPartitions.put(nparts)
    _cases(bpd.DataFrame, _frame())


def test_mirror_uneven_partitions_two_keys_and_forty_columns(dev):
    import modin_b200.pandas as bpd

    config.NPartitions.put(1)
    pdf = _frame(53, seed=8)
    cuts = [0, 3, 4, 30, 53]  # row partitions of 3, 1, 26 and 23 rows
    df = bpd.concat([bpd.DataFrame(pdf.iloc[a:b]) for a, b in zip(cuts, cuts[1:])], ignore_index=True)
    assert [len(r) for r in df._query_compiler._modin_frame._partitions] == [1, 1, 1, 1]
    for fn in ("first", "last"):
        for kw in ({}, {"skipna": False}):
            _same(getattr(df.groupby("key"), fn)(**kw)._to_pandas(), getattr(pdf.groupby("key"), fn)(**kw))
    config.NPartitions.put(3)
    two = pdf.assign(k2=(np.arange(len(pdf)) % 3).astype(np.int64))
    kinds = ["f", "i", "b", "z", "inf"]
    wide = pandas.DataFrame({"key": pdf["key"], **{f"c{j}": np.roll(pdf[kinds[j % 5]].to_numpy(), j) for j in range(40)}})
    for fn in ("first", "last"):
        for kw in ({}, {"skipna": False}):
            _same(getattr(bpd.DataFrame(two).groupby(["key", "k2"]), fn)(**kw)._to_pandas(),
                  getattr(two.groupby(["key", "k2"]), fn)(**kw))  # fmt: skip
            _same(getattr(bpd.DataFrame(wide).groupby("key"), fn)(**kw)._to_pandas(), getattr(wide.groupby("key"), fn)(**kw))


@pytest.mark.parametrize("dense", [True, False])
def test_mirror_dense_and_hashed_tables(dev, dense):
    import modin_b200.pandas as bpd

    old = config.GroupbyDenseKeys.get()
    config.GroupbyDenseKeys.put(dense)
    try:
        config.NPartitions.put(2)
        pdf = _frame(97, seed=2, groups=11)
        for fn in ("first", "last"):
            _same(getattr(bpd.DataFrame(pdf).groupby("key"), fn)()._to_pandas(), getattr(pdf.groupby("key"), fn)())
    finally:
        config.GroupbyDenseKeys.put(old)


def test_mirror_refusals(dev):
    import modin_b200.pandas as bpd

    df = bpd.DataFrame(_frame())
    for fn in ("first", "last"):
        with pytest.raises(NotImplementedError, match="min_count"):
            getattr(df.groupby("key"), fn)(min_count=2)


def test_position_table_stand_in_runs_on_across_calls(dev):
    """Positions continue across accumulate calls; NULL columns count every row; -1 for a group without a value."""
    from tests import cpu_double

    keys = cpu_double._col(np.array([5, 7, 5], dtype=np.int64))
    v = cpu_double._col(np.array([np.nan, 1.0, 2.0]))
    for flag, want in ((_lib.GB_FIRST, ([0, 1], [2, -1])), (_lib.GB_LAST, ([5, 4], [5, 4]))):
        t = ops.GroupTable(16, 2, flag)
        t.accumulate(keys, [None, v])
        t.accumulate(cpu_double._col(np.array([7, 9, 5], dtype=np.int64)), [None, cpu_double._col(np.array([np.nan] * 3))])
        k, s, _, _ = ops.emit_counted(t)
        assert k.data.numpy().tolist() == [5, 7, 9]
        if flag == _lib.GB_FIRST:
            assert s[0].data.numpy().tolist() == [0, 1, 4] and s[1].data.numpy().tolist() == [2, 1, -1]
        else:
            assert s[0].data.numpy().tolist() == [5, 3, 4] and s[1].data.numpy().tolist() == [2, 1, -1]
        with pytest.raises(_lib.B200Error):
            t.merge_partial(k, s)
    with pytest.raises(TypeError):
        ops.GroupTable(16, 1, _lib.GB_MAX).accumulate(keys, [None])


# ------------------------------------------------------------------ real modin.pandas with the plug-in
needs_modin = pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "modin")),
                                 reason="reference Modin not installed under oracle/_ref")  # fmt: skip


@pytest.fixture(scope="module")
def mpd():
    if REF not in sys.path:
        sys.path.insert(0, REF)
    import warnings

    warnings.filterwarnings("ignore")
    from modin_b200 import modin_plugin

    modin_plugin.register()
    import modin
    import modin.config as cfg
    import modin.pandas as mpd

    modin.set_execution(engine="B200", storage_format="Arrow")
    cfg.NPartitions.put(4)
    yield mpd


@needs_modin
@pytest.mark.parametrize("nparts", [1, 3])
def test_plugin_first_last_match_pandas(mpd, dev, nparts):
    import modin.config as cfg

    cfg.NPartitions.put(nparts)
    config.NPartitions.put(nparts)
    pdf = _frame()
    _cases(mpd.DataFrame, pdf)
    # float key (NaN group kept or dropped), two int64 keys, level=0, Series groupby
    fk = pdf.assign(key=np.where(pdf["key"] == 2, np.nan, pdf["key"] * 0.5 - 1.0))
    two = pdf.assign(k2=(np.arange(len(pdf)) % 3).astype(np.int64))
    lab = pdf.drop(columns="key").set_axis(pandas.Index(pdf["key"].to_numpy(), name="lab"))
    for fn in ("first", "last"):
        for dropna in (True, False):
            _same(getattr(mpd.DataFrame(fk).groupby("key", dropna=dropna), fn)()._to_pandas(),
                  getattr(fk.groupby("key", dropna=dropna), fn)())  # fmt: skip
        _same(getattr(mpd.DataFrame(two).groupby(["key", "k2"]), fn)()._to_pandas(), getattr(two.groupby(["key", "k2"]), fn)())
        _same(getattr(mpd.DataFrame(lab).groupby(level=0), fn)()._to_pandas(), getattr(lab.groupby(level=0), fn)())
        got = getattr(mpd.DataFrame(pdf).groupby("key")["f"], fn)()._to_pandas()
        pandas.testing.assert_series_equal(got, getattr(pdf.groupby("key")["f"], fn)())


@needs_modin
def test_plugin_refusals(mpd, dev):
    df = mpd.DataFrame(_frame())
    for fn in ("first", "last"):
        with pytest.raises(NotImplementedError, match="min_count"):
            getattr(df.groupby("key"), fn)(min_count=2)


# ------------------------------------------------------------------ ranks (gloo, one process per rank)
def _free_port():
    import socket

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, ws, port, ret):
    import torch.distributed as tdist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(ws))
    tdist.init_process_group("gloo", rank=rank, world_size=ws)
    try:
        ret[rank] = _rank_job(rank, ws)
    finally:
        tdist.destroy_process_group()


def _rank_frames(ws):
    """``full``: 14 rows per rank, every group on every rank; group 1 has one valid ``f`` before the last rank (row 1)
    and the rest on the last rank, so its first comes from rank 0 and its last from the last rank; ``tiny``: fewer rows
    than ranks, so the last rank has none -- both with a bool column, which crosses the exchange as int64."""
    n = 14 * ws
    r = np.arange(n)
    key = (r % 4).astype(np.int64)
    f = np.where(r % 5 == 0, np.nan, np.sin(r))
    f[(key == 1) & (r < n - 14)] = np.nan
    f[(key == 1) & (r == 1)] = 7.5
    full = pandas.DataFrame({"key": key, "f": f, "i": r * 3 - 20, "b": r % 3 == 1})
    return {"full": full, "tiny": full.iloc[: ws - 1].copy()}


def _rank_job(rank, ws):
    import modin_b200.pandas as bpd

    out = {}
    with double_installed():
        config.NPartitions.put(2)
        for dense in (True, False):
            config.GroupbyDenseKeys.put(dense)
            for name, pdf in _rank_frames(ws).items():
                df = bpd.DataFrame(pdf)
                for fn in ("first", "last"):
                    for skipna in (True, False):
                        out[(dense, name, fn, skipna)] = getattr(df.groupby("key"), fn)(skipna=skipna)._to_pandas()
            # rows of rank ws - 2 are filtered away (row selection takes frames without bool columns)
            pdf = _rank_frames(ws)["full"].drop(columns="b")
            keep = np.arange(len(pdf)) // 14 != ws - 2
            dm = bpd.DataFrame(pdf)[bpd.DataFrame(pandas.DataFrame({"m": keep}))["m"]]
            for fn in ("first", "last"):
                out[(dense, "masked", fn, True)] = getattr(dm.groupby("key"), fn)()._to_pandas()
    return out


@pytest.mark.parametrize("ws", [2, 3])
def test_ranks_combine_in_rank_order(ws):
    import torch.multiprocessing as mp

    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(ws, _free_port(), ret), nprocs=ws, join=True)
    frames = _rank_frames(ws)
    full = frames["full"].drop(columns="b")
    frames["masked"] = full[np.arange(len(full)) // 14 != ws - 2]
    for r in range(ws):  # every rank holds the whole answer
        assert len(ret[r]) == 2 * (2 * 2 * 2 + 2)
        for (dense, name, fn, skipna), got in ret[r].items():
            _same(got, getattr(frames[name].groupby("key"), fn)(skipna=skipna))
    assert frames["full"].groupby("key")["f"].first()[1] == 7.5
