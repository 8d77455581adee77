"""``groupby.nunique`` through both front doors, with the device replaced by the numpy test double: the functor (one
NUNIQUE table per column batch over every row partition, the distinct-set emit, sort and key-range exchange across
ranks), the shared groupby caller (keys of every kind, ``as_index=False``, ``agg`` and dictionaries, refusals) and 2 and
3 gloo ranks.  Results are compared with pandas 3.0.2 for values, index, column labels and dtypes.  ``NuniqueTable``
below is the numpy twin of a NUNIQUE group table (csrc/groupby.cu): pass 1 is the SIZE table, pass 2 inserts (group,
column, image) entries into a set of fixed capacity and counts the new ones, a full set raises the overflow flag, and
``emit_distinct`` lists one (key, -1, 0) row per group, then the entries."""

import contextlib
import os
import sys

import numpy as np
import pandas
import pytest

from modin_b200 import _lib, config, functors, ops

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref")
NUNIQUE = _lib.GB_SIZE | _lib.GB_NUNIQUE
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
NAN_IMAGE = 0x7FF8000000000000

pytestmark = pytest.mark.skipif(pandas.__version__ != "3.0.2", reason="the expected results are pandas 3.0.2's")


def images(x: np.ndarray, dropna: bool):
    """(image, counted) of raw values: int64 as is; float64 through the order-preserving image, -0.0 as 0.0, every NaN
    one image (left out under ``dropna``)."""
    if x.dtype == np.int64:
        return x.copy(), np.ones(len(x), dtype=bool)
    b = x.view(np.int64)
    img = b ^ ((b >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))
    img = np.where(x == 0.0, 0, img)
    nan = np.isnan(x)
    return np.where(nan, NAN_IMAGE, img).astype(np.int64), ~nan | (not dropna)


@contextlib.contextmanager
def double_installed():
    sys.path.insert(0, HERE)
    import cpu_double

    class NuniqueTable(cpu_double.GroupTable):
        """The double's group table, playing NUNIQUE tables as well."""

        def _setup(self, kbase, capacity, nvals, flags, arrays, kind):
            if flags & _lib.GB_NUNIQUE and flags != NUNIQUE:
                raise _lib.B200Error("mb200_gb_create: a NUNIQUE table is SIZE | NUNIQUE")
            super()._setup(kbase, capacity, nvals, flags, arrays, kind)
            if flags & _lib.GB_NUNIQUE:
                self.cnt = arrays["cnt"]
                self.cnt.zero_()
            self.dset, self.dcap, self.distinct_filled = None, 0, False

        def _pass1(self):
            if self.distinct_filled:
                raise _lib.B200Error("a NUNIQUE table takes no rows after mb200_gb_accumulate_distinct")

        def accumulate(self, keys, vals):
            self._pass1()
            return super().accumulate(keys, [] if self.flags & _lib.GB_NUNIQUE else vals)

        def merge_partial(self, keys, sums, cnts=None, sizes=None):
            self._pass1()
            return super().merge_partial(keys, sums, cnts, sizes)

        def reserve_distinct(self, capacity):
            if not self.flags & _lib.GB_NUNIQUE:
                raise _lib.B200Error("mb200_gb_reserve_distinct: not a NUNIQUE table")
            if capacity < 1 or capacity & (capacity - 1):
                raise _lib.B200Error("mb200_gb_reserve_distinct: capacity must be a power of two")
            self.dset, self.dcap = {}, int(capacity)  # entry image -> nothing, in insertion order

        def _lookup(self, k):
            """Read-only group ids: pass 2 adds no group."""
            if self.kbase is not None:
                g = k - self.kbase
                return g, (g >= 0) & (g < self.capacity)
            order = np.argsort(self.keys, kind="stable")
            pos = np.minimum(np.searchsorted(self.keys[order], k), max(len(order) - 1, 0))
            live = self.keys[order][pos] == k if len(order) else np.zeros(len(k), dtype=bool)
            return (order[pos] if len(order) else np.zeros(len(k), dtype=np.int64)), live

        def accumulate_distinct(self, keys, vals=None, dropna=True, col_ids=None, images=None):
            if self.dset is None:
                raise _lib.B200Error("mb200_gb_accumulate_distinct: no distinct set")
            self.distinct_filled = True
            g, live = self._lookup(cpu_double._np(keys))
            pairs = []
            if col_ids is None:
                for v, col in enumerate(vals):
                    img, ok = globals()["images"](cpu_double._np(col), dropna)
                    ok &= live
                    pairs += list(zip((g[ok] * self.vs + v).tolist(), img[ok].tolist()))
            else:
                j, img = cpu_double._np(col_ids), cpu_double._np(images)
                ok = live & (j >= 0) & (j < self.nvals)
                pairs += list(zip((g[ok] * self.vs + j[ok]).tolist(), img[ok].tolist()))
            cnt = self.cnt.numpy()
            for pair in pairs:
                if pair in self.dset:
                    continue
                if len(self.dset) >= self.dcap:
                    self.overflow = True
                    continue
                self.dset[pair] = None
                cnt[pair[0]] += 1

        def emit_distinct(self, ngroups, capacity):
            g = self._rows(False)
            assert len(g) == ngroups
            key_of = (lambda gid: gid + self.kbase) if self.kbase is not None else (lambda gid: self.keys[gid])
            rows = [(int(key_of(x)), -1, 0) for x in g] + [(int(key_of(e // self.vs)), e % self.vs, i) for e, i in self.dset]
            n = len(rows)
            out = np.zeros((max(capacity, 0), 3), dtype=np.int64)
            if rows:
                out[: min(n, capacity)] = np.array(rows[:capacity], dtype=np.int64)
            count = cpu_double.torch.tensor([n, int(self.overflow or n > capacity)], dtype=cpu_double.torch.int64)
            return (cpu_double._col(out[:, 0]), cpu_double._col(out[:, 1]), cpu_double._col(out[:, 2]), count)

    with cpu_double.installed():
        ops.GroupTable = NuniqueTable
        yield NuniqueTable


@pytest.fixture
def dev():
    old = config.NPartitions.get()
    with double_installed():
        yield
    config.NPartitions.put(old)


@contextlib.contextmanager
def distinct_budget(nbytes):
    old = config.GroupbyDistinctBytes.get()
    config.GroupbyDistinctBytes.put(nbytes)
    try:
        yield
    finally:
        config.GroupbyDistinctBytes.put(old)


def _frame(n=120, seed=5, groups=7):
    """Keys 0..groups-1 plus a one-row group (key 50).  ``f``: few values with NaN, group 3 all NaN; ``z``: +-0.0, NaN
    payloads and +-inf; ``c``: constant; ``i``: int64 with the extremes, 0 and -1 (the images of the empty slot);
    ``b``: bool; ``u``: all distinct."""
    rng = np.random.default_rng(seed)
    key = np.tile(np.arange(groups), n // groups + 1)[:n]
    rng.shuffle(key)
    key[-1] = 50
    f = rng.integers(0, 4, n) * 0.5
    f[rng.random(n) < 0.25] = np.nan
    f[key == 3] = np.nan
    payloads = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0x7FF8DEADBEEF0001],
                        dtype=np.uint64).view(np.float64)  # fmt: skip
    z = rng.choice(np.concatenate([[0.0, -0.0, np.inf, -np.inf, 1.0], payloads]), n)
    i = rng.choice(np.array([I64_MIN, I64_MAX, 0, -1, 7], dtype=np.int64), n)
    return pandas.DataFrame({"key": key.astype(np.int64), "f": f, "z": z, "c": np.full(n, 0.1), "i": i,
                             "b": rng.random(n) < 0.5, "u": rng.standard_normal(n)})  # fmt: skip


def _same(got, want):
    if isinstance(want, pandas.Series):
        pandas.testing.assert_series_equal(got, want, check_index_type=False)
        return
    pandas.testing.assert_index_equal(got.index, want.index, exact=False)
    assert got.index.name == want.index.name and list(got.index.names) == list(want.index.names)
    assert list(got.columns) == list(want.columns), (list(got.columns), list(want.columns))
    assert list(got.dtypes) == list(want.dtypes), (list(got.dtypes), list(want.dtypes))
    for j in range(want.shape[1]):
        a, b = got.iloc[:, j].to_numpy(), want.iloc[:, j].to_numpy()
        if a.dtype.kind == "f":  # the sums / means of a mixed dictionary; every count is compared exactly
            np.testing.assert_allclose(a, b, rtol=1e-12)
        else:
            assert np.array_equal(a, b), (j, a, b)


def _cases(mk, pdf):
    df = mk(pdf)
    for dropna in (True, False):
        _same(df.groupby("key").nunique(dropna=dropna)._to_pandas(), pdf.groupby("key").nunique(dropna=dropna))
        _same(df.groupby("key", as_index=False).nunique(dropna=dropna)._to_pandas(),
              pdf.groupby("key", as_index=False).nunique(dropna=dropna))  # fmt: skip
    _same(df.groupby("key").agg("nunique")._to_pandas(), pdf.groupby("key").agg("nunique"))
    _same(df.groupby("key").nunique()._to_pandas(), pdf.groupby("key").nunique())
    spec = {"f": "nunique", "c": "sum", "z": "nunique", "u": "mean", "i": "nunique"}
    _same(df.groupby("key").agg(spec)._to_pandas(), pdf.groupby("key").agg(spec))


# ------------------------------------------------------------------ the Modin-free mirror (modin_b200.pandas)
@pytest.mark.parametrize("nparts", [1, 2, 3, 4])
def test_mirror_nunique_matches_pandas(dev, nparts):
    import modin_b200.pandas as bpd

    config.NPartitions.put(nparts)
    pdf = _frame()
    _cases(bpd.DataFrame, pdf)
    two = pdf.assign(k2=(np.arange(len(pdf)) % 3).astype(np.int64))
    for dropna in (True, False):
        _same(bpd.DataFrame(two).groupby(["key", "k2"]).nunique(dropna=dropna)._to_pandas(),
              two.groupby(["key", "k2"]).nunique(dropna=dropna))  # fmt: skip
    # one-column frames of each dtype
    for col in ("f", "z", "i", "b"):
        one = pdf[["key", col]]
        _same(bpd.DataFrame(one).groupby("key").nunique()._to_pandas(), one.groupby("key").nunique())


@pytest.mark.parametrize("dense", [True, False])
def test_mirror_dense_and_hashed_tables_forty_columns_and_one_column_batches(dev, dense):
    """40 value columns run in two batches of at most 32; a budget below one column's set runs one column per batch;
    both give the columns back in order."""
    import modin_b200.pandas as bpd

    old = config.GroupbyDenseKeys.get()
    config.GroupbyDenseKeys.put(dense)
    try:
        config.NPartitions.put(3)
        pdf = _frame(131, seed=2, groups=11)
        kinds = ["f", "z", "c", "i", "b", "u"]
        wide = pandas.DataFrame({"key": pdf["key"], **{f"c{j}": np.roll(pdf[kinds[j % 6]].to_numpy(), 7 * j)
                                                       for j in range(40)}})  # fmt: skip
        assert functors.distinct_batches(131, 40) == [(0, 32), (32, 40)]
        for dropna in (True, False):
            _same(bpd.DataFrame(wide).groupby("key").nunique(dropna=dropna)._to_pandas(),
                  wide.groupby("key").nunique(dropna=dropna))  # fmt: skip
        with distinct_budget(16):
            assert functors.distinct_batches(131, 5) == [(j, j + 1) for j in range(5)]
            _same(bpd.DataFrame(pdf).groupby("key").nunique()._to_pandas(), pdf.groupby("key").nunique())
    finally:
        config.GroupbyDenseKeys.put(old)


def test_batches_follow_the_budget():
    """``next_pow2(2 * rows * width) * 16`` bytes per batch; one column even above the budget; at most 32 columns."""
    with distinct_budget(8 << 30):
        assert functors.distinct_batches(1 << 26, 8) == [(0, 4), (4, 8)]  # 2^29 slots = 8 GiB per 4 columns
        assert functors.distinct_batches(5 * 10**8, 2) == [(0, 1), (1, 2)]  # one 16 GiB set per column
        assert functors.distinct_batches(10, 70) == [(0, 32), (32, 64), (64, 70)]
        assert functors.distinct_batches(0, 3) == [(0, 3)]
        assert functors.distinct_batches(10, 0) == []


def test_mirror_edge_groups_empty_frame_and_refusals(dev):
    import modin_b200.pandas as bpd

    # all-NaN, one-row and constant groups; every NaN payload is one value and +-0.0 one value
    key = np.array([0, 0, 0, 1, 2, 2, 2, 2, 3, 3], dtype=np.int64)
    nan2 = np.array([0xFFF8000000000000], dtype=np.uint64).view(np.float64)[0]
    x = np.array([np.nan, nan2, np.nan, 5.0, 0.0, -0.0, np.inf, -np.inf, 2.0, 2.0])
    pdf = pandas.DataFrame({"key": key, "x": x, "n": np.full(10, np.nan)})
    for dropna in (True, False):
        want = pdf.groupby("key").nunique(dropna=dropna)
        assert want["x"].tolist() == ([0, 1, 3, 1] if dropna else [1, 1, 3, 1])
        for nparts in (1, 3):
            config.NPartitions.put(nparts)
            _same(bpd.DataFrame(pdf).groupby("key").nunique(dropna=dropna)._to_pandas(), want)
    empty = _frame().iloc[:0]
    got = bpd.DataFrame(empty).groupby("key").nunique()._to_pandas()
    want = empty.groupby("key").nunique()
    assert list(got.columns) == list(want.columns) and len(got) == 0
    assert list(got.dtypes) == list(want.dtypes) == [np.dtype(np.int64)] * 6
    keys_only = pdf[["key"]]
    _same(bpd.DataFrame(keys_only).groupby("key").nunique()._to_pandas(), keys_only.groupby("key").nunique())
    df = bpd.DataFrame(pdf)
    g = df.groupby("key")
    with pytest.raises(NotImplementedError, match="extra"):
        g._wrap_aggregation(type(df._query_compiler).groupby_nunique, agg_kwargs=dict(dropna=True, extra=1))
    with pytest.raises(ValueError, match="dropna"):
        g.nunique(dropna="no")


def test_nunique_table_stand_in(dev):
    """Pass 1 inserts the groups only; pass 2 counts each (group, column, image) once, from raw rows and from partial
    rows; pass 1 is refused after pass 2; a full set raises the overflow flag; flags other than SIZE | NUNIQUE are
    refused."""
    from tests import cpu_double

    keys = cpu_double._col(np.array([5, 7, 5, 5, 7, 9], dtype=np.int64))
    f = cpu_double._col(np.array([1.0, np.nan, -0.0, 0.0, np.nan, 4.0]))
    i = cpu_double._col(np.array([I64_MIN, -1, I64_MIN, 0, 0, -1], dtype=np.int64))
    for dense in (False, True):
        t = ops.GroupTable.dense(5, 9, 2, NUNIQUE) if dense else ops.GroupTable(16, 2, NUNIQUE)
        t.accumulate(keys, [])
        t.reserve_distinct(32)
        t.accumulate_distinct(keys, [f, i], dropna=True)
        k, s, c, z = ops.emit_counted(t)
        assert k.data.numpy().tolist() == [5, 7, 9] and s is None and z.data.numpy().tolist() == [3, 2, 1]
        assert c[0].data.numpy().tolist() == [2, 0, 1] and c[1].data.numpy().tolist() == [2, 2, 1]
        with pytest.raises(_lib.B200Error):
            t.accumulate(keys, [])
        ek, ec, ei, count = t.emit_distinct(3, 3 + 12)
        n, ov = count.tolist()
        assert n == 3 + 8 and not ov
        # the partial rows of that emit, twice over, rebuild the same counts in a fresh table
        rk, rc, ri = (cpu_double._col(np.tile(x.data.numpy()[:n], 2)) for x in (ek, ec, ei))
        t2 = ops.GroupTable(16, 2, NUNIQUE)
        t2.accumulate(rk, [])
        t2.reserve_distinct(64)
        t2.accumulate_distinct(rk, col_ids=rc, images=ri)
        k2, _, c2, _ = ops.emit_counted(t2)
        assert k2.data.numpy().tolist() == [5, 7, 9]
        assert [x.data.numpy().tolist() for x in c2] == [[2, 0, 1], [2, 2, 1]]
        # dropna=False counts NaN once; a set of 2 slots overflows
        t3 = ops.GroupTable(16, 1, NUNIQUE)
        t3.accumulate(keys, [])
        t3.reserve_distinct(8)
        t3.accumulate_distinct(keys, [f], dropna=False)
        assert ops.emit_counted(t3)[2][0].data.numpy().tolist() == [2, 1, 1]
        t4 = ops.GroupTable(16, 1, NUNIQUE)
        t4.accumulate(keys, [])
        t4.reserve_distinct(2)
        t4.accumulate_distinct(keys, [f])
        assert t4.ngroups()[1]
    with pytest.raises(_lib.B200Error, match="full"):
        functors._distinct_filled(t4, 0, [])
    for bad in (_lib.GB_NUNIQUE, _lib.GB_COUNT | _lib.GB_NUNIQUE, NUNIQUE | _lib.GB_SUM):
        with pytest.raises(_lib.B200Error):
            ops.GroupTable(16, 1, bad)


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
def test_plugin_nunique_matches_pandas(mpd, dev, nparts):
    import modin.config as cfg

    cfg.NPartitions.put(nparts)
    config.NPartitions.put(nparts)
    pdf = _frame()
    _cases(mpd.DataFrame, pdf)
    two = pdf.assign(k2=(np.arange(len(pdf)) % 3).astype(np.int64))
    lab = pdf.drop(columns="key").set_axis(pandas.Index(pdf["key"].to_numpy(), name="lab"))
    fk = pdf.assign(key=np.where(pdf["key"] == 2, np.nan, pdf["key"] * 0.5 - 1.0))
    _same(mpd.DataFrame(two).groupby(["key", "k2"]).nunique()._to_pandas(), two.groupby(["key", "k2"]).nunique())
    _same(mpd.DataFrame(lab).groupby(level=0).nunique()._to_pandas(), lab.groupby(level=0).nunique())
    for dropna in (True, False):
        _same(mpd.DataFrame(fk).groupby("key", dropna=dropna).nunique()._to_pandas(),
              fk.groupby("key", dropna=dropna).nunique())  # fmt: skip
        got = mpd.DataFrame(pdf).groupby("key")["z"].nunique(dropna=dropna)._to_pandas()
        _same(got, pdf.groupby("key")["z"].nunique(dropna=dropna))


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
    """``full``: 14 rows per rank, every group on every rank, group 3's ``f`` NaN on every rank; ``tiny``: fewer rows
    than ranks, so the last rank has none."""
    n = 14 * ws
    r = np.arange(n)
    key = (r % 4).astype(np.int64)
    f = np.where(key == 3, np.nan, np.where(r % 5 == 0, -0.0, np.round(np.sin(r), 1)))
    full = pandas.DataFrame({"key": key, "f": f, "i": (r * 3 - 20) % 7, "b": r % 3 == 1})
    return {"full": full, "tiny": full.iloc[: ws - 1]}


def _rank_job(rank, ws):
    import modin_b200.pandas as bpd

    out = {}
    with double_installed():
        config.NPartitions.put(2)
        for dense in (True, False):
            config.GroupbyDenseKeys.put(dense)
            frames = _rank_frames(ws)
            for name in ("full", "tiny"):
                df = bpd.DataFrame(frames[name])
                for dropna in (True, False):
                    out[(dense, name, dropna)] = df.groupby("key").nunique(dropna=dropna)._to_pandas()
            with distinct_budget(16):  # one column per batch: one exchange still serves them all
                out[(dense, "batched", True)] = bpd.DataFrame(frames["full"]).groupby("key").nunique()._to_pandas()
            try:
                bpd.DataFrame(frames["full"]).groupby("key").agg({"f": "nunique", "i": "count"})
                out[(dense, "mixed", True)] = "no error"
            except NotImplementedError as e:
                out[(dense, "mixed", True)] = str(e)
    return out


@pytest.mark.parametrize("ws", [2, 3])
def test_ranks_count_distinct_across_ranks(ws):
    import torch.multiprocessing as mp

    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(ws, _free_port(), ret), nprocs=ws, join=True)
    frames = _rank_frames(ws)
    for r in range(ws):  # every rank holds the whole answer and refuses the same dictionaries
        assert len(ret[r]) == 2 * 6
        for (dense, name, dropna), got in ret[r].items():
            if name == "mixed":
                assert "across ranks" in got, got
            else:
                frame = frames["full" if name == "batched" else name]
                _same(got, frame.groupby("key").nunique(dropna=dropna))
