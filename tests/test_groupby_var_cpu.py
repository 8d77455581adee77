"""``groupby.var`` / ``std`` through both front doors, with the device replaced by the numpy test double: the functors
(one VAR table per partition filled in two passes, the pairwise merge of partial sums / counts / M2s, the division by
``count - ddof`` on the device), the shared groupby caller (keys of every kind, ``as_index=False``, ``agg`` and
dictionaries, refusals) and the key-range exchange under 2 and 3 gloo ranks.  Results are compared with pandas for
values, index and dtypes.  ``VarTable`` below is the numpy twin of a VAR group table (csrc/groupby.cu): pass 1 is the
SUM | COUNT table, pass 2 adds squared deviations from ``acc / cnt`` into ``m2`` from raw rows or from partial rows,
pass 1 is refused after pass 2, and emit writes the sums, then the M2s."""

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
VAR = _lib.GB_SUM | _lib.GB_COUNT | _lib.GB_VAR
DDOFS = (0, 1, 2, 1.5, -1, -0.5)  # pandas 3.0.2 truncates a float ddof towards zero


@contextlib.contextmanager
def double_installed():
    sys.path.insert(0, HERE)
    import cpu_double

    class VarTable(cpu_double.GroupTable):
        """The double's group table, playing VAR tables as well."""

        def _setup(self, kbase, capacity, nvals, flags, arrays, kind):
            if flags & _lib.GB_VAR and flags != VAR:
                raise _lib.B200Error("mb200_gb_create: a VAR table is SUM | COUNT | VAR")
            super()._setup(kbase, capacity, nvals, flags, arrays, kind)
            self.m2 = np.zeros(self.capacity * self.vs) if flags & _lib.GB_VAR else None
            self.m2_filled = False

        def _pass1(self):
            if self.m2_filled:
                raise _lib.B200Error("a VAR table takes no rows after mb200_gb_accumulate_m2")

        def accumulate(self, keys, vals):
            self._pass1()
            return super().accumulate(keys, vals)

        def merge_partial(self, keys, sums, cnts=None, sizes=None):
            self._pass1()
            return super().merge_partial(keys, sums, cnts, sizes)

        def accumulate_m2(self, keys, vals, cnts=None, m2s=None):
            if self.m2 is None:
                raise _lib.B200Error("mb200_gb_accumulate_m2: not a VAR table")
            self.m2_filled = True
            k = cpu_double._np(keys)
            if self.kbase is not None:
                g = k - self.kbase
                live = (g >= 0) & (g < self.capacity)
            else:  # read-only lookup: pass 2 adds no group
                order = np.argsort(self.keys, kind="stable")
                pos = np.minimum(np.searchsorted(self.keys[order], k), max(len(order) - 1, 0))
                live = self.keys[order][pos] == k if len(order) else np.zeros(len(k), dtype=bool)
                g = order[pos] if len(order) else np.zeros(len(k), dtype=np.int64)
            acc, cnt = self.acc.numpy(), self.cnt.numpy()
            for v, col in enumerate(vals):
                x = cpu_double._np(col)
                ok = live & (cpu_double._np(cnts[v]) != 0 if cnts is not None else ~np.isnan(x))
                o = np.where(ok, g * self.vs + v, 0)
                ok &= cnt[o] > 0
                with np.errstate(all="ignore"):
                    mean = acc[o] / cnt[o]
                    if cnts is None:
                        term = (x - mean) ** 2
                    else:
                        n_p = cpu_double._np(cnts[v]).astype(np.float64)
                        term = cpu_double._np(m2s[v]) + n_p * (x / n_p - mean) ** 2
                np.add.at(self.m2, o[ok], term[ok])

        def _emit(self, g):
            keys, sums, cnts, sizes = super()._emit(g)
            if self.m2 is not None:
                m = self.m2.reshape(self.capacity, self.vs)[g]
                sums = sums + [cpu_double._col(np.ascontiguousarray(m[:, v])) for v in range(self.nvals)]
            return keys, sums, cnts, sizes

    with cpu_double.installed():
        ops.GroupTable = VarTable
        yield VarTable


@pytest.fixture
def dev():
    old = config.NPartitions.get()
    with double_installed():
        yield
    config.NPartitions.put(old)


def _frame(n=90, seed=5, groups=7):
    """Keys 0..groups-1 plus a one-row group (key 50); ``f``: NaN, with group 3 all NaN; ``c``: a constant group value
    (0.1); ``big``: values around 1e9 with unit spread; ``i``: int64; ``b``: bool."""
    rng = np.random.default_rng(seed)
    key = np.tile(np.arange(groups), n // groups + 1)[:n]
    rng.shuffle(key)
    key[-1] = 50
    f = np.round(rng.standard_normal(n), 2)
    f[rng.random(n) < 0.25] = np.nan
    f[key == 3] = np.nan
    return pandas.DataFrame({"key": key.astype(np.int64), "f": f, "c": np.full(n, 0.1),
                             "big": 1e9 + rng.integers(-3, 4, n).astype(np.float64),
                             "i": rng.integers(-1000, 1000, n).astype(np.int64), "b": rng.random(n) < 0.5})  # fmt: skip


def _same(got, want):
    pandas.testing.assert_index_equal(got.index, want.index, exact=False)
    assert got.index.name == want.index.name and list(got.index.names) == list(want.index.names)
    assert list(got.columns) == list(want.columns), (list(got.columns), list(want.columns))
    assert list(got.dtypes) == list(want.dtypes), (list(got.dtypes), list(want.dtypes))
    for j in range(want.shape[1]):
        a, b = got.iloc[:, j].to_numpy(), want.iloc[:, j].to_numpy()
        if a.dtype.kind == "f":
            assert np.array_equal(np.isnan(a), np.isnan(b)), (j, a, b)
            # pandas' Welford loop loses ~n u max|x| on the mean-1e9 column, which the two-pass result does not: a
            # relative 1e-7 tells a right answer from a wrong one; the exact bound is checked on the GPU
            np.testing.assert_allclose(a[~np.isnan(a)], b[~np.isnan(b)], rtol=1e-7, atol=1e-12)
        else:
            assert np.array_equal(a, b), (j, a, b)


def _cases(mk, pdf):
    df = mk(pdf)
    for fn in ("var", "std"):
        _same(getattr(df.groupby("key"), fn)()._to_pandas(), getattr(pdf.groupby("key"), fn)())
        for ddof in DDOFS:
            _same(getattr(df.groupby("key"), fn)(ddof=ddof)._to_pandas(), getattr(pdf.groupby("key"), fn)(ddof=ddof))
        _same(df.groupby("key").agg(fn)._to_pandas(), pdf.groupby("key").agg(fn))
        _same(df.groupby("key").agg(fn, ddof=2)._to_pandas(), pdf.groupby("key").agg(fn, ddof=2))
        _same(getattr(df.groupby("key", as_index=False), fn)()._to_pandas(), getattr(pdf.groupby("key", as_index=False), fn)())
    spec = {"f": "var", "c": "sum", "big": "std", "i": "mean", "b": "var"}
    _same(df.groupby("key").agg(spec)._to_pandas(), pdf.groupby("key").agg(spec))


# ------------------------------------------------------------------ the Modin-free mirror (modin_b200.pandas)
@pytest.mark.parametrize("nparts", [1, 2, 3, 4])
def test_mirror_var_std_match_pandas(dev, nparts):
    import modin_b200.pandas as bpd

    config.NPartitions.put(nparts)
    pdf = _frame()
    _cases(bpd.DataFrame, pdf)
    two = pdf.assign(k2=(np.arange(len(pdf)) % 3).astype(np.int64))
    for fn in ("var", "std"):
        _same(getattr(bpd.DataFrame(two).groupby(["key", "k2"]), fn)()._to_pandas(), getattr(two.groupby(["key", "k2"]), fn)())


@pytest.mark.parametrize("dense", [True, False])
def test_mirror_dense_and_hashed_tables_and_forty_columns(dev, dense):
    """40 value columns: two VAR tables per partition whose sums-then-M2s layouts are joined in column order, in the
    map and in the reduce over 3 row partitions."""
    import modin_b200.pandas as bpd

    old = config.GroupbyDenseKeys.get()
    config.GroupbyDenseKeys.put(dense)
    try:
        config.NPartitions.put(3)
        pdf = _frame(131, seed=2, groups=11)
        kinds = ["f", "c", "big", "i", "b"]
        wide = pandas.DataFrame({"key": pdf["key"], **{f"c{j}": np.roll(pdf[kinds[j % 5]].to_numpy(), 7 * j) * (j + 1)
                                                       for j in range(40)}})  # fmt: skip
        for fn in ("var", "std"):
            _same(getattr(bpd.DataFrame(pdf).groupby("key"), fn)()._to_pandas(), getattr(pdf.groupby("key"), fn)())
            for ddof in (0, 1.5):
                _same(getattr(bpd.DataFrame(wide).groupby("key"), fn)(ddof=ddof)._to_pandas(),
                      getattr(wide.groupby("key"), fn)(ddof=ddof))  # fmt: skip
    finally:
        config.GroupbyDenseKeys.put(old)


def test_mirror_empty_frame_all_nan_and_refusals(dev):
    import modin_b200.pandas as bpd

    pdf = _frame()
    empty = pdf.iloc[:0]
    for fn in ("var", "std"):
        got = getattr(bpd.DataFrame(empty).groupby("key"), fn)()._to_pandas()
        want = getattr(empty.groupby("key"), fn)()
        assert list(got.columns) == list(want.columns) and len(got) == 0
        assert list(got.dtypes) == list(want.dtypes) == [np.dtype(np.float64)] * 5
    # an all-NaN group with ddof=-1 gives 0.0, as in pandas; with ddof >= 0 NaN
    nan = pdf.assign(f=np.where(pdf["key"] == 2, np.nan, pdf["f"]))
    assert pandas.isna(nan.groupby("key")["f"].var().loc[2])
    assert nan.groupby("key")["f"].var(ddof=-1).loc[2] == 0.0
    for ddof in DDOFS:
        _same(bpd.DataFrame(nan).groupby("key").var(ddof=ddof)._to_pandas(), nan.groupby("key").var(ddof=ddof))
    df = bpd.DataFrame(pdf)
    for fn in ("var", "std"):
        with pytest.raises(NotImplementedError, match="engine"):
            getattr(df.groupby("key"), fn)(engine="numba")
        g = df.groupby("key")
        with pytest.raises(NotImplementedError, match="min_count"):
            g._wrap_aggregation(getattr(type(df._query_compiler), f"groupby_{fn}"), agg_kwargs=dict(ddof=1, min_count=2))
        with pytest.raises(NotImplementedError, match="engine"):
            g._wrap_aggregation(getattr(type(df._query_compiler), f"groupby_{fn}"), agg_kwargs=dict(engine="numba"))


def test_special_values_and_constant_groups(dev):
    """Infinities give NaN, squares that overflow give inf, -0.0 is a zero; a constant 0.1 group is within the bound
    of 0.0 (pandas gives exactly 0.0)."""
    import modin_b200.pandas as bpd

    key = np.array([0, 0, 0, 1, 1, 2, 2, 3, 3, 3], dtype=np.int64)
    x = np.array([2.0, 3.0, np.inf, 1e300, -1e300, -0.0, 0.0, 0.1, 0.1, 0.1])
    pdf = pandas.DataFrame({"key": key, "x": x})
    want = pdf.groupby("key").var()
    assert np.isnan(want.loc[0, "x"]) and want.loc[1, "x"] == np.inf and want.loc[2, "x"] == 0.0
    assert want.loc[3, "x"] == 0.0
    for nparts in (1, 3):
        config.NPartitions.put(nparts)
        got = bpd.DataFrame(pdf).groupby("key").var()._to_pandas()
        assert np.isnan(got.loc[0, "x"]) and got.loc[1, "x"] == np.inf and got.loc[2, "x"] == 0.0
        u = 2.0**-53
        assert abs(got.loc[3, "x"]) <= (3 * 3 + 8) * u * 5 * 3 * ((3 + 2) * u * 0.1) ** 2 + 5 * 3 * ((3 + 2) * u * 0.1) ** 2


def test_var_table_stand_in(dev):
    """Pass 1 into sums / counts; pass 2 from raw rows and from partial rows; pass 1 refused after pass 2; the emit
    writes the sums, then the M2s; flags other than SUM | COUNT | VAR are refused."""
    from tests import cpu_double

    keys = cpu_double._col(np.array([5, 7, 5, 5, 7, 9], dtype=np.int64))
    f = cpu_double._col(np.array([1.0, np.nan, 2.0, 6.0, np.nan, 4.0]))
    for dense in (False, True):
        t = ops.GroupTable.dense(5, 9, 1, VAR) if dense else ops.GroupTable(16, 1, VAR)
        ops.fill_table(t, [(keys, [f])])
        k, s, c, _ = ops.emit_counted(t)
        assert k.data.numpy().tolist() == [5, 7, 9] and len(s) == 2
        assert s[0].data.numpy().tolist() == [9.0, 0.0, 4.0] and c[0].data.numpy().tolist() == [3, 0, 1]
        assert s[1].data.numpy().tolist() == [14.0, 0.0, 0.0]
        with pytest.raises(_lib.B200Error):
            t.accumulate(keys, [f])
        with pytest.raises(_lib.B200Error):
            t.merge_partial(k, s[:1], c)
        # the partials of two tables merge pairwise: {1, 2} and {6} -> M2 of {1, 2, 6}
        a = ops.hash_aggregate([(cpu_double._col(np.array([5, 5], dtype=np.int64)), [cpu_double._col(np.array([1.0, 2.0]))])], VAR, 16)
        b = ops.hash_aggregate([(cpu_double._col(np.array([5], dtype=np.int64)), [cpu_double._col(np.array([6.0]))])], VAR, 16)
        pk = cpu_double._col(np.concatenate([a[0].data.numpy(), b[0].data.numpy()]))
        cat = lambda j: cpu_double._col(np.concatenate([a[j][0].data.numpy(), b[j][0].data.numpy()]))  # noqa: E731
        m2 = cpu_double._col(np.concatenate([a[1][1].data.numpy(), b[1][1].data.numpy()]))
        k2, s2, c2, _ = ops.hash_aggregate([(pk, [cat(1), m2], [cat(2)], None)], VAR, 16, partial=True)
        assert k2.data.numpy().tolist() == [5] and s2[0].data.numpy().tolist() == [9.0] and c2[0].data.numpy().tolist() == [3]
        assert s2[1].data.numpy().tolist() == [14.0]
    for bad in (_lib.GB_VAR, _lib.GB_SUM | _lib.GB_VAR, VAR | _lib.GB_SIZE, _lib.GB_COUNT | _lib.GB_VAR):
        with pytest.raises(_lib.B200Error):
            ops.GroupTable(16, 1, bad)


def test_split_above_max_cols_keeps_the_sums_then_m2_layout(dev):
    """``hash_aggregate`` over 40 value columns runs two tables and joins their emits as 40 sums, then 40 M2s, in raw
    and in partial form."""
    from tests import cpu_double

    rng = np.random.default_rng(3)
    k = cpu_double._col(rng.integers(0, 5, 200).astype(np.int64))
    xs = [rng.standard_normal(200) + j for j in range(40)]
    keys, sums, cnts, _ = ops.hash_aggregate([(k, [cpu_double._col(x) for x in xs])], VAR, 16)
    assert len(sums) == 80 and len(cnts) == 40
    kk = k.data.numpy()
    for j, x in enumerate(xs):
        for r, g in enumerate(keys.data.numpy()):
            sel = x[kk == g]
            assert sums[j].data.numpy()[r] == pytest.approx(sel.sum(), rel=1e-12)
            assert sums[40 + j].data.numpy()[r] == pytest.approx(((sel - sel.mean()) ** 2).sum(), rel=1e-9)
    k2, s2, c2, _ = ops.hash_aggregate([(keys, sums, cnts, None)], VAR, 16, partial=True)
    assert len(s2) == 80
    for j in range(80):
        np.testing.assert_allclose(s2[j].data.numpy(), sums[j].data.numpy(), rtol=1e-12)


def test_int64_groupby_sum_and_min_stay_refused(dev):
    import modin_b200.pandas as bpd
    from tests import shape_cases

    _, refused = shape_cases.int64_bool_and_mixed(bpd)
    for call in refused[1:]:
        with pytest.raises(NotImplementedError):
            call()


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
def test_plugin_var_std_match_pandas(mpd, dev, nparts):
    import modin.config as cfg

    cfg.NPartitions.put(nparts)
    config.NPartitions.put(nparts)
    pdf = _frame()
    _cases(mpd.DataFrame, pdf)
    two = pdf.assign(k2=(np.arange(len(pdf)) % 3).astype(np.int64))
    lab = pdf.drop(columns="key").set_axis(pandas.Index(pdf["key"].to_numpy(), name="lab"))
    fk = pdf.assign(key=np.where(pdf["key"] == 2, np.nan, pdf["key"] * 0.5 - 1.0))
    for fn in ("var", "std"):
        _same(getattr(mpd.DataFrame(two).groupby(["key", "k2"]), fn)()._to_pandas(), getattr(two.groupby(["key", "k2"]), fn)())
        _same(getattr(mpd.DataFrame(lab).groupby(level=0), fn)()._to_pandas(), getattr(lab.groupby(level=0), fn)())
        for dropna in (True, False):
            _same(getattr(mpd.DataFrame(fk).groupby("key", dropna=dropna), fn)(ddof=0)._to_pandas(),
                  getattr(fk.groupby("key", dropna=dropna), fn)(ddof=0))  # fmt: skip
        got = getattr(mpd.DataFrame(pdf).groupby("key")["f"], fn)()._to_pandas()
        pandas.testing.assert_series_equal(got, getattr(pdf.groupby("key")["f"], fn)(), rtol=1e-9)
        _same(mpd.DataFrame(pdf).groupby("key").agg({"f": fn, "c": "sum"})._to_pandas(),
              pdf.groupby("key").agg({"f": fn, "c": "sum"}))  # fmt: skip


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
    """``full``: 14 rows per rank, every group on every rank; ``tiny``: fewer rows than ranks, so the last rank has
    none."""
    n = 14 * ws
    r = np.arange(n)
    full = pandas.DataFrame({"key": (r % 4).astype(np.int64), "f": np.where(r % 5 == 0, np.nan, np.sin(r)),
                             "i": r * 3 - 20, "b": r % 3 == 1})  # fmt: skip
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
                for fn in ("var", "std"):
                    out[(dense, name, fn)] = getattr(df.groupby("key"), fn)(ddof=0)._to_pandas()
            for fn in ("var", "std"):
                try:
                    bpd.DataFrame(frames["full"]).groupby("key").agg({"f": fn, "i": "count"})
                    out[(dense, "mixed", fn)] = "no error"
                except NotImplementedError as e:
                    out[(dense, "mixed", fn)] = str(e)
    return out


@pytest.mark.parametrize("ws", [2, 3])
def test_ranks_merge_partials_across_ranks(ws):
    import torch.multiprocessing as mp

    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(ws, _free_port(), ret), nprocs=ws, join=True)
    frames = _rank_frames(ws)
    for r in range(ws):  # every rank holds the whole answer and refuses the same dictionaries
        assert len(ret[r]) == 2 * 6
        for (dense, name, fn), got in ret[r].items():
            if name == "mixed":
                assert "across ranks" in got, got
            else:
                _same(got, getattr(frames[name].groupby("key"), fn)(ddof=0))
