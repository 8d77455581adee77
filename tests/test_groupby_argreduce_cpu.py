"""``groupby.idxmax`` / ``idxmin`` through both front doors, with the device replaced by the numpy test double: the
functors (one ARGMAX / ARGMIN table per partition, one gather per column for the winning value and its row label, the
reduce over concatenated partial values), the shared groupby caller (keys of every kind, ``as_index=False``,
dictionaries, refusals, the all-NaN error) and the rank-order combine under 2 and 3 gloo ranks.  Results are compared
with pandas for values, index and dtypes.  ``ArgTable`` below is the numpy twin of an ARGMAX / ARGMIN group table
(csrc/groupby.cu): extreme images with -0.0 folded into +0.0, the smallest position among the rows holding the
extreme, one fill per table, and -1 for a group without a value on emit."""

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
ARG = _lib.GB_ARGMIN | _lib.GB_ARGMAX
ALL_NA = "with skipna=True encountered all NA values in a group"


def arg_image(x: np.ndarray) -> np.ndarray:
    """Order-preserving int64 image of float64 values, -0.0 folded into +0.0 (NaN: not defined); int64 as is."""
    if x.dtype == np.int64:
        return x.copy()
    b = np.where(x == 0.0, 0.0, x).view(np.int64)
    return b ^ ((b >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))


@contextlib.contextmanager
def double_installed():
    sys.path.insert(0, HERE)
    import cpu_double

    class ArgTable(cpu_double.GroupTable):
        """The double's group table, playing ARGMIN / ARGMAX tables as well."""

        def _setup(self, kbase, capacity, nvals, flags, arrays, kind):
            super()._setup(kbase, capacity, nvals, flags, arrays, kind)
            self.filled = False
            if flags & ARG:
                self.acc, self.cnt = arrays["acc"], arrays["cnt"]
                self.acc.fill_(I64_MAX)
                self.cnt.fill_(I64_MIN if flags & _lib.GB_ARGMAX else I64_MAX)

        def accumulate(self, keys, vals):
            if not self.flags & ARG:
                return super().accumulate(keys, vals)
            if any(v is None or v.dtype not in (np.float64, np.int64) for v in vals):
                raise TypeError("device groupby.idxmax / idxmin take float64 and int64 value columns")
            if self.filled:
                raise _lib.B200Error("mb200_gb_accumulate_arg: an ARGMIN / ARGMAX table is filled by one call")
            self.filled = True
            g = self._gids(keys)
            live = g < self.capacity
            if self.present is not None:
                self.present.numpy()[g[live]] = 1
            pos = np.arange(len(g), dtype=np.int64)
            for v, col in enumerate(vals):
                x = col.data.numpy()
                ok = live & (~np.isnan(x) if x.dtype == np.float64 else True)
                img = arg_image(x[ok])
                o = g[ok] * self.vs + v
                (np.maximum.at if self.flags & _lib.GB_ARGMAX else np.minimum.at)(self.cnt.numpy(), o, img)
                win = img == self.cnt.numpy()[o]  # pass 2: rows holding the final extreme
                np.minimum.at(self.acc.numpy(), o[win], pos[ok][win])

        def merge_partial(self, keys, sums, cnts=None, sizes=None):
            if self.flags & ARG:
                raise _lib.B200Error("mb200_gb_merge_partial: ARGMIN / ARGMAX tables do not merge partial tables")
            return super().merge_partial(keys, sums, cnts, sizes)

        def _emit(self, g):
            if not self.flags & ARG:
                return super()._emit(g)
            acc, cnt, self.acc, self.cnt = self.acc, self.cnt, None, None
            try:
                keys, _, _, sizes = super()._emit(g)
            finally:
                self.acc, self.cnt = acc, cnt
            a = acc.numpy().reshape(self.capacity, self.vs)[g]
            a = np.where(a == I64_MAX, -1, a)
            return keys, [cpu_double._col(np.ascontiguousarray(a[:, v])) for v in range(self.nvals)], None, sizes

    with cpu_double.installed():
        ops.GroupTable = ArgTable
        yield ArgTable


@pytest.fixture
def dev():
    old = config.NPartitions.get()
    with double_installed():
        yield
    config.NPartitions.put(old)


def _frame(n=48, seed=5, groups=6):
    """Keys 0..groups-1; every group has a value in every column.  ``f``: NaN, repeated extremes; ``z``: signed zeros
    only (the earlier zero wins, whatever its sign); ``inf``: -inf / NaN / +inf; ``i``: int64 limits; ``b``: bool."""
    rng = np.random.default_rng(seed)
    key = np.tile(np.arange(groups), n // groups + 1)[:n]
    rng.shuffle(key)
    f = np.round(rng.standard_normal(n), 1)
    f[rng.random(n) < 0.3] = np.nan
    z = np.where(rng.random(n) < 0.5, -0.0, 0.0)
    inf = np.where(np.arange(n) % 3 == 0, np.inf, np.where(np.arange(n) % 3 == 1, -np.inf, np.nan))
    lim = np.where(np.arange(n) % 4 == 0, I64_MIN, np.where(np.arange(n) % 4 == 1, I64_MAX, np.arange(n)))
    for k in range(groups):  # a non-NaN value in every float column of every group
        r = np.flatnonzero(key == k)[0]
        f[r] = 0.5 if np.isnan(f[r]) else f[r]
        inf[r] = -np.inf if np.isnan(inf[r]) else inf[r]
    return pandas.DataFrame({"key": key.astype(np.int64), "f": f, "z": z, "inf": inf, "i": lim.astype(np.int64),
                             "b": rng.random(n) < 0.5})  # fmt: skip


def _same(got, want):
    pandas.testing.assert_index_equal(got.index, want.index, exact=False)
    assert got.index.name == want.index.name and list(got.index.names) == list(want.index.names)
    assert list(got.columns) == list(want.columns), (list(got.columns), list(want.columns))
    assert list(got.dtypes) == list(want.dtypes), (list(got.dtypes), list(want.dtypes))
    for j in range(want.shape[1]):
        a, b = got.iloc[:, j].to_numpy(), want.iloc[:, j].to_numpy()
        assert np.array_equal(a, b, equal_nan=a.dtype.kind == "f"), (j, a, b)


def _cases(mk, pdf):
    df = mk(pdf)
    for fn in ("idxmax", "idxmin"):
        _same(getattr(df.groupby("key"), fn)()._to_pandas(), getattr(pdf.groupby("key"), fn)())
        _same(df.groupby("key").agg(fn)._to_pandas(), pdf.groupby("key").agg(fn))
        _same(getattr(df.groupby("key", as_index=False), fn)()._to_pandas(), getattr(pdf.groupby("key", as_index=False), fn)())
    spec = {"f": "idxmax", "z": "sum", "inf": "idxmin", "i": "idxmin", "b": "idxmax"}
    _same(df.groupby("key").agg(spec)._to_pandas(), pdf.groupby("key").agg(spec))


def _labelled(pdf):
    """Row-label kinds: a RangeIndex with an offset, int64 labels left by a boolean mask, float64 labels, repeated
    labels (concat), a named index."""
    mask = (np.arange(len(pdf)) % 3 != 1)
    return {
        "offset": pdf.set_axis(pandas.RangeIndex(100, 100 + len(pdf))),
        "masked": pdf[mask],
        "float": pdf.set_axis(pandas.Index(np.arange(len(pdf)) * 0.5 - 3.0)),
        "repeated": pandas.concat([pdf.iloc[: len(pdf) // 2], pdf.iloc[len(pdf) // 2 :]]).set_axis(
            np.concatenate([np.arange(len(pdf) // 2), np.arange(len(pdf) - len(pdf) // 2)])),
        "named": pdf.set_axis(pandas.Index(np.arange(len(pdf)) * 7, name="row")),
    }  # fmt: skip


# ------------------------------------------------------------------ the Modin-free mirror (modin_b200.pandas)
@pytest.mark.parametrize("nparts", [1, 3, 4])
def test_mirror_idxmax_idxmin_match_pandas(dev, nparts):
    import modin_b200.pandas as bpd

    config.NPartitions.put(nparts)
    pdf = _frame()
    _cases(bpd.DataFrame, pdf)
    for name, lab in _labelled(pdf).items():
        for fn in ("idxmax", "idxmin"):
            _same(getattr(bpd.DataFrame(lab).groupby("key"), fn)()._to_pandas(), getattr(lab.groupby("key"), fn)())
    nob = pdf.drop(columns="b").fillna(1.0)  # row selection takes frames without bool columns
    masked = bpd.DataFrame(nob)[bpd.DataFrame(pandas.DataFrame({"m": np.arange(len(pdf)) % 3 != 1}))["m"]]
    want = nob[np.arange(len(pdf)) % 3 != 1]
    for fn in ("idxmax", "idxmin"):
        _same(getattr(masked.groupby("key"), fn)()._to_pandas(), getattr(want.groupby("key"), fn)())
    two = pdf.fillna(1.0).assign(k2=(np.arange(len(pdf)) % 3).astype(np.int64))  # no all-NaN (key, k2) group
    for fn in ("idxmax", "idxmin"):
        _same(getattr(bpd.DataFrame(two).groupby(["key", "k2"]), fn)()._to_pandas(), getattr(two.groupby(["key", "k2"]), fn)())


def test_mirror_ties_across_partition_boundaries(dev):
    """Equal extremes on both sides of every row-partition boundary: the earlier row wins, however the rows are cut
    (1 or 4 row partitions), and -0.0 ties 0.0."""
    import modin_b200.pandas as bpd

    n = 40
    key = (np.arange(n) % 2).astype(np.int64)
    f = np.zeros(n)
    f[[9, 10, 11, 19, 20, 21, 29, 30]] = 5.0
    f[[12, 13]] = -3.0
    z = np.where(np.arange(n) % 4 == 0, -0.0, 0.0)
    pdf = pandas.DataFrame({"key": key, "f": f, "z": z, "i": np.where(f == 5.0, I64_MAX, I64_MIN).astype(np.int64),
                            "b": f > 0})  # fmt: skip
    for nparts in (1, 4):
        config.NPartitions.put(nparts)
        cuts = [0, 10, 20, 30, 40] if nparts == 4 else [0, 40]
        df = bpd.concat([bpd.DataFrame(pdf.iloc[a:b]) for a, b in zip(cuts, cuts[1:])])
        assert len(df._query_compiler._modin_frame._partitions) == nparts
        for fn in ("idxmax", "idxmin"):
            _same(getattr(df.groupby("key"), fn)()._to_pandas(), getattr(pdf.groupby("key"), fn)())
    assert pdf.groupby("key")["f"].idxmax().tolist() == [10, 9]
    # -0.0 before 0.0 and the reverse
    zz = pandas.DataFrame({"key": np.array([2, 2, 3, 3], dtype=np.int64), "v": [-0.0, 0.0, 0.0, -0.0]},
                          index=pandas.Index([12, 13, 14, 15]))  # fmt: skip
    for fn in ("idxmax", "idxmin"):
        got = getattr(bpd.DataFrame(zz).groupby("key"), fn)()._to_pandas()
        _same(got, getattr(zz.groupby("key"), fn)())
        assert got["v"].tolist() == [12, 14]


@pytest.mark.parametrize("dense", [True, False])
def test_mirror_dense_and_hashed_tables_and_forty_columns(dev, dense):
    import modin_b200.pandas as bpd

    old = config.GroupbyDenseKeys.get()
    config.GroupbyDenseKeys.put(dense)
    try:
        config.NPartitions.put(2)
        pdf = _frame(97, seed=2, groups=11)
        kinds = ["f", "z", "inf", "i", "b"]
        wide = pandas.DataFrame({"key": pdf["key"], **{f"c{j}": np.roll(pdf[kinds[j % 5]].to_numpy(), 11 * j) for j in range(40)}})
        for name in kinds[:3]:  # the roll may leave a group without a float value: give every group one
            for j in range(40):
                if kinds[j % 5] == name:
                    col = wide[f"c{j}"].to_numpy().copy()
                    for k in range(11):
                        r = np.flatnonzero(wide["key"].to_numpy() == k)[0]
                        col[r] = 1.25 if np.isnan(col[r]) else col[r]
                    wide[f"c{j}"] = col
        for fn in ("idxmax", "idxmin"):
            _same(getattr(bpd.DataFrame(pdf).groupby("key"), fn)()._to_pandas(), getattr(pdf.groupby("key"), fn)())
            _same(getattr(bpd.DataFrame(wide).groupby("key"), fn)()._to_pandas(), getattr(wide.groupby("key"), fn)())
    finally:
        config.GroupbyDenseKeys.put(old)


def test_mirror_all_nan_group_raises(dev):
    import modin_b200.pandas as bpd

    config.NPartitions.put(2)
    pdf = _frame()
    pdf.loc[pdf["key"] == 3, "f"] = np.nan
    for fn in ("idxmax", "idxmin"):
        with pytest.raises(ValueError, match=f"{fn} {ALL_NA}"):
            getattr(pdf.groupby("key"), fn)()
        with pytest.raises(ValueError, match=f"{fn} {ALL_NA}"):
            getattr(bpd.DataFrame(pdf).groupby("key"), fn)()
        # a column without NaN is fine
        _same(getattr(bpd.DataFrame(pdf[["key", "i", "b"]]).groupby("key"), fn)()._to_pandas(),
              getattr(pdf[["key", "i", "b"]].groupby("key"), fn)())  # fmt: skip


def test_mirror_empty_frame_and_refusals(dev):
    import modin_b200.pandas as bpd

    pdf = _frame()
    empty = pdf.iloc[:0]
    for fn in ("idxmax", "idxmin"):
        got = getattr(bpd.DataFrame(empty).groupby("key"), fn)()._to_pandas()
        want = getattr(empty.groupby("key"), fn)()
        assert list(got.columns) == list(want.columns) and len(got) == 0
        assert list(got.dtypes) == list(want.dtypes) == [np.dtype(np.int64)] * 5
    df = bpd.DataFrame(pdf)
    for fn in ("idxmax", "idxmin"):
        with pytest.raises(NotImplementedError, match="skipna=False"):
            getattr(df.groupby("key"), fn)(skipna=False)
        g = df.groupby("key")
        with pytest.raises(NotImplementedError, match="axis=1"):
            g._wrap_aggregation(getattr(type(df._query_compiler), f"groupby_{fn}"), agg_kwargs=dict(axis=1, skipna=True))
        with pytest.raises(NotImplementedError, match="str"):
            getattr(bpd.DataFrame(pdf.set_axis([f"r{j}" for j in range(len(pdf))])).groupby("key"), fn)()


def test_arg_table_stand_in(dev):
    """Images with -0.0 folded, the smallest position among ties, -1 on emit, one fill per table, no merge."""
    from tests import cpu_double

    keys = cpu_double._col(np.array([5, 7, 5, 5, 7, 9], dtype=np.int64))
    f = cpu_double._col(np.array([-0.0, np.nan, 0.0, -1.0, np.nan, np.nan]))
    i = cpu_double._col(np.array([I64_MIN, I64_MIN, 3, I64_MIN, I64_MIN, 4], dtype=np.int64))
    for flag, want_f, want_i in ((_lib.GB_ARGMAX, [0, -1, -1], [2, 1, 5]), (_lib.GB_ARGMIN, [3, -1, -1], [0, 1, 5])):
        for dense in (False, True):
            t = ops.GroupTable.dense(5, 9, 2, flag) if dense else ops.GroupTable(16, 2, flag)
            t.accumulate(keys, [f, i])
            k, s, c, _ = ops.emit_counted(t)
            assert k.data.numpy().tolist() == [5, 7, 9] and c is None
            assert s[0].data.numpy().tolist() == want_f and s[1].data.numpy().tolist() == want_i
            with pytest.raises(_lib.B200Error):
                t.accumulate(keys, [f, i])
            with pytest.raises(_lib.B200Error):
                t.merge_partial(k, s)


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
def test_plugin_idxmax_idxmin_match_pandas(mpd, dev, nparts):
    import modin.config as cfg

    cfg.NPartitions.put(nparts)
    config.NPartitions.put(nparts)
    pdf = _frame()
    _cases(mpd.DataFrame, pdf)
    for name, lab in _labelled(pdf).items():
        for fn in ("idxmax", "idxmin"):
            _same(getattr(mpd.DataFrame(lab).groupby("key"), fn)()._to_pandas(), getattr(lab.groupby("key"), fn)())
    two = pdf.fillna(1.0).assign(k2=(np.arange(len(pdf)) % 3).astype(np.int64))  # no all-NaN (key, k2) group
    lab = pdf.drop(columns="key").set_axis(pandas.Index(pdf["key"].to_numpy(), name="lab"))
    for fn in ("idxmax", "idxmin"):
        _same(getattr(mpd.DataFrame(two).groupby(["key", "k2"]), fn)()._to_pandas(), getattr(two.groupby(["key", "k2"]), fn)())
        _same(getattr(mpd.DataFrame(lab).groupby(level=0), fn)()._to_pandas(), getattr(lab.groupby(level=0), fn)())
        got = getattr(mpd.DataFrame(pdf).groupby("key")["f"], fn)()._to_pandas()
        pandas.testing.assert_series_equal(got, getattr(pdf.groupby("key")["f"], fn)())


@needs_modin
def test_plugin_float_key_nan_group_and_refusals(mpd, dev):
    """Under a float key the NaN-key group whose values are all NaN does not raise with dropna=True (it is not in the
    result) and raises with dropna=False."""
    pdf = _frame()
    fk = pdf.assign(key=np.where(pdf["key"] == 2, np.nan, pdf["key"] * 0.5 - 1.0))
    fk.loc[fk["key"].isna(), ["f", "inf"]] = np.nan
    for fn in ("idxmax", "idxmin"):
        _same(getattr(mpd.DataFrame(fk).groupby("key"), fn)()._to_pandas(), getattr(fk.groupby("key"), fn)())
        with pytest.raises(ValueError, match=f"{fn} {ALL_NA}"):
            getattr(fk.groupby("key", dropna=False), fn)()
        with pytest.raises(ValueError, match=f"{fn} {ALL_NA}"):
            getattr(mpd.DataFrame(fk).groupby("key", dropna=False), fn)()
    nanfree = pdf.assign(key=pdf["key"] * 0.5 - 1.0)
    for fn in ("idxmax", "idxmin"):
        _same(getattr(mpd.DataFrame(nanfree).groupby("key", dropna=False), fn)()._to_pandas(),
              getattr(nanfree.groupby("key", dropna=False), fn)())  # fmt: skip
    df = mpd.DataFrame(pdf)
    for fn in ("idxmax", "idxmin"):
        with pytest.raises(NotImplementedError, match="skipna=False"):
            getattr(df.groupby("key"), fn)(skipna=False)
        with pytest.raises(ValueError, match=f"{fn} {ALL_NA}"):
            getattr(mpd.DataFrame(pdf.assign(f=np.nan)).groupby("key"), fn)()


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
    """``full``: 14 rows per rank, every group on every rank; group 1's maximum of ``f`` (9.5) sits at the last row of
    every rank but the last and at the first row of the next, so the lowest rank's row wins; ``tiny``: fewer rows than
    ranks, so the last rank has none, with float64 row labels; ``nan``: group 3 has no value in ``f``."""
    n = 14 * ws
    r = np.arange(n)
    key = (r % 4).astype(np.int64)
    f = np.where(r % 5 == 0, np.nan, np.sin(r))
    for b in range(1, ws):
        for row in (14 * b - 1, 14 * b):
            key[row], f[row] = 1, 9.5
    f[key == 1] = np.where(np.isnan(f[key == 1]), 0.0, f[key == 1])
    full = pandas.DataFrame({"key": key, "f": f, "i": r * 3 - 20, "b": r % 3 == 1})
    tiny = full.fillna(0.0).iloc[: ws - 1].set_axis(pandas.Index(np.arange(ws - 1) * 0.25 + 1.0))
    nan = full.assign(f=np.where(key == 3, np.nan, np.nan_to_num(f)))
    return {"full": full, "tiny": tiny, "nan": nan}


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
                for fn in ("idxmax", "idxmin"):
                    out[(dense, name, fn)] = getattr(df.groupby("key"), fn)()._to_pandas()
            for fn in ("idxmax", "idxmin"):
                try:
                    getattr(bpd.DataFrame(frames["nan"]).groupby("key"), fn)()
                    out[(dense, "nan", fn)] = "no error"
                except ValueError as e:
                    out[(dense, "nan", fn)] = str(e)
                try:
                    bpd.DataFrame(frames["full"]).groupby("key").agg({"f": fn, "i": "count"})
                    out[(dense, "mixed", fn)] = "no error"
                except NotImplementedError as e:
                    out[(dense, "mixed", fn)] = str(e)
    return out


@pytest.mark.parametrize("ws", [2, 3])
def test_ranks_combine_in_rank_order(ws):
    import torch.multiprocessing as mp

    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(ws, _free_port(), ret), nprocs=ws, join=True)
    frames = _rank_frames(ws)
    assert frames["full"].groupby("key")["f"].idxmax()[1] == 13
    assert frames["tiny"].index.dtype == np.float64
    for r in range(ws):  # every rank holds the whole answer and raises the same errors
        assert len(ret[r]) == 2 * 8
        for (dense, name, fn), got in ret[r].items():
            if name == "nan":
                assert got == f"{fn} {ALL_NA}.", got
            elif name == "mixed":
                assert "across ranks" in got, got
            else:
                _same(got, getattr(frames[name].groupby("key"), fn)())
