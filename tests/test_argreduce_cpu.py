"""``idxmax`` / ``idxmin`` (and ``Series.argmax`` / ``argmin``) through both front doors, with the device replaced by
the numpy test double: the Reduce-template wiring, the row -> label mapping for every label kind, pandas' errors and
refusals, and the rank-order combine of the W-vectors under 2 and 3 gloo ranks (one of them without rows).  Results
are compared with pandas for values, index, name and dtype.  ``arg_reduce_columns`` below is the numpy twin of
``ops.arg_reduce_columns`` (csrc/reduce.cu ``mb200_reduce_arg_columns``)."""

import contextlib
import os
import sys

import numpy as np
import pandas
import pytest
import torch

from modin_b200 import config, ops

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref")
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max


def arg_reduce_columns(op, cols, variant=0):
    """numpy twin of ``ops.arg_reduce_columns``: (extreme value, first row holding it or -1, #non-NaN) per column."""
    vals, poss, cnts = [], [], []
    for c in cols:
        x = c.data.numpy()
        if c.dtype == np.bool_:
            raise TypeError("arg-reductions over bool columns are not on the B200 path (widen them to int64)")
        ok = ~np.isnan(x) if x.dtype == np.float64 else np.ones(len(x), dtype=bool)
        n = int(ok.sum())
        if n:
            best = x[ok].max() if op == "max" else x[ok].min()
            pos = int(np.flatnonzero(ok & (x == best))[0])
        else:
            if x.dtype == np.float64:
                best = -np.inf if op == "max" else np.inf
            else:
                best = I64_MIN if op == "max" else I64_MAX
            pos = -1
        vals.append(torch.tensor([best], dtype=torch.from_numpy(x[:0]).dtype))
        poss.append(torch.tensor([pos], dtype=torch.int64))
        cnts.append(torch.tensor([n], dtype=torch.int64))
    return vals, poss, cnts


@contextlib.contextmanager
def double_installed():
    sys.path.insert(0, HERE)
    import cpu_double

    saved = ops.arg_reduce_columns
    with cpu_double.installed():
        ops.arg_reduce_columns = arg_reduce_columns
        try:
            yield
        finally:
            ops.arg_reduce_columns = saved


@pytest.fixture
def dev():
    old = config.NPartitions.get()
    with double_installed():
        yield
    config.NPartitions.put(old)


def _same(got, want):
    pandas.testing.assert_series_equal(got, want, check_index_type=False)


def _frame(n=23, seed=3):
    """float64 / int64 / bool columns with NaN, ties, signed zeros, infinities and the int64 limits."""
    rng = np.random.default_rng(seed)
    f = rng.integers(-3, 4, n).astype(np.float64)
    f[rng.random(n) < 0.3] = np.nan
    z = np.where(np.arange(n) % 2 == 0, -0.0, 0.0)
    inf = np.full(n, -np.inf)
    inf[5] = np.nan
    i = rng.integers(-2, 3, n)
    lim = np.where(np.arange(n) % 3 == 0, I64_MIN, I64_MAX)
    return pandas.DataFrame({"f": f, "i": i, "b": rng.random(n) < 0.4, "z": z, "ninf": inf, "lim": lim,
                             "none": np.zeros(n, dtype=bool)})  # fmt: skip


def _check_both(pdf, mk, **kw):
    df = mk(pdf)
    _same(df.idxmax(**kw), pdf.idxmax(**kw))
    _same(df.idxmin(**kw), pdf.idxmin(**kw))


def _label_cases():
    base = _frame()
    mask = (base["i"] != 0).to_numpy()
    rep = pandas.concat([base.iloc[:11], base.iloc[3:]])  # repeated labels
    return {
        "range offset": base.set_axis(pandas.RangeIndex(7, 7 + len(base))),
        "int64 after mask": base[mask],
        "float64 labels": base.set_axis(pandas.Index(np.arange(len(base)) * 0.5 - 3.0)),
        "repeated labels": rep,
    }


def _errors(df, pdf, calls=(lambda d: d.idxmax(), lambda d: d.idxmin(), lambda d: d.idxmax(skipna=False))):
    for call in calls:
        with pytest.raises(ValueError) as want:
            call(pdf)
        with pytest.raises(ValueError, match=str(want.value)):
            call(df)


# ------------------------------------------------------------------ the Modin-free mirror (modin_b200.pandas)
@pytest.mark.parametrize("nparts", [1, 3])
def test_mirror_idxmax_idxmin_match_pandas(dev, nparts):
    import modin_b200.pandas as bpd

    config.NPartitions.put(nparts)
    for name, pdf in _label_cases().items():
        _check_both(pdf, bpd.DataFrame)
        _check_both(pdf[["i", "b", "lim", "none"]], bpd.DataFrame, skipna=False)  # no NaN: skipna=False is fine


def test_mirror_forty_interleaved_columns(dev):
    import modin_b200.pandas as bpd

    config.NPartitions.put(2)
    base = _frame(37, seed=9)
    kinds = ["f", "i", "b", "z", "lim", "f", "b", "i"]
    pdf = pandas.DataFrame({f"c{j}": np.roll(base[kinds[j % len(kinds)]].to_numpy(), j) for j in range(40)})
    assert len(bpd.DataFrame(pdf)._query_compiler._modin_frame._partitions[0]) == 2  # two column partitions
    _check_both(pdf, bpd.DataFrame)
    _check_both(pdf.set_axis(pandas.RangeIndex(100, 137)), bpd.DataFrame)


def test_mirror_refusals_errors_and_edge_shapes(dev):
    import modin_b200.pandas as bpd

    config.NPartitions.put(2)
    pdf = _frame()
    with pytest.raises(NotImplementedError):
        bpd.DataFrame(pdf.set_axis([f"r{i}" for i in range(len(pdf))])).idxmax()
    with pytest.raises(NotImplementedError):
        bpd.DataFrame(pdf).idxmax(axis=1)
    bad = pdf[["f", "i"]].copy()
    bad["all_nan"] = np.nan
    _errors(bpd.DataFrame(bad), bad)
    _errors(bpd.DataFrame(pdf[["f", "i"]]), pdf[["f", "i"]], [lambda d: d.idxmin(skipna=False)])  # a NaN
    empty = pdf.iloc[:0]
    _errors(bpd.DataFrame(empty), empty)  # zero rows: argmax / argmin of an empty sequence
    for nocols in (pandas.DataFrame(index=range(4)), pandas.DataFrame()):
        _same(bpd.DataFrame(nocols).idxmax(), nocols.idxmax())


def test_mirror_series_idxmax_argmax_argmin(dev):
    import modin_b200.pandas as bpd

    config.NPartitions.put(3)
    pdf = _frame().set_axis(pandas.RangeIndex(40, 63))
    for c in ("f", "i", "z", "ninf", "lim"):
        s, ps = bpd.Series(pdf[c]), pdf[c]
        for got, want in ((s.idxmax(), ps.idxmax()), (s.idxmin(), ps.idxmin()), (s.argmax(), ps.argmax()),
                          (s.argmin(), ps.argmin())):  # fmt: skip
            assert got == want and isinstance(got, (int, np.integer)) == isinstance(want, (int, np.integer)), (c, got)
    masked = pdf[pdf["i"] > 0]["f"]
    fi = bpd.DataFrame(pdf[["f", "i"]])  # row selection takes frames without bool columns
    s = fi[fi["i"] > 0]["f"]
    assert (s.idxmax(), s.argmax(), s.argmin()) == (masked.idxmax(), masked.argmax(), masked.argmin())
    with pytest.raises(ValueError, match="Encountered all NA values"):
        bpd.Series(pandas.Series([np.nan, np.nan])).argmax()


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
    for name, pdf in _label_cases().items():
        got = mpd.DataFrame(pdf)
        pandas.testing.assert_series_equal(got.idxmax()._to_pandas(), pdf.idxmax(), check_index_type=False)
        pandas.testing.assert_series_equal(got.idxmin()._to_pandas(), pdf.idxmin(), check_index_type=False)
    pdf = _frame()
    s, ps = mpd.DataFrame(pdf)["f"], pdf["f"]
    assert (s.idxmax(), s.argmax(), s.argmin()) == (ps.idxmax(), ps.argmax(), ps.argmin())
    # float64 labels from a groupby on a float key
    keyed = pandas.DataFrame({"k": np.array([0.5, -1.5, 2.0, 0.5, 2.0, -1.5]), "v": [3.0, 1.0, 7.0, 2.0, 0.0, 9.0],
                              "w": [1.0, 5.0, 5.0, 0.0, 2.0, 2.0]})  # fmt: skip
    g, pg = mpd.DataFrame(keyed).groupby("k").sum(), keyed.groupby("k").sum()
    pandas.testing.assert_series_equal(g.idxmax()._to_pandas(), pg.idxmax(), check_index_type=False)
    pandas.testing.assert_series_equal(g.idxmin()._to_pandas(), pg.idxmin(), check_index_type=False)


@needs_modin
def test_plugin_refusals_and_errors(mpd, dev):
    pdf = _frame()
    with pytest.raises(NotImplementedError):
        mpd.DataFrame(pdf.set_axis([f"r{i}" for i in range(len(pdf))])).idxmax()
    with pytest.raises(NotImplementedError):
        mpd.DataFrame(pdf).idxmax(axis=1)
    bad = pdf[["f", "i"]].copy()
    bad["all_nan"] = np.nan
    _errors(mpd.DataFrame(bad), bad)
    # the other Reduce registrations stay refused
    with pytest.raises(NotImplementedError):
        mpd.DataFrame(pdf[["f"]]).median()


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


def _rank_frame(ws):
    """12 rows per rank.  ``tie``: the maximum sits at the last row of rank 0 and the first row of rank 1 (rank 0 must
    win); ``last``: valid values on the last rank only; ``ninf``: all -inf; ``lim``: int64 limits on every rank."""
    n = 12 * ws
    r = np.arange(n)
    tie = np.where((r == 11) | (r == 12), 9.0, np.sin(r))
    last = np.where(r >= n - 12, np.cos(r), np.nan)
    lim = np.where(r % 5 == 0, I64_MAX, np.where(r % 5 == 1, I64_MIN, r))
    return pandas.DataFrame({"tie": tie, "last": last, "ninf": np.full(n, -np.inf), "lim": lim, "b": r % 7 == 3,
                             "z": np.where(r % 2 == 0, 0.0, -0.0)})  # fmt: skip


def _rank_job(rank, ws):
    import modin_b200.pandas as bpd

    out = {}
    with double_installed():
        config.NPartitions.put(2)
        pdf = _rank_frame(ws)
        df = bpd.DataFrame(pdf)
        empty_rank = ws - 2  # rows of this rank are filtered away
        keep = np.arange(len(pdf)) // 12 != empty_rank
        nb = [c for c in pdf.columns if c != "b"]  # row selection takes frames without bool columns
        dm = df[nb][bpd.DataFrame(pandas.DataFrame({"m": keep}))["m"]]
        for key, d in (("full", df), ("masked", dm)):
            out[key] = (d.idxmax(), d.idxmin())
        out["series"] = (df["tie"].idxmax(), df["tie"].argmax(), df["last"].argmin())
        bad = pdf.copy()
        bad["nan"] = np.nan
        try:
            bpd.DataFrame(bad).idxmax()
            out["all_nan"] = None
        except ValueError as e:
            out["all_nan"] = str(e)
        try:
            bpd.DataFrame(pdf[["tie", "last"]]).idxmin(skipna=False)
            out["skipna"] = None
        except ValueError as e:
            out["skipna"] = str(e)
    return out


@pytest.mark.parametrize("ws", [2, 3])
def test_ranks_combine_in_rank_order(ws):
    import torch.multiprocessing as mp

    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(ws, _free_port(), ret), nprocs=ws, join=True)
    pdf = _rank_frame(ws)
    keep = np.arange(len(pdf)) // 12 != ws - 2
    for r in range(ws):  # every rank holds the whole answer
        o = ret[r]
        for key, want in (("full", pdf), ("masked", pdf.drop(columns="b")[keep])):
            _same(o[key][0], want.idxmax())
            _same(o[key][1], want.idxmin())
        assert o["series"] == (pdf["tie"].idxmax(), pdf["tie"].argmax(), pdf["last"].argmin())
        assert o["all_nan"] == "Encountered all NA values"
        assert o["skipna"] == "Encountered an NA value with skipna=False"
    assert pdf["tie"].idxmax() == 11  # the tie across the rank boundary goes to the lower rank
