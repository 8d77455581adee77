"""CPU tests of the host-side stack (templates -> frame -> partition manager -> partitions -> functors)
with the device replaced by the numpy test double (tests/cpu_double.py).  What is under test is the
HOST LOGIC -- grids, call-queue fusion, argument plumbing, metadata, error behaviour -- against the
oracle; kernel arithmetic is checked by the ``gpu`` tests."""

import numpy as np
import pandas
import pytest

from modin_b200 import config, synth
from oracle import reference_path as orc


def _same(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(((a == b) | (np.isnan(a) & np.isnan(b))).all())


@pytest.fixture(autouse=True)
def _np4():
    old = config.NPartitions.get()
    config.NPartitions.put(4)
    yield
    config.NPartitions.put(old)


def test_map_binary_tree_reduce_through_the_api(cpu_device):
    import modin_b200.pandas as bpd

    pdf = synth.host_frame(1003, 5, seed=3, nan_per_64k=4000)
    df = bpd.DataFrame(pdf)
    assert df._query_compiler._modin_frame._partitions.shape == (4, 1)
    assert _same(df.abs()._to_pandas().to_numpy(), orc.df_abs(pdf, 4).to_numpy())
    assert _same((df * 1.5 + 2.0)._to_pandas().to_numpy(), orc.a_mul_b_add_c(pdf, 1.5, 2.0, 4).to_numpy())
    assert _same((-df)._to_pandas().to_numpy(), (-pdf).to_numpy())
    assert _same(df.fillna(0.25)._to_pandas().to_numpy(), orc.df_fillna(pdf, 0.25, 4).to_numpy())
    assert np.allclose(df.sum().to_numpy(), orc.df_sum(pdf, 4).to_numpy(), rtol=0, atol=1e-9)
    assert np.allclose(df.mean().to_numpy(), orc.df_mean(pdf, 4).to_numpy(), rtol=0, atol=1e-12)
    assert _same(df.count().to_numpy(), orc.df_count(pdf, 4).to_numpy())
    assert _same(df.min().to_numpy(), orc.df_min(pdf, 4).to_numpy())
    assert _same(df.max(skipna=False).to_numpy(), orc.df_max(pdf, 4, skipna=False).to_numpy())
    assert _same(df.sum(min_count=1).to_numpy(), orc.df_sum(pdf, 4, min_count=1).to_numpy()) or \
        np.allclose(df.sum(min_count=1).to_numpy(), orc.df_sum(pdf, 4, min_count=1).to_numpy(), atol=1e-9, equal_nan=True)
    res = df.sum()
    assert isinstance(res, pandas.Series) and list(res.index) == list(pdf.columns) and res.name is None
    small = synth.host_frame(40, 3, seed=9, nan_per_64k=6000) * 1.5
    assert np.allclose(bpd.DataFrame(small).prod().to_numpy(), orc.df_prod(small, 4).to_numpy(), rtol=1e-12)


def test_frame_frame_ops_and_fusion(cpu_device):
    import modin_b200.pandas as bpd

    a, b, c = (synth.host_frame(600, 3, seed=s) for s in (1, 2, 3))
    A, B, C = bpd.DataFrame(a), bpd.DataFrame(b), bpd.DataFrame(c)
    out = A * B + C
    parts = out._query_compiler._modin_frame._partitions
    assert all(len(p.call_queue) == 2 for p in parts.flatten())  # mul, add queued -> fused at drain
    assert _same(out._to_pandas().to_numpy(), orc.a_mul_b_add_c(a, b, c, 4).to_numpy())
    assert _same((A / B)._to_pandas().to_numpy(), (a / b).to_numpy())
    assert _same((A >= B)._to_pandas().to_numpy(), (a >= b).to_numpy())
    # differently LABELLED operands are aligned like pandas: the row labels are joined, missing rows become NaN
    # (the reindexing half of _copartition, df.py:3799-3840)
    hs = synth.host_frame(599, 3)
    got = (A + bpd.DataFrame(hs))._to_pandas()
    assert got.index.equals((a + hs).index) and _same(got.to_numpy(), (a + hs).to_numpy())


@pytest.mark.parametrize("dense", [True, False])
def test_groupby_and_merge_through_the_api(cpu_device, dense):
    import modin_b200.pandas as bpd

    config.GroupbyDenseKeys.put(dense)  # fused dense table vs map -> regroup; restored below
    try:
        _groupby_and_merge_checks(bpd)
    finally:
        config.GroupbyDenseKeys.put(True)


def _groupby_and_merge_checks(bpd):
    pdf = synth.host_frame(5003, 3, seed=42, nan_per_64k=2000, key_modulus=41)
    df = bpd.DataFrame(pdf)
    g = df.groupby("key")
    for agg in ("sum", "count", "mean", "min", "max"):
        got = getattr(g, agg)()._to_pandas()
        want = orc.groupby_reduce(pdf, "key", agg, 4)
        assert list(got.index) == list(want.index) and got.index.name == "key"
        assert list(got.columns) == list(want.columns)
        assert np.allclose(got.to_numpy(), want.to_numpy(), rtol=0, atol=1e-9, equal_nan=True)
    assert _same(g.size()._to_pandas().to_numpy(), orc.groupby_reduce(pdf, "key", "size", 4).to_numpy())
    # result frame metadata
    res = g.sum()
    assert len(res) == 41 and list(res.columns) == ["c0", "c1", "c2"]

    rng = np.random.RandomState(0)
    dim = pandas.DataFrame({"key": rng.permutation(41)[:35].astype(np.int64), "d0": rng.randn(35),
                            "c0": np.arange(35, dtype=np.int64)})  # fmt: skip
    left = df.merge(bpd.DataFrame(dim), on="key", how="left")._to_pandas()
    wl = orc.broadcast_merge(pdf, dim, "key", "left", 4)
    assert list(left.columns) == list(wl.columns)  # overlapping "c0" gets _x / _y suffixes
    assert _same(left.to_numpy(dtype=np.float64), wl.to_numpy(dtype=np.float64))
    inner = df.merge(bpd.DataFrame(dim), on="key", how="inner")._to_pandas()
    assert _same(inner.to_numpy(dtype=np.float64),
                 orc.broadcast_merge(pdf, dim, "key", "inner", 4).to_numpy(dtype=np.float64))
    dup = pandas.DataFrame({"key": np.array([1, 1, 2], dtype=np.int64), "d": [1.0, 2.0, 3.0]})
    # repeated right keys: many-to-many like pandas.merge (one output row per matching right row, left order kept)
    for how in ("left", "inner"):
        got = df.merge(bpd.DataFrame(dup), on="key", how=how)._to_pandas()
        want = pdf.merge(dup, on="key", how=how)
        assert list(got.columns) == list(want.columns) and _same(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64))


def test_errors_match_pandas_types(cpu_device):
    import modin_b200.pandas as bpd

    df = bpd.DataFrame(synth.host_frame(50, 2))
    with pytest.raises(ValueError):
        df.fillna()
    with pytest.raises(TypeError):
        df.fillna([1, 2])
    with pytest.raises(KeyError):
        df["nope"]
    with pytest.raises(KeyError):
        df.groupby("nope")
    with pytest.raises(NotImplementedError):
        df.sum(axis=1)
    with pytest.raises(NotImplementedError):
        df.merge(df, how="outer", on="c0")
    with pytest.raises(TypeError):
        bpd.DataFrame(pandas.DataFrame({"s": ["a", "b"]}))


def test_wide_frames_use_a_2d_grid(cpu_device):
    import modin_b200.pandas as bpd

    pdf = pandas.DataFrame(np.arange(64 * 40, dtype=np.float64).reshape(64, 40))
    df = bpd.DataFrame(pdf)
    f = df._query_compiler._modin_frame
    assert f._partitions.shape == (2, 2) and f.column_widths == [32, 8] and f.row_lengths == [32, 32]
    assert _same((df * 2.0)._to_pandas().to_numpy(), (pdf * 2.0).to_numpy())
    assert _same(df.sum().to_numpy(), pdf.sum().to_numpy())
    assert _same(df[[0, 35]]._to_pandas().to_numpy(), pdf[[0, 35]].to_numpy())


def test_series_operands_both_axes(cpu_device):
    """frame (op) Series: along columns = row vector (lazy map), along rows = broadcast_apply."""
    import modin_b200.pandas as bpd

    pdf = synth.host_frame(900, 3, seed=6)
    df = bpd.DataFrame(pdf)
    col = pdf["c1"]
    ser = df["c1"]
    assert isinstance(ser, bpd.Series) and ser.name == "c1" and len(ser) == 900
    assert _same(df.mul(ser, axis=0)._to_pandas().to_numpy(), pdf.mul(col, axis=0).to_numpy())
    assert _same(df.sub(ser, axis=0)._to_pandas().to_numpy(), pdf.sub(col, axis=0).to_numpy())
    assert _same(df.rsub(ser, axis=0)._to_pandas().to_numpy(), pdf.rsub(col, axis=0).to_numpy())
    rowvec = pandas.Series([1.0, -2.0, 0.5], index=pdf.columns)
    assert _same((df + bpd.Series(rowvec))._to_pandas().to_numpy(), (pdf + rowvec).to_numpy())
    assert np.isclose(ser.sum(), col.sum()) and ser.count() == 900


def test_round_clip_var_std_through_the_api(cpu_device):
    import modin_b200.pandas as bpd

    pdf = synth.host_frame(2003, 4, seed=8, nan_per_64k=3000)
    df = bpd.DataFrame(pdf)
    assert _same(df.round(2)._to_pandas().to_numpy(), orc.df_round(pdf, 2, 4).to_numpy())
    assert _same((df * 100.0).round(-1)._to_pandas().to_numpy(), orc.df_round(pdf * 100.0, -1, 4).to_numpy())
    assert _same(df.clip(-0.5, 0.75)._to_pandas().to_numpy(), orc.df_clip(pdf, -0.5, 0.75, 4).to_numpy())
    assert _same(df.clip(upper=0.1)._to_pandas().to_numpy(), orc.df_clip(pdf, None, 0.1, 4).to_numpy())
    for ddof in (0, 1):
        assert np.allclose(df.var(ddof=ddof).to_numpy(), orc.df_var(pdf, 4, ddof=ddof).to_numpy(), rtol=1e-12, atol=0)
        assert np.allclose(df.std(ddof=ddof).to_numpy(), orc.df_std(pdf, 4, ddof=ddof).to_numpy(), rtol=1e-12, atol=0)
    assert np.isnan(df.var(skipna=False).to_numpy()).all()
    v = df.var()
    assert isinstance(v, pandas.Series) and list(v.index) == list(pdf.columns) and v.name is None
    assert np.isclose(df["c1"].std(), pdf["c1"].std(), rtol=1e-12)
    with pytest.raises(NotImplementedError):
        df.round(1.5)
    with pytest.raises(NotImplementedError):
        df.clip(lower=[1, 2, 3, 4])
    with pytest.raises(NotImplementedError):
        df.var(axis=1)


@pytest.mark.parametrize("dense", [True, False])
def test_groupby_dictionary_aggregation(cpu_device, dense):
    import modin_b200.pandas as bpd

    config.GroupbyDenseKeys.put(dense)
    try:
        pdf = synth.host_frame(4001, 4, seed=5, nan_per_64k=2500, key_modulus=53)
        spec = {"c2": "max", "c0": "sum", "c3": "count", "c1": "sum"}
        got = bpd.DataFrame(pdf).groupby("key").agg(spec)._to_pandas()
        want = pdf.groupby("key").agg(spec)
        assert list(got.columns) == list(want.columns) and list(got.index) == list(want.index) and got.index.name == "key"
        assert np.allclose(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64), rtol=0, atol=1e-9, equal_nan=True)
        got = bpd.DataFrame(pdf).groupby("key", as_index=False).agg(spec)._to_pandas()
        want = pdf.groupby("key", as_index=False).agg(spec)
        assert list(got.columns) == list(want.columns) and got.index.equals(want.index)
        assert np.allclose(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64), rtol=0, atol=1e-9, equal_nan=True)
        with pytest.raises(NotImplementedError):
            bpd.DataFrame(pdf).groupby("key").agg({"c0": "median"})
        with pytest.raises(KeyError):
            bpd.DataFrame(pdf).groupby("key").agg({"nope": "sum"})
    finally:
        config.GroupbyDenseKeys.put(True)


def test_binary_ops_between_differently_partitioned_frames(cpu_device):
    """The row half of _copartition (df.py:3709-3848): same labels, different row cuts -> the right operand is
    re-cut along the left's partition lengths (views, or a D2D concat where a target spans several sources)."""
    import modin_b200.pandas as bpd

    a, b = synth.host_frame(1001, 3, seed=1), synth.host_frame(1001, 3, seed=2, nan_per_64k=5000)
    A = bpd.DataFrame(a)  # 4 row partitions
    config.NPartitions.put(3)
    B = bpd.DataFrame(b)  # 3 row partitions
    config.NPartitions.put(4)
    fa, fb = A._query_compiler._modin_frame, B._query_compiler._modin_frame
    assert fa.row_lengths != fb.row_lengths and sum(fa.row_lengths) == sum(fb.row_lengths)
    out = A * B + B
    assert out._query_compiler._modin_frame.row_lengths == fa.row_lengths
    assert _same(out._to_pandas().to_numpy(), (a * b + b).to_numpy())
    assert _same((B - A)._to_pandas().to_numpy(), (b - a).to_numpy())  # and the other way round (3 cuts)
    assert _same((A >= B)._to_pandas().to_numpy(), (a >= b).to_numpy())
    re = fb._repartition_rows([0, 1001])  # empty partitions are filtered by the frame constructor, as in Modin
    assert sum(re.row_lengths) == 1001 and _same(re.to_pandas().to_numpy(), b.to_numpy())
    re = fb._repartition_rows([1, 500, 500])
    assert re.row_lengths == [1, 500, 500] and _same(re.to_pandas().to_numpy(), b.to_numpy())


def test_dlpack_interchange_is_zero_copy(cpu_device):
    import torch

    import modin_b200.pandas as bpd

    a = torch.arange(10, dtype=torch.float64)
    k = torch.arange(10, dtype=torch.int64) % 3
    df = bpd.from_dlpack({"x": a, "key": k})
    assert list(df.columns) == ["x", "key"] and len(df) == 10
    views = bpd.to_dlpack(df)
    assert views["x"].data_ptr() == a.data_ptr() and views["key"].data_ptr() == k.data_ptr()  # no copy either way
    assert _same((df[["x"]] * 2.0)._to_pandas().to_numpy().ravel(), (a * 2).numpy())
    got = df.groupby("key").sum()._to_pandas()
    assert list(got.index) == [0, 1, 2] and _same(got["x"].to_numpy(), [18.0, 12.0, 15.0])
    out = bpd.to_dlpack(bpd.DataFrame(synth.host_frame(100, 2)))  # 4 row partitions -> one device concatenation
    assert out["c0"].shape == (100,) and torch.from_dlpack(out["c1"]).shape == (100,)
    with pytest.raises(TypeError):
        bpd.from_dlpack({"x": torch.zeros(3, dtype=torch.float32)})
    with pytest.raises(ValueError):
        bpd.from_dlpack({"x": a, "y": torch.zeros(3, dtype=torch.float64)})


def test_sort_values_is_a_stable_sort_with_nan_last(cpu_device):
    import modin_b200.pandas as bpd

    pdf = synth.host_frame(3001, 3, seed=2, nan_per_64k=4000, key_modulus=17)
    df = bpd.DataFrame(pdf)
    for by, asc in (("key", True), ("key", False), ("c1", True), ("c1", False)):
        got = df.sort_values(by, ascending=asc)._to_pandas()
        want = pdf.sort_values(by, ascending=asc, kind="stable")
        assert list(got.index) == list(want.index), (by, asc)  # permuted row labels travel with the rows
        assert _same(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64)), (by, asc)
    got = df.sort_values("c0", ignore_index=True)._to_pandas()
    want = pdf.sort_values("c0", kind="stable", ignore_index=True)
    assert list(got.index) == list(want.index) and _same(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64))
    with pytest.raises(NotImplementedError):
        df.sort_values(["key", "c0"])
    with pytest.raises(KeyError):
        df.sort_values("nope")


def test_series_nunique_and_value_counts(cpu_device):
    import modin_b200.pandas as bpd

    pdf = synth.host_frame(4001, 1, seed=3, key_modulus=29, key_skew=True)
    s = bpd.DataFrame(pdf)["key"]
    assert s.nunique() == pdf["key"].nunique()
    got = s.value_counts()._to_pandas()
    want = pdf["key"].value_counts()
    assert list(got.to_numpy()) == list(want.to_numpy())  # counts, most frequent first
    assert dict(zip(got.index, got.to_numpy())) == dict(zip(want.index, want.to_numpy()))
    asc = s.value_counts(ascending=True)._to_pandas()
    assert list(asc.to_numpy()) == sorted(want.to_numpy())
    assert len(s.value_counts(sort=False)) == pdf["key"].nunique()


def test_boolean_pipelines(cpu_device):
    """Comparisons produce bool frames; & | ^ ~, any / all, and sum / mean / count over them stay on the device."""
    import modin_b200.pandas as bpd

    pdf = synth.host_frame(2003, 3, seed=4, nan_per_64k=2000)
    df = bpd.DataFrame(pdf)
    m, pm = (df > 0.0) & (df < 1.0), (pdf > 0.0) & (pdf < 1.0)
    assert _same(m._to_pandas().to_numpy().astype(float), pm.to_numpy().astype(float))
    assert _same(((df > 0.5) | (df < -0.5))._to_pandas().to_numpy().astype(float), ((pdf > 0.5) | (pdf < -0.5)).to_numpy().astype(float))
    assert _same(((df > 0.0) ^ (df > 1.0))._to_pandas().to_numpy().astype(float), ((pdf > 0.0) ^ (pdf > 1.0)).to_numpy().astype(float))
    assert _same((~m)._to_pandas().to_numpy().astype(float), (~pm).to_numpy().astype(float))
    assert list(m.sum().to_numpy()) == list(pm.sum().to_numpy()) and m.sum().dtype == np.int64
    assert list(m.count().to_numpy()) == list(pm.count().to_numpy())
    assert np.allclose(m.mean().to_numpy(), pm.mean().to_numpy(), rtol=1e-12)
    assert list(m.any().to_numpy()) == list(pm.any().to_numpy()) and m.any().dtype == np.bool_
    assert list(m.all().to_numpy()) == list(pm.all().to_numpy())
    assert list((df > -100.0).all().to_numpy()) == list((pdf > -100.0).all().to_numpy())  # NaN > x is False
    assert list((df > 100.0).any().to_numpy()) == [False, False, False]
    with pytest.raises(NotImplementedError):
        df.any()  # numeric frames: compare first
    with pytest.raises(NotImplementedError):
        m & df
    with pytest.raises(NotImplementedError):
        m.max()


def test_repartition_rows_random_cuts(cpu_device):
    """Property: re-cutting never changes the rows, whatever the source and target cuts."""
    import modin_b200.pandas as bpd

    rng = np.random.RandomState(7)
    pdf = synth.host_frame(257, 2, seed=9, nan_per_64k=9000)
    for trial in range(25):
        config.NPartitions.put(int(rng.randint(1, 7)))
        frame = bpd.DataFrame(pdf)._query_compiler._modin_frame
        k = int(rng.randint(1, 6))
        cuts = np.sort(rng.randint(0, 258, size=k - 1)) if k > 1 else np.array([], dtype=int)
        lengths = np.diff(np.concatenate([[0], cuts, [257]])).tolist()
        re = frame._repartition_rows(lengths)
        assert sum(re.row_lengths) == 257 and [n for n in lengths if n] == re.row_lengths, (trial, lengths)
        assert _same(re.to_pandas().to_numpy(), pdf.to_numpy())
    config.NPartitions.put(4)


@pytest.mark.parametrize("dense", [True, False])
def test_multi_key_groupby_packs_the_keys(cpu_device, dense):
    import modin_b200.pandas as bpd

    config.GroupbyDenseKeys.put(dense)
    try:
        pdf = synth.host_frame(6007, 3, seed=12, nan_per_64k=2000, key_modulus=7)
        pdf["k2"] = synth.gen_i64(6007, 99, 1, 5) * 10 - 20  # negative base, gaps
        pdf["k3"] = synth.gen_i64(6007, 98, 2, 3)
        for keys in (["key", "k2"], ["k2", "key", "k3"]):
            src = pdf if "k3" in keys else pdf.drop(columns="k3")  # value columns must be float64 on this path
            g, pg = bpd.DataFrame(src).groupby(keys), src.groupby(keys)
            for agg in ("sum", "count", "mean", "min", "max"):
                got, want = getattr(g, agg)()._to_pandas(), getattr(pg, agg)()
                assert list(got.index.names) == keys and list(got.columns) == list(want.columns)
                assert got.index.equals(want.index), (keys, agg)
                assert np.allclose(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64), rtol=0, atol=1e-9,
                                   equal_nan=True), (keys, agg)  # fmt: skip
            sz = g.size()._to_pandas()
            assert sz.index.equals(pg.size().index) and list(sz.to_numpy()) == list(pg.size().to_numpy())
        df = bpd.DataFrame(pdf.drop(columns="k3"))
        got = df.groupby(["key", "k2"]).agg({"c1": "max", "c0": "sum"})._to_pandas()
        want = pdf.groupby(["key", "k2"]).agg({"c1": "max", "c0": "sum"})
        assert got.index.equals(want.index) and np.allclose(got.to_numpy(), want.to_numpy(), atol=1e-9, equal_nan=True)
        # as_index=False: the keys are unpacked first, then become the leading columns
        got = df.groupby(["key", "k2"], as_index=False).sum()._to_pandas()
        want = pdf.drop(columns="k3").groupby(["key", "k2"], as_index=False).sum()
        assert list(got.columns) == list(want.columns) and got.index.equals(want.index)
        assert np.allclose(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64), rtol=0, atol=1e-9, equal_nan=True)
        with pytest.raises(KeyError):
            df.groupby(["key", "nope"])
        with pytest.raises(NotImplementedError):
            df.groupby(["key", "c0"])  # float key
    finally:
        config.GroupbyDenseKeys.put(True)


def test_boolean_row_selection_and_dropna(cpu_device):
    import modin_b200.pandas as bpd

    pdf = synth.host_frame(3001, 3, seed=21, nan_per_64k=6000, key_modulus=9)
    df = bpd.DataFrame(pdf)
    for got, want in (
        (df[df["c0"] > 0.5], pdf[pdf["c0"] > 0.5]),
        (df[(df["c0"] > 0.0) & (df["c1"] < 0.0)], pdf[(pdf["c0"] > 0.0) & (pdf["c1"] < 0.0)]),
        (df[df["key"] == 3], pdf[pdf["key"] == 3]),
        (df[df["c2"] > 100.0], pdf[pdf["c2"] > 100.0]),  # nothing survives
        (df.dropna(), pdf.dropna()),
        (df.dropna(how="all", subset=["c0", "c1"]), pdf.dropna(how="all", subset=["c0", "c1"])),
        (df.dropna(subset=["c2"]), pdf.dropna(subset=["c2"])),
    ):
        g = got._to_pandas()
        assert list(g.index) == list(want.index) and list(g.columns) == list(want.columns)
        assert _same(g.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64))
    # the filtered frame is a normal frame: reduce / group / filter again
    sel = df[df["c0"] > 0.0]
    assert np.allclose(sel.sum().to_numpy(), pdf[pdf["c0"] > 0.0].sum().to_numpy(), atol=1e-9)
    g = sel.groupby("key").count()._to_pandas()
    assert _same(g.to_numpy(), pdf[pdf["c0"] > 0.0].groupby("key").count().to_numpy())
    again = sel[sel["c1"] > 0.0]._to_pandas()
    want = pdf[(pdf["c0"] > 0.0) & (pdf["c1"] > 0.0)]
    assert list(again.index) == list(want.index) and _same(again.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64))
    with pytest.raises(pandas.errors.IndexingError):  # pandas: "Unalignable boolean Series provided as indexer"
        df[bpd.DataFrame(pdf.iloc[:100])["c0"] > 0.0]
    with pytest.raises(NotImplementedError):
        df[df["c0"]]


def test_structural_ops_share_buffers(cpu_device):
    """setitem / assign / drop / rename / head / tail are metadata: no kernel, no copy."""
    import modin_b200.pandas as bpd

    pdf = synth.host_frame(1003, 3, seed=31, nan_per_64k=1000, key_modulus=5)
    df = bpd.DataFrame(pdf)
    df2 = df.copy()
    df2["d"] = df2["c0"] * 2.0
    want = pdf.copy()
    want["d"] = want["c0"] * 2.0
    assert list(df2.columns) == list(want.columns) and _same(df2._to_pandas().to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64))
    assert list(df.columns) == list(pdf.columns)  # the original is untouched
    df2["c1"] = df2["c0"] + df2["c2"]  # replace in place, order kept
    want["c1"] = want["c0"] + want["c2"]
    assert list(df2.columns) == list(want.columns) and _same(df2._to_pandas().to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64))
    a = df.assign(e=lambda x: x["c0"] - x["c1"], f=df["c2"])
    wa = pdf.assign(e=lambda x: x["c0"] - x["c1"], f=pdf["c2"])
    assert list(a.columns) == list(wa.columns) and _same(a._to_pandas().to_numpy(dtype=np.float64), wa.to_numpy(dtype=np.float64))
    assert list(df.drop(columns=["c1", "key"]).columns) == ["c0", "c2"]
    assert list(df.rename(columns={"c0": "x"}).columns) == ["key", "x", "c1", "c2"]
    with pytest.raises(KeyError):
        df.drop(columns=["nope"])
    for n in (0, 1, 5, 250, 251, 1003, 5000):
        assert _same(df.head(n)._to_pandas().to_numpy(dtype=np.float64), pdf.head(n).to_numpy(dtype=np.float64)), n
        assert _same(df.tail(n)._to_pandas().to_numpy(dtype=np.float64), pdf.tail(n).to_numpy(dtype=np.float64)), n
    assert list(df.tail(7)._to_pandas().index) == list(pdf.tail(7).index)
    # a pipeline on top: filter, derive, aggregate
    out = df[df["c0"] > 0.0].assign(g=lambda x: x["c1"] * x["c2"]).groupby("key").sum()._to_pandas()
    w = pdf[pdf["c0"] > 0.0].assign(g=lambda x: x["c1"] * x["c2"]).groupby("key").sum()
    assert list(out.columns) == list(w.columns) and np.allclose(out.to_numpy(), w.to_numpy(), atol=1e-9)


def test_concat_lines_up_partitions_without_copying(cpu_device):
    """concat(axis=0) of equal-column frames and concat(axis=1) of equal-row frames: values AND row labels as pandas."""
    import modin_b200.pandas as bpd

    pa = synth.host_frame(1003, 3, seed=41, nan_per_64k=1000, key_modulus=5)
    pb = synth.host_frame(517, 3, seed=42, nan_per_64k=1000, key_modulus=5)
    a, b = bpd.DataFrame(pa), bpd.DataFrame(pb)
    for ignore in (False, True):
        got = bpd.concat([a, b, a], ignore_index=ignore)._to_pandas()
        want = pandas.concat([pa, pb, pa], ignore_index=ignore)
        assert list(got.columns) == list(want.columns)
        # labels restart at 0 for every input unless ignore_index: they are NOT one running range
        assert list(got.index) == list(want.index), ignore
        assert _same(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64)), ignore
    # the result is an ordinary frame: operators run over the lined-up partitions
    cat = bpd.concat([a, b], ignore_index=True)
    wcat = pandas.concat([pa, pb], ignore_index=True)
    assert len(cat) == len(wcat)
    s, ws = cat[["c0", "c1", "c2"]].sum(), wcat[["c0", "c1", "c2"]].sum()
    s = s._to_pandas() if hasattr(s, "_to_pandas") else s
    assert list(s.index) == list(ws.index) and np.allclose(np.asarray(s), ws.to_numpy(), rtol=0, atol=1e-9)
    g = cat.groupby("key").sum()._to_pandas()
    wg = wcat.groupby("key").sum()
    assert list(g.index) == list(wg.index) and np.allclose(g.to_numpy(), wg.to_numpy(), atol=1e-9)
    assert _same((cat * 2.0)._to_pandas().to_numpy(dtype=np.float64), (wcat * 2.0).to_numpy(dtype=np.float64))
    # inputs are untouched and a single-frame concat is the frame
    assert list(a._to_pandas().index) == list(pa.index)
    assert _same(bpd.concat([b])._to_pandas().to_numpy(dtype=np.float64), pb.to_numpy(dtype=np.float64))
    # axis=1: distinct labels over the same rows
    right = a[["c0", "c1"]].rename(columns={"c0": "x", "c1": "y"})
    wide = bpd.concat([a, right], axis=1)._to_pandas()
    wwide = pandas.concat([pa, pa[["c0", "c1"]].rename(columns={"c0": "x", "c1": "y"})], axis=1)
    assert list(wide.columns) == list(wwide.columns)
    assert _same(wide.to_numpy(dtype=np.float64), wwide.to_numpy(dtype=np.float64))
    # what needs label alignment or dtype promotion is refused, not approximated
    with pytest.raises(NotImplementedError):
        bpd.concat([a, a[["c0", "c1"]]])
    with pytest.raises(NotImplementedError):
        bpd.concat([a[["c0"]], a[["key"]].rename(columns={"key": "c0"})])
    with pytest.raises(ValueError):
        bpd.concat([a, b], axis=1)
    with pytest.raises(ValueError):
        bpd.concat([a, b], axis=2)


def test_astype_widening_casts_and_frame_nunique(cpu_device):
    import modin_b200.pandas as bpd

    rng = np.random.default_rng(51)
    n = 1003
    pdf = pandas.DataFrame({
        "k": rng.integers(-7, 7, n),
        "big": rng.integers(-(2**62), 2**62, n),  # above 2**53: the cast has to round like numpy
        "x": rng.standard_normal(n),
        "flag": rng.integers(0, 2, n).astype(bool),
    })  # fmt: skip
    pdf.loc[::97, "x"] = np.nan
    df = bpd.DataFrame(pdf)

    got, want = df.astype("float64"), pdf.astype("float64")
    assert list(got.dtypes) == list(want.dtypes)
    assert _same(got._to_pandas().to_numpy(), want.to_numpy())
    got, want = df.astype({"k": np.float64, "flag": "int64"}), pdf.astype({"k": np.float64, "flag": "int64"})
    assert list(got.dtypes) == list(want.dtypes)
    gp = got._to_pandas()
    for c in want.columns:
        assert gp[c].dtype == want[c].dtype and _same(gp[c].to_numpy(), want[c].to_numpy()), c
    assert list(df.dtypes) == list(pdf.dtypes)  # the source frame keeps its dtypes
    s = df["flag"].astype(float)
    assert _same(s._to_pandas().to_numpy(), pdf["flag"].astype(float).to_numpy())
    # a cast that changes nothing is a no-op on the same buffers
    same = df[["x"]].astype("float64")
    assert _same(same._to_pandas().to_numpy(), pdf[["x"]].to_numpy())
    # the result feeds the operators
    assert np.allclose((df[["k"]].astype("float64") * 0.5)._to_pandas().to_numpy(), (pdf[["k"]].astype("float64") * 0.5).to_numpy())
    # refused before anything is launched: narrowing / truncating casts, unknown columns, other dtypes
    with pytest.raises(NotImplementedError):
        df.astype("int64")  # float64 -> int64 (pandas raises on the NaNs, truncates otherwise)
    with pytest.raises(NotImplementedError):
        df[["k"]].astype(bool)
    with pytest.raises(NotImplementedError):
        df.astype("float32")
    with pytest.raises(KeyError):
        df.astype({"nope": "float64"})
    with pytest.raises(KeyError):
        pdf.astype({"nope": "float64"})  # same error type as pandas

    ints = df[["k", "big"]]
    got, want = ints.nunique(), pdf[["k", "big"]].nunique()
    assert list(got.index) == list(want.index) and list(got) == list(want) and got.dtype == want.dtype
    with pytest.raises(NotImplementedError):
        df.nunique()  # float / bool columns
    with pytest.raises(NotImplementedError):
        ints.nunique(axis=1)


def test_drop_duplicates_keeps_first_or_last_in_row_order(cpu_device):
    import modin_b200.pandas as bpd

    def check(pdf, **kw):
        got = bpd.DataFrame(pdf).drop_duplicates(**kw)._to_pandas()
        want = pdf.drop_duplicates(**kw)
        assert list(got.columns) == list(want.columns), kw
        assert list(got.index) == list(want.index), (kw, len(pdf))
        assert _same(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64)), (kw, len(pdf))

    rng = np.random.default_rng(61)
    for n, lo, hi in ((1003, -6, 7), (1003, 0, 10**12), (1003, 5, 6), (2, 0, 2), (2, 3, 4), (1, 0, 3), (700, -(2**62), 2**62)):
        pdf = pandas.DataFrame({"key": rng.integers(lo, hi, n), "x": rng.standard_normal(n), "y": rng.standard_normal(n)})
        pdf.loc[::13, "x"] = np.nan
        for keep in ("first", "last"):
            for ignore in (False, True):
                check(pdf, subset=["key"], keep=keep, ignore_index=ignore)
        check(pdf, subset="key")
    # sorted and reverse-sorted keys (runs already contiguous), and a shifted range index
    pdf = pandas.DataFrame({"key": np.repeat(np.arange(50), 7), "x": rng.standard_normal(350)})
    check(pdf, subset=["key"], keep="last")
    check(pdf.iloc[::-1].reset_index(drop=True), subset=["key"])
    shifted = pdf.copy()
    shifted.index = pandas.RangeIndex(1000, 1350)
    check(shifted, subset=["key"], keep="last")
    # labels that are already a device index column: the rows a filter left behind
    big = pandas.DataFrame({"key": rng.integers(0, 40, 2003), "x": rng.standard_normal(2003)})
    df = bpd.DataFrame(big)
    got = df[df["x"] > 0.0].drop_duplicates(subset=["key"])._to_pandas()
    want = big[big["x"] > 0.0].drop_duplicates(subset=["key"])
    assert list(got.index) == list(want.index) and _same(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64))
    # Series form, and a one-column frame with subset=None (= all columns)
    s, ws = df["key"].drop_duplicates()._to_pandas(), big["key"].drop_duplicates()
    assert list(s.index) == list(ws.index) and list(np.asarray(s).ravel()) == list(ws)
    check(big[["key"]])
    assert len(df.drop_duplicates(subset=["key"])) == big["key"].nunique() == df["key"].nunique()
    # the source frame is untouched; what is not on the path is refused with pandas' error types where it has one
    assert len(df) == len(big)
    with pytest.raises(NotImplementedError):
        df.drop_duplicates()  # all columns
    with pytest.raises(NotImplementedError):
        df.drop_duplicates(subset=["key", "x"])
    with pytest.raises(NotImplementedError):
        df.drop_duplicates(subset=["x"])  # float subset: NaN == NaN and -0.0 == 0.0 need their own handling
    with pytest.raises(NotImplementedError):
        df.drop_duplicates(subset=["key"], keep=False)
    with pytest.raises(KeyError):
        df.drop_duplicates(subset=["nope"])
    with pytest.raises(KeyError):
        big.drop_duplicates(subset=["nope"])
    with pytest.raises(ValueError):
        df.drop_duplicates(subset=["key"], keep="middle")


def test_block_set_axis_relabels_without_copying(cpu_device):
    """What real Modin's deferred label synchronisation applies to every partition (df.py:940-1030)."""
    from modin_b200.block import DeviceBlock

    pdf = pandas.DataFrame({"a": np.arange(5, dtype=np.float64), "b": np.arange(5, dtype=np.int64) * 3})
    blk = DeviceBlock.from_pandas(pdf)
    cols = blk.set_axis(pandas.Index(["x", "y"]), axis="columns")
    assert list(cols.columns) == ["x", "y"] and cols.cols[0] is blk.cols[0] and list(blk.columns) == ["a", "b"]
    assert blk.set_axis(pandas.RangeIndex(0, 5), axis="index") is blk  # nothing to do
    shifted = blk.set_axis(pandas.RangeIndex(10, 15), axis="index")
    assert shifted.has_range_index() and shifted.range_start == 10 and shifted.cols[1] is blk.cols[1]
    for labels in (pandas.Index([7, 3, 9, 1, 5]), pandas.Index([0.5, 1.5, 2.5, 3.5, 4.5], name="t"),
                   pandas.Index(list("vwxyz")), pandas.RangeIndex(0, 10, 2)):  # fmt: skip
        out = blk.set_axis(labels, axis=0)
        want = pdf.set_axis(labels, axis=0)
        got = out.to_pandas()
        assert got.index.equals(want.index) and got.index.name == want.index.name, labels
        assert _same(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64))
    with pytest.raises(ValueError):
        blk.set_axis(pandas.Index(["only"]), axis=1)
    with pytest.raises(ValueError):
        blk.set_axis(pandas.RangeIndex(4), axis=0)
    with pytest.raises(ValueError):
        blk.set_axis(pandas.RangeIndex(5), axis=2)


def test_pandas_method_on_a_block_is_a_clear_refusal(cpu_device):
    """A pandas lambda reaching a device block (an operation without a device functor) must say so -- and must not
    disturb attribute probing by numpy / torch / copy."""
    import copy

    from modin_b200.block import DeviceBlock, NotOnDevicePath

    blk = DeviceBlock.from_pandas(pandas.DataFrame({"a": [1.0, 2.0]}))
    with pytest.raises(NotImplementedError, match="no device implementation"):
        blk.cumsum(axis=0)
    with pytest.raises(AttributeError):
        blk.rolling
    assert issubclass(NotOnDevicePath, NotImplementedError) and issubclass(NotOnDevicePath, AttributeError)
    assert not hasattr(blk, "cumsum") and getattr(blk, "iloc", None) is None
    assert blk.squeeze(axis=1) is blk  # a one-column block is this package's Series (what Modin's broadcast branch asks)
    assert not hasattr(blk, "__array__") and not hasattr(blk, "__cuda_array_interface__")
    dup = copy.copy(blk)
    assert dup.nrows == 2 and dup.cols[0] is blk.cols[0] and list(dup.columns) == ["a"]
    assert np.asarray([[blk]], dtype=object).shape == (1, 1)  # still an opaque object to numpy, not a sequence


def test_series_surface(cpu_device):
    """A Series is a one-column frame: the whole surface against pandas -- values, row labels, NAME and dtype."""
    import modin_b200.pandas as bpd

    pa = synth.host_frame(1003, 3, seed=1, nan_per_64k=3000, key_modulus=11)
    d = bpd.DataFrame(pa)
    s, ws, k, wk = d["c0"], pa["c0"], d["key"], pa["key"]
    assert s.name == "c0" and len(s) == len(ws) and s.dtype == ws.dtype and k.dtype == wk.dtype
    series_cases = {
        "abs": (lambda: s.abs(), lambda: ws.abs()), "neg": (lambda: -s, lambda: -ws), "round": (lambda: s.round(1), lambda: ws.round(1)),
        "clip": (lambda: s.clip(-0.5, 0.5), lambda: ws.clip(-0.5, 0.5)), "fillna": (lambda: s.fillna(0.0), lambda: ws.fillna(0.0)),
        "isna": (lambda: s.isna(), lambda: ws.isna()), "affine": (lambda: s * 2.0 + 1.0, lambda: ws * 2.0 + 1.0),
        "reflected": (lambda: 2.0 - s, lambda: 2.0 - ws), "series / series": (lambda: s / d["c1"], lambda: ws / pa["c1"]),
        "comparison": (lambda: s > 0.0, lambda: ws > 0.0), "series > series": (lambda: s > d["c1"], lambda: ws > pa["c1"]),
        "mask and": (lambda: (s > 0.0) & (d["c1"] < 0.0), lambda: (ws > 0.0) & (pa["c1"] < 0.0)), "mask not": (lambda: ~(s > 0.0), lambda: ~(ws > 0.0)),
        "s[mask]": (lambda: s[s > 0.0], lambda: ws[ws > 0.0]), "dropna": (lambda: s.dropna(), lambda: ws.dropna()),
        "head": (lambda: s.head(7), lambda: ws.head(7)), "tail": (lambda: s.tail(7), lambda: ws.tail(7)), "copy": (lambda: s.copy(), lambda: ws.copy()),
        "sort_values": (lambda: s.sort_values(), lambda: ws.sort_values(kind="stable")),
        "sort_values descending": (lambda: s.sort_values(ascending=False), lambda: ws.sort_values(ascending=False, kind="stable")),
        "rename": (lambda: s.rename("zz"), lambda: ws.rename("zz")), "rename(None)": (lambda: s.rename(None), lambda: ws.rename(None)),
        "astype": (lambda: k.astype("float64"), lambda: wk.astype("float64")), "isin": (lambda: k.isin([1, 2]), lambda: wk.isin([1, 2])),
        "drop_duplicates": (lambda: k.drop_duplicates(), lambda: wk.drop_duplicates()),
        "drop_duplicates last": (lambda: k.drop_duplicates(keep="last"), lambda: wk.drop_duplicates(keep="last")),
        "int == int": (lambda: k == 3, lambda: wk == 3), "int > float": (lambda: k > 2.5, lambda: wk > 2.5), "int * 2": (lambda: k * 2, lambda: wk * 2),
    }  # fmt: skip
    for name, (dev, host) in series_cases.items():
        got, want = dev(), host()
        assert isinstance(got, bpd.Series), name
        g = got._to_pandas()
        assert g.name == want.name and g.dtype == want.dtype and list(g.index) == list(want.index), name
        assert _same(g.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64)), name
    scalar_cases = {
        "sum": (lambda: s.sum(), lambda: ws.sum()), "mean": (lambda: s.mean(), lambda: ws.mean()), "min": (lambda: s.min(), lambda: ws.min()),
        "max": (lambda: s.max(), lambda: ws.max()), "count": (lambda: s.count(), lambda: ws.count()), "var": (lambda: s.var(), lambda: ws.var()),
        "std": (lambda: s.std(), lambda: ws.std()), "prod": (lambda: s.head(20).prod(), lambda: ws.head(20).prod()),
        "sum skipna=False": (lambda: s.sum(skipna=False), lambda: ws.sum(skipna=False)), "nunique": (lambda: k.nunique(), lambda: wk.nunique()),
        "mask sum": (lambda: (s > 0.0).sum(), lambda: (ws > 0.0).sum()), "mask any": (lambda: (s > 0.0).any(), lambda: (ws > 0.0).any()),
        "mask all": (lambda: (s > -100.0).all(), lambda: (ws > -100.0).all()), "mask mean": (lambda: (s > 0.0).mean(), lambda: (ws > 0.0).mean()),
        "int sum": (lambda: k.sum(), lambda: wk.sum()), "int min": (lambda: k.min(), lambda: wk.min()), "int mean": (lambda: k.mean(), lambda: wk.mean()),
    }  # fmt: skip
    for name, (dev, host) in scalar_cases.items():
        g, want = dev(), host()
        assert np.ndim(g) == 0, name
        assert (np.isnan(g) and np.isnan(want)) or np.isclose(g, want, rtol=1e-12, atol=1e-9), (name, g, want)
    for refused in (lambda: s[0], lambda: s.dropna(inplace=True), lambda: s.rename({0: 1}), lambda: s.sort_values(inplace=True)):
        with pytest.raises(NotImplementedError):
            refused()


def test_isin_is_a_join_probe(cpu_device):
    import modin_b200.pandas as bpd

    pdf = synth.host_frame(2003, 2, seed=5, key_modulus=50)
    pdf["k2"] = synth.gen_i64(2003, 3, 1, 9) - 4
    df = bpd.DataFrame(pdf)
    vals = [3, 7, 7, 41, -2, 1000]
    got = df[["key", "k2"]].isin(vals)._to_pandas()
    want = pdf[["key", "k2"]].isin(vals)
    assert _same(got.to_numpy().astype(float), want.to_numpy().astype(float))
    sel = df[df["key"].isin([1, 2, 3])]._to_pandas()
    w = pdf[pdf["key"].isin([1, 2, 3])]
    assert list(sel.index) == list(w.index) and _same(sel.to_numpy(dtype=np.float64), w.to_numpy(dtype=np.float64))
    assert not df["key"].isin([])._to_pandas().any()
    with pytest.raises(NotImplementedError):
        df[["c0"]].isin([1])
    with pytest.raises(NotImplementedError):
        df["key"].isin([1.5])


def test_late_gpu_tests_are_sound_on_the_double(cpu_device, golden_dir):
    """tests/test_zz_gpu_row_selection.py could not be run on a GPU in the round it was written; run its bodies on
    the device double so that at least the test logic (and the host side it drives) is known to be right."""
    import importlib.util
    import os

    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_zz_gpu_row_selection.py")
    spec = importlib.util.spec_from_file_location("late_gpu_tests", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.test_boolean_row_selection_and_dropna_on_device()
    mod.test_pipeline_filter_derive_aggregate_on_device()
    mod.test_isin_is_a_join_probe_on_device()
    mod.test_baseline_config0_abs_and_sum_at_its_own_size()
    mod.test_concat_on_device()
    mod.test_astype_and_frame_nunique_on_device()
    mod.test_second_batch_vs_reference_golden(golden_dir)
    mod.test_third_batch_vs_reference_golden(golden_dir)


def test_round1_advisor_findings_stay_fixed(cpu_device):
    """The advisor's round-1 reproductions (ADVICE.md): label-blind pairing in setitem / concat / mask / by-Series,
    FMA3 fusion on non-float64 operands, dtype of a fused affine on an empty frame, int64 overflow in the multi-key
    packing, dtype disagreement between the row partitions of a left merge with int64 payload."""
    import modin_b200.pandas as bpd

    old = config.NPartitions.get()
    config.NPartitions.put(2)
    try:
        df = pandas.DataFrame({"a": [3.0, 1.0, 2.0, 5.0, 4.0], "b": [1.0, 2.0, 3.0, 4.0, 5.0]})
        m = bpd.DataFrame(df)
        m["d"] = m["a"].sort_values()  # pandas realigns by label: d == a
        want = df.copy()
        want["d"] = df["a"].sort_values()
        assert m._to_pandas().equals(want)
        x = pandas.DataFrame({"p": [1.0, 2.0, 3.0]}, index=[10, 11, 12])
        y = pandas.DataFrame({"q": [7.0, 8.0, 9.0]}, index=[12, 11, 10])
        assert bpd.concat([bpd.DataFrame(x), bpd.DataFrame(y)], axis=1)._to_pandas().equals(pandas.concat([x, y], axis=1))
        mask = pandas.Series([True, True, False, False, False], index=[3, 4, 0, 1, 2])
        got = m[bpd.Series(mask)]._to_pandas()
        assert list(got.index) == [3, 4]
        keys = pandas.Series(np.array([0, 0, 1, 1, 1], dtype=np.int64), index=[4, 3, 2, 1, 0], name="k")
        got = bpd.DataFrame(df).groupby(bpd.Series(keys)).sum()._to_pandas()
        assert _same(got.to_numpy(), df.groupby(keys).sum().to_numpy())
        # fusion only where the fused kernel is valid
        ip = pandas.DataFrame({"a": np.arange(10, dtype=np.int64), "b": np.arange(10, dtype=np.int64) * 3})
        fp = pandas.DataFrame({"a": np.arange(10) * 0.5, "b": np.arange(10) * 1.5})
        ia, fa = bpd.DataFrame(ip), bpd.DataFrame(fp)
        assert (ia * ia + ia)._to_pandas().equals(ip * ip + ip)
        assert (fa * ia + fa)._to_pandas().equals(fp * ip + fp)
        empty = (ia[ia["a"] > 50] * 2 + 1.5)._to_pandas()
        assert list(empty.dtypes) == list((ip[ip["a"] > 50] * 2 + 1.5).dtypes) and empty.shape == (0, 2)
        # multi-key packing with timestamp-sized keys
        rng = np.random.RandomState(0)
        ts = (1_700_000_000_000_000_000 + rng.randint(0, 50, 3000)).astype(np.int64)
        pdf = pandas.DataFrame({"ts": ts, "k2": rng.randint(0, 5001, 3000).astype(np.int64), "v": rng.randn(3000)})
        got = bpd.DataFrame(pdf).groupby(["ts", "k2"]).sum()._to_pandas()
        w = pdf.groupby(["ts", "k2"]).sum()
        assert got.index.equals(w.index) and np.allclose(got.to_numpy(), w.to_numpy())
        # left merge, int64 payload: misses only in the SECOND row partition -> every partition must still be float64
        fact = pandas.DataFrame({"key": np.array([0, 1, 2, 3, 4, 9], dtype=np.int64), "v": np.arange(6) * 1.0})
        dim = pandas.DataFrame({"key": np.arange(5, dtype=np.int64), "tag": np.arange(5, dtype=np.int64) * 10})
        res = bpd.DataFrame(fact).merge(bpd.DataFrame(dim), on="key", how="left")
        dts = {str(p.get().dtypes["tag"]) for p in res._query_compiler._modin_frame._partitions[:, 0]}
        assert dts == {"float64"}
        assert _same(res._to_pandas().to_numpy(dtype=np.float64), fact.merge(dim, on="key", how="left").to_numpy(dtype=np.float64))
    finally:
        config.NPartitions.put(old)


def test_pandas3_shims_accept_only_the_removed_defaults():
    from modin_b200.modin_plugin import apply_pandas3_shims

    apply_pandas3_shims()
    d = pandas.DataFrame({"a": [1.0, None], "b": [1.0, 2.0]})
    assert d.fillna(0.0, method=None, downcast=None)["a"].tolist() == [1.0, 0.0]
    assert len(d.groupby("b", axis=0)) == 2
    with pytest.raises(TypeError):
        d.groupby("b", axis=1)
    with pytest.raises(TypeError):
        d.fillna(method="ffill")
