"""GPU parity tests (``-m gpu``): the B200 execution, driven through its public pandas-style API
(modin_b200.pandas -> query compiler -> templates -> partitions -> C ABI -> sm_90a kernels),
against (1) the golden vectors produced by the unmodified reference and (2) the CPU oracle on
fresh seeded inputs.

Tolerances (SURVEY.md §8d): elementwise / predicates / min / max / count / size / keys / merge are
BIT-EXACT (NaN == NaN); float sums and means satisfy
``|got - ref| <= 4 * log2(n) * 2**-53 * sum|x|`` per output value.
"""

import glob
import os

import numpy as np
import pandas
import pytest

from modin_b200 import synth
from oracle import reference_path as orc
from tests.exact import EPS, assert_exact, assert_sum_close, assert_within_sum_bound, exact_group_sums

pytestmark = pytest.mark.gpu


def bpd():
    import modin_b200.pandas as m

    return m


@pytest.fixture(autouse=True)
def _four_partitions():
    """The reference's own tests force NPartitions=4 (modin/tests/pandas/dataframe/test_reduce.py:41)."""
    from modin_b200 import config

    old = config.NPartitions.get()
    config.NPartitions.put(4)
    yield
    config.NPartitions.put(old)


@pytest.fixture(params=["dense", "dense_global_atomics", "hash"])
def gb_table_kind(request):
    """Run a groupby test with the direct-addressed table (narrow key range; small ranges are privatised in
    shared memory), with the same table but global atomics only, and with the hash table."""
    from modin_b200 import config

    old = config.GroupbyDenseKeys.get()
    config.GroupbyDenseKeys.put(request.param != "hash")
    if request.param == "dense_global_atomics":
        os.environ["MB200_GB_SMEM"] = "0"
    yield request.param
    os.environ.pop("MB200_GB_SMEM", None)
    config.GroupbyDenseKeys.put(old)


def _load(golden_dir, pattern):
    files = sorted(glob.glob(os.path.join(golden_dir, pattern)))
    assert files
    return [(os.path.basename(f), np.load(f, allow_pickle=False)) for f in files]


# ---------------------------------------------------------------------------------------------
def test_device_generators_match_numpy_twin():
    from modin_b200 import ops

    for n, off in ((1, 0), (1000, 0), (4097, 12345)):
        a = ops.gen_f64(n, 42, 3, off, 1000).to_numpy()
        assert_exact(a, synth.gen_f64(n, 42, 3, off, 1000), f"gen_f64 n={n}")
        k = ops.gen_i64(n, 43, 0, 1000, off).to_numpy()
        assert np.array_equal(k, synth.gen_i64(n, 43, 0, 1000, off))


def test_map_binary_vs_reference_golden(golden_dir):
    m = bpd()
    for name, z in [(n, z) for n, z in _load(golden_dir, "frame_*.npz") if not n.endswith("_fma3.npz")]:
        n, W, seed, nan = (int(x) for x in z["meta"])
        pdf = synth.host_frame(n, W, seed=seed, nan_per_64k=nan)
        df = m.DataFrame(pdf)
        assert_exact(df.abs()._to_pandas().to_numpy(), z["abs"], f"{name}:abs")
        assert_exact((-df)._to_pandas().to_numpy(), z["neg"], f"{name}:neg")
        assert_exact(df.isna()._to_pandas().to_numpy(), z["isna"], f"{name}:isna")
        assert_exact(df.fillna(1.5)._to_pandas().to_numpy(), z["fillna"], f"{name}:fillna")
        assert_exact((df * 1.25 + 0.5)._to_pandas().to_numpy(), z["affine"], f"{name}:affine (fused)")
        mul = list(np.arange(1, W + 1) * 0.5)
        add = list(np.arange(W) * 0.25)
        assert_exact((df * mul + add)._to_pandas().to_numpy(), z["rowvec"], f"{name}:row-vector affine")
        assert_exact((df < 0.0)._to_pandas().to_numpy(), z["lt0"], f"{name}:lt0")


def test_three_frame_fma_vs_reference_golden(golden_dir):
    m = bpd()
    for name, z in _load(golden_dir, "frame_*_fma3.npz"):
        n, W, seed, nan, sb, sc = (int(x) for x in z["meta"])
        a = m.DataFrame(synth.host_frame(n, W, seed=seed, nan_per_64k=nan))
        b = m.DataFrame(synth.host_frame(n, W, seed=sb))
        c = m.DataFrame(synth.host_frame(n, W, seed=sc))
        assert_exact((a * b + c)._to_pandas().to_numpy(), z["out"], f"{name}:a*b+c (fused, two roundings)")
        assert_exact((a - b)._to_pandas().to_numpy(), z["sub"], f"{name}:sub")
        assert_exact((a / b)._to_pandas().to_numpy(), z["div"], f"{name}:div")
        assert_exact((a >= b)._to_pandas().to_numpy(), z["ge"], f"{name}:ge")


def test_tree_reduce_vs_reference_golden(golden_dir):
    m = bpd()
    for name, z in [(n, z) for n, z in _load(golden_dir, "frame_*.npz") if not n.endswith("_fma3.npz")]:
        n, W, seed, nan = (int(x) for x in z["meta"])
        pdf = synth.host_frame(n, W, seed=seed, nan_per_64k=nan)
        abs_sums = np.nansum(np.abs(pdf.to_numpy()), axis=0)
        df = m.DataFrame(pdf)
        assert_sum_close(df.sum().to_numpy(), z["sum"], abs_sums, n, f"{name}:sum")
        assert_sum_close(df.sum(skipna=False).to_numpy(), z["sum_noskip"], abs_sums, n, f"{name}:sum skipna=False")
        assert_sum_close(df.sum(min_count=1).to_numpy(), z["sum_mc1"], abs_sums, n, f"{name}:sum min_count=1")
        cnt = np.maximum(z["count"], 1)
        assert_sum_close(df.mean().to_numpy(), z["mean"], abs_sums / cnt, n, f"{name}:mean")
        assert_exact(df.min().to_numpy(), z["min"], f"{name}:min")
        assert_exact(df.max().to_numpy(), z["max"], f"{name}:max")
        assert_exact(df.count().to_numpy(), z["count"], f"{name}:count")
        assert df.count().dtype == np.int64


def test_groupby_vs_reference_golden(golden_dir, gb_table_kind):
    m = bpd()
    for name, z in _load(golden_dir, "groupby_*.npz"):
        n, G, V, nan, seed, kseed = (int(x) for x in z["meta"])
        pdf = synth.host_frame(n, V, seed=seed, nan_per_64k=nan, key_modulus=G, key_seed=kseed)
        df = m.DataFrame(pdf)
        g = df.groupby("key")
        s = g.sum()._to_pandas()
        assert_exact(s.index.to_numpy(), z["keys"], f"{name}:keys sorted")
        assert s.index.name == "key" and list(s.columns) == [f"c{i}" for i in range(V)]
        abs_by_group = pdf.drop(columns="key").abs().groupby(pdf["key"]).sum().to_numpy()
        assert_sum_close(s.to_numpy(), z["sum"], abs_by_group, n, f"{name}:sum")
        assert_exact(g.count()._to_pandas().to_numpy(), z["count"], f"{name}:count")
        assert_exact(g.size()._to_pandas().to_numpy(), z["size"], f"{name}:size")
        cnt = np.maximum(z["count"], 1)
        assert_sum_close(g.mean()._to_pandas().to_numpy(), z["mean"], abs_by_group / cnt, n, f"{name}:mean")


@pytest.fixture(params=["dense", "hash"])
def join_table_kind(request):
    """Dim keys in a narrow range get a direct-addressed table; MB200_JOIN_DENSE=0 forces the hash table."""
    if request.param == "hash":
        os.environ["MB200_JOIN_DENSE"] = "0"
    yield request.param
    os.environ.pop("MB200_JOIN_DENSE", None)


def test_merge_vs_reference_golden(golden_dir, join_table_kind):
    m = bpd()
    for name, z in _load(golden_dir, "merge_*.npz"):
        n, nd, hit = (int(x) for x in z["meta"])
        fact = synth.host_frame(n, 3, seed=42, key_modulus=nd, key_seed=43)
        dim_keys = z["dim_keys"]
        dim = pandas.DataFrame({"key": dim_keys, "d0": synth.gen_f64(len(dim_keys), 11, 0),
                                "d1": np.arange(len(dim_keys), dtype=np.int64) * 3})  # fmt: skip
        left = m.DataFrame(fact).merge(m.DataFrame(dim), on="key", how="left")._to_pandas()
        assert list(left.columns) == [str(c) for c in z["left_cols"]]
        assert_exact(left.to_numpy(dtype=np.float64), z["left"], f"{name}:left")
        assert isinstance(left.index, pandas.RangeIndex) and len(left) == n
        inner = m.DataFrame(fact).merge(m.DataFrame(dim), on="key", how="inner")._to_pandas()
        assert_exact(inner.to_numpy(dtype=np.float64), z["inner"], f"{name}:inner")


# ------------------------------------------------------------------ fresh inputs vs the oracle
@pytest.mark.parametrize("n,W,nan", [(1, 1, 0), (31, 3, 0), (33, 2, 30000), (100003, 8, 500), (262144, 16, 0)])
def test_against_oracle_various_shapes(n, W, nan):
    m = bpd()
    pdf = synth.host_frame(n, W, seed=5, nan_per_64k=nan)
    df = m.DataFrame(pdf)
    NPART = 4
    assert_exact(df.abs()._to_pandas().to_numpy(), orc.df_abs(pdf, NPART).to_numpy(), "abs")
    assert_exact((df * 0.75 + 2.0)._to_pandas().to_numpy(), orc.a_mul_b_add_c(pdf, 0.75, 2.0, NPART).to_numpy(), "affine")
    abs_sums = np.nansum(np.abs(pdf.to_numpy()), axis=0)
    assert_sum_close(df.sum().to_numpy(), orc.df_sum(pdf, NPART).to_numpy(), abs_sums, n, "sum")
    assert_exact(df.count().to_numpy(), orc.df_count(pdf, NPART).to_numpy(), "count")
    assert_exact(df.min().to_numpy(), orc.df_min(pdf, NPART).to_numpy(), "min")
    assert_exact(df.max().to_numpy(), orc.df_max(pdf, NPART).to_numpy(), "max")


def test_groupby_min_max_bit_exact(gb_table_kind):
    """storage_formats/pandas/groupby.py:237-248: min -> (min, min), max -> (max, max); no rounding involved."""
    m = bpd()
    pdf = synth.host_frame(30011, 3, seed=13, nan_per_64k=20000, key_modulus=977)
    pdf.loc[pdf["key"] == 5, "c1"] = np.nan  # an all-NaN group -> NaN
    pdf.loc[3, "c2"] = np.inf
    pdf.loc[4, "c2"] = -np.inf
    g = m.DataFrame(pdf).groupby("key")
    for agg in ("min", "max"):
        got = getattr(g, agg)()._to_pandas()
        want = orc.groupby_reduce(pdf, "key", agg, 4)
        assert_exact(got.index.to_numpy(), want.index.to_numpy(), f"{agg} keys")
        assert_exact(got.to_numpy(), want.to_numpy(), f"groupby {agg}")


def test_prod_tree_reduce():
    m = bpd()
    pdf = synth.host_frame(300, 4, seed=21, nan_per_64k=3000) * 1.7
    got = m.DataFrame(pdf).prod().to_numpy()
    want = orc.df_prod(pdf, 4).to_numpy()
    assert np.allclose(got, want, rtol=1e-12, atol=0)
    ints = pandas.DataFrame({"a": np.arange(1, 21, dtype=np.int64), "b": np.full(20, -2, dtype=np.int64)})
    assert_exact(m.DataFrame(ints).prod().to_numpy(), ints.prod().to_numpy(), "int64 prod (wrapping, exact)")


def test_series_column_vector_broadcast():
    m = bpd()
    pdf = synth.host_frame(5000, 3, seed=6)
    df = m.DataFrame(pdf)
    assert_exact(df.mul(df["c1"], axis=0)._to_pandas().to_numpy(), pdf.mul(pdf["c1"], axis=0).to_numpy(), "mul axis=0")
    assert_exact(df.rsub(df["c2"], axis=0)._to_pandas().to_numpy(), pdf.rsub(pdf["c2"], axis=0).to_numpy(), "rsub axis=0")


def test_reduce_variants_agree():
    """TMA-staged and direct-load reductions are two schedules of the same arithmetic."""
    from modin_b200 import config

    m = bpd()
    pdf = synth.host_frame(300007, 5, seed=9, nan_per_64k=100)
    abs_sums = np.nansum(np.abs(pdf.to_numpy()), axis=0)
    res = []
    for v in (0, 1):
        config.ReduceVariant.put(v)
        res.append(m.DataFrame(pdf).sum().to_numpy())
    config.ReduceVariant.put(0)
    assert_sum_close(res[0], res[1], abs_sums, len(pdf), "variants")


def test_int64_columns_are_exact():
    m = bpd()
    rng = np.random.RandomState(3)
    pdf = pandas.DataFrame({"a": rng.randint(-10**12, 10**12, 70001), "b": rng.randint(-5, 5, 70001)}).astype("int64")
    df = m.DataFrame(pdf)
    assert_exact(df.sum().to_numpy(), pdf.sum().to_numpy(), "int sum")
    assert_exact(df.min().to_numpy(), pdf.min().to_numpy(), "int min")
    assert_exact(df.abs()._to_pandas().to_numpy(), pdf.abs().to_numpy(), "int abs")
    assert_exact((df * 3 + 1)._to_pandas().to_numpy(), (pdf * 3 + 1).to_numpy(), "int affine (unfused)")
    assert_exact((df == 0)._to_pandas().to_numpy(), (pdf == 0).to_numpy(), "int eq")


def test_edge_cases_and_errors():
    m = bpd()
    # all-NaN column, +-inf, -0.0
    pdf = pandas.DataFrame({"a": [np.nan, np.nan, np.nan], "b": [np.inf, 1.0, -0.0], "c": [-np.inf, np.inf, 2.0]})
    df = m.DataFrame(pdf)
    # The truth is the REFERENCE (restated by the oracle), not plain pandas: Modin's tree reduce returns 0.0 for
    # the sum of [-inf, inf, 2.0] (the NaN partial of the map phase is skipped by the skipna reduce phase) where
    # pandas returns NaN -- checked against the unmodified reference in the build container.
    assert_exact(df.sum().to_numpy(), orc.df_sum(pdf, 4).to_numpy(), "sum with inf / all-NaN")
    assert_exact(df.sum().to_numpy(), np.array([0.0, np.inf, 0.0]), "sum quirk reproduced")
    assert_exact(df.sum(min_count=1).to_numpy(), orc.df_sum(pdf, 4, min_count=1).to_numpy(), "min_count=1 all-NaN -> NaN")
    assert_exact(df.mean().to_numpy(), orc.df_mean(pdf, 4).to_numpy(), "mean with inf / all-NaN")
    assert_exact(df.min().to_numpy(), orc.df_min(pdf, 4).to_numpy(), "min all-NaN -> NaN")
    assert_exact(df.max(skipna=False).to_numpy(), orc.df_max(pdf, 4, skipna=False).to_numpy(), "max skipna=False")
    assert_exact(df.abs()._to_pandas().to_numpy(), pdf.abs().to_numpy(), "abs(-0.0) = +0.0")
    # errors surface like pandas / the reference does
    with pytest.raises(ValueError):
        df.fillna()
    with pytest.raises(KeyError):
        df.groupby("nope")
    with pytest.raises(TypeError):
        m.DataFrame(pandas.DataFrame({"s": ["x", "y"]}))
    with pytest.raises(NotImplementedError):
        df.merge(df, how="outer", on="a")


def test_groupby_with_empty_and_skewed_partitions(gb_table_kind):
    """cf. test_groupby_with_empty_partition (modin/tests/core/storage_formats/pandas/test_internals.py:863)."""
    m = bpd()
    n = 9001
    keys = np.zeros(n, dtype=np.int64)
    keys[-3:] = [7, 7, -2]  # one giant group + tiny ones, all in the last partition
    pdf = pandas.DataFrame({"key": keys, "v": synth.gen_f64(n, 1, 0)})
    got = m.DataFrame(pdf).groupby("key").sum()._to_pandas()
    want = orc.groupby_reduce(pdf, "key", "sum", 4)
    assert_exact(got.index.to_numpy(), want.index.to_numpy(), "keys")
    assert_sum_close(got.to_numpy(), want.to_numpy(), pdf["v"].abs().groupby(pdf["key"]).sum().to_numpy()[:, None], n, "sum")


def test_groups_whose_rows_leave_no_trace_are_still_groups(gb_table_kind):
    """Dense tables infer presence from the accumulators; rows that change nothing (all values NaN or -0.0)
    must still create their group: sum 0.0 / count 0 / min, max NaN (or -0.0) exactly as pandas."""
    m = bpd()
    n = 4096 + 37
    pdf = synth.host_frame(n, 3, seed=17, nan_per_64k=3000, key_modulus=10)
    pdf.loc[pdf["key"] == 3, ["c0", "c1", "c2"]] = np.nan
    pdf.loc[pdf["key"] == 5, ["c0", "c1", "c2"]] = -0.0
    pdf.loc[pdf["key"] == 7, ["c0", "c2"]] = np.nan
    pdf.loc[pdf["key"] == 7, "c1"] = -0.0
    pdf["key"] = pdf["key"] * 3 - 9  # gaps in the range: absent keys must stay absent
    g = m.DataFrame(pdf).groupby("key")
    for agg in ("sum", "count", "size", "min", "max", "mean"):
        got = getattr(g, agg)()._to_pandas()
        want = orc.groupby_reduce(pdf, "key", agg, 4)
        assert_exact(got.index.to_numpy(), want.index.to_numpy(), f"{agg} keys")
        w = want.to_numpy(dtype=np.float64).reshape(len(want), -1)
        gt = got.to_numpy(dtype=np.float64).reshape(len(got), -1)
        if agg == "sum":
            keys, exact = exact_group_sums(pdf["key"].to_numpy(), pdf[["c0", "c1", "c2"]].to_numpy())
            assert_exact(keys, want.index.to_numpy(), "exact reference keys")
            abs_by_group = pdf[["c0", "c1", "c2"]].abs().groupby(pdf["key"]).sum().to_numpy()
            assert_within_sum_bound(gt, exact, abs_by_group, n, "groupby sum vs exact")
            assert_exact(gt[np.isin(want.index.to_numpy(), [0, 6, 12])], w[np.isin(want.index.to_numpy(), [0, 6, 12])],
                         "all-NaN / all -0.0 groups sum to +0.0")  # fmt: skip
        elif agg == "mean":
            assert np.allclose(gt, w, rtol=0, atol=1e-9, equal_nan=True), agg
        else:
            assert_exact(gt, w, f"groupby {agg}")


def test_merge_with_wide_and_negative_dim_keys():
    """Dim keys spread over a wide range fall back to the hash table; a narrow range with a negative base and
    fact keys outside it exercise the dense table's bounds check.  Both against the oracle, bit for bit."""
    m = bpd()
    n, nd = 20011, 500
    rng = np.random.RandomState(3)
    for scale, shift in ((1, -250), (1_000_003_019, -250)):
        fact = synth.host_frame(n, 2, seed=42, key_modulus=nd + 80, key_seed=43)  # keys >= nd miss the dim
        fact["key"] = (fact["key"] + shift) * scale
        dk = ((rng.permutation(nd)[: nd - 37]).astype(np.int64) + shift) * scale
        dim = pandas.DataFrame({"key": dk, "d0": synth.gen_f64(len(dk), 11, 0), "d1": np.arange(len(dk), dtype=np.int64)})
        for how in ("left", "inner"):
            got = m.DataFrame(fact).merge(m.DataFrame(dim), on="key", how=how)._to_pandas()
            want = orc.broadcast_merge(fact, dim, "key", how, 4)
            assert list(got.columns) == list(want.columns)
            assert_exact(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64), f"merge {how} scale={scale}")


def test_skewed_keys_take_the_hot_group_cache_and_match_the_oracle(gb_table_kind):
    """Zipf-like keys (SURVEY 8d skew variant): the key pre-pass must flag them, the accumulate kernel then
    caches hot groups per CTA in shared memory -- same results as the oracle either way."""
    from modin_b200 import ops
    from modin_b200.block import DeviceColumn

    m = bpd()
    n, G = 200_003, 50_000
    for nn, off in ((1000, 0), (4097, 12345)):
        assert np.array_equal(ops.gen_i64(nn, 43, 0, G, off, skew=True).to_numpy(), synth.gen_i64_skew(nn, 43, 0, G, off))
    pdf = synth.host_frame(n, 3, seed=23, nan_per_64k=700, key_modulus=G, key_skew=True)
    assert (pdf["key"] == 0).mean() > 0.08  # a heavy hitter
    lo, hi, sampled, dup = (int(v) for v in ops.key_range_device([DeviceColumn.from_numpy(pdf["key"].to_numpy())]).tolist())
    assert (lo, hi) == (int(pdf["key"].min()), int(pdf["key"].max())) and ops.keys_are_skewed(sampled, dup)
    uni = synth.gen_i64(n, 43, 0, G)
    assert not ops.keys_are_skewed(*(int(v) for v in ops.key_range_device([DeviceColumn.from_numpy(uni)]).tolist()[2:]))
    g = m.DataFrame(pdf).groupby("key")
    abs_by_group = pdf.drop(columns="key").abs().groupby(pdf["key"]).sum().to_numpy()
    for agg in ("sum", "count", "mean", "size", "max"):
        got = getattr(g, agg)()._to_pandas()
        want = orc.groupby_reduce(pdf, "key", agg, 4)
        assert_exact(got.index.to_numpy(), want.index.to_numpy(), f"{agg} keys")
        w = want.to_numpy(dtype=np.float64).reshape(len(want), -1)
        gt = got.to_numpy(dtype=np.float64).reshape(len(got), -1)
        if agg == "sum":
            assert_sum_close(gt, w, abs_by_group, n, "skewed sum")
        elif agg == "mean":
            cnt = np.maximum(orc.groupby_reduce(pdf, "key", "count", 4).to_numpy(), 1)
            assert_sum_close(gt, w, abs_by_group / cnt, n, "skewed mean")
        else:
            assert_exact(gt, w, f"skewed {agg}")


def test_dense_and_hash_tables_agree_and_wide_keys_fall_back():
    """The dense table is chosen from the measured key range; keys spread over a wide range must take the
    hash table and give the same groups.  Counts / sizes / keys / min / max are bit-identical either way."""
    from modin_b200 import config, ops

    m = bpd()
    n = 50021
    base = synth.host_frame(n, 3, seed=21, nan_per_64k=9000, key_modulus=613)
    wide = base.copy()
    wide["key"] = (base["key"] - 300) * 1_000_003_019  # same grouping, range ~6e11: not dense-able
    assert ops.dense_range_ok(0, 612, 1024, n, 3, 1) and not ops.dense_range_ok(int(wide["key"].min()), int(wide["key"].max()), 1 << 20, n, 3, 1)
    res = {}
    for kind, pdf in (("dense", base), ("hash", wide)):
        g = m.DataFrame(pdf).groupby("key")
        res[kind] = {a: getattr(g, a)()._to_pandas() for a in ("sum", "count", "size", "min", "max", "mean")}
    want_keys = np.sort(base["key"].unique())
    assert_exact(res["dense"]["sum"].index.to_numpy(), want_keys, "dense keys")
    assert_exact(res["hash"]["sum"].index.to_numpy(), (want_keys - 300) * 1_000_003_019, "wide keys")
    for a in ("count", "size", "min", "max"):
        assert_exact(res["dense"][a].to_numpy(), res["hash"][a].to_numpy(), f"dense vs hash {a}")
    abs_by_group = base.drop(columns="key").abs().groupby(base["key"]).sum().to_numpy()
    assert_sum_close(res["dense"]["sum"].to_numpy(), res["hash"]["sum"].to_numpy(), abs_by_group, n, "dense vs hash sum")
    # ops level: key range kernel, negative base, ragged lengths
    for nn in (1, 15, 16, 17, 4099, 100000):
        kk = synth.gen_i64(nn, 7, 0, 1000) - 500
        from modin_b200.block import DeviceColumn
        assert ops.key_range([DeviceColumn.from_numpy(kk)]) == (int(kk.min()), int(kk.max()))
    assert config.GroupbyDenseKeys.get()


def test_large_scale_invariants(gb_table_kind):
    """Properties that do not need a CPU pass over the data (SURVEY.md §8d "parity at scale")."""
    m = bpd()
    from modin_b200 import config

    config.NPartitions.put(2)
    n, W, G = 1 << 24, 8, 100_000
    df = synth.device_frame(n, W, key_modulus=G, npartitions=2)
    vals = df[[f"c{i}" for i in range(W)]]
    col_sum = vals.sum().to_numpy()
    col_abs = vals.abs().sum().to_numpy()
    g = df.groupby("key")
    gs = g.sum()._to_pandas()
    assert len(gs) == G and gs.index.is_monotonic_increasing and gs.index[0] == 0 and gs.index[-1] == G - 1
    assert_sum_close(gs.sum().to_numpy(), col_sum, col_abs, n, "sum of group sums == column sums")
    sz = g.size()._to_pandas()
    assert int(sz.sum()) == n
    # sampled elementwise equality against the numpy twin of the generator
    out = (vals * 1.5 + 0.25)._to_pandas()
    rows = np.array([0, 1, 4095, 4096, n // 2, n - 1])
    for j in range(W):
        ref = np.array([synth.gen_f64(1, 42, j, int(r))[0] for r in rows]) * 1.5 + 0.25
        assert_exact(out.iloc[rows, j].to_numpy(), ref, f"sampled affine col {j}")
    mean = vals.mean().to_numpy()
    assert np.all(np.abs(mean - col_sum / n) <= 1e-15 + 4 * EPS * col_abs / n)


def test_more_registrations_vs_reference_golden(golden_dir):
    """SURVEY 8f-3: round / clip (bit-exact), var / std (two device passes; relative 1e-12 against the reference's
    two-pass nanvar), prod, groupby min / max (bit-exact) -- golden vectors from the unmodified reference."""
    m = bpd()
    for name, z in _load(golden_dir, "ext_n*.npz"):
        n, W, seed, nan = (int(x) for x in z["meta"])
        pdf = synth.host_frame(n, W, seed=seed, nan_per_64k=nan)
        df = m.DataFrame(pdf)
        assert_exact(df.round(2)._to_pandas().to_numpy(), z["round2"], f"{name}:round(2)")
        assert_exact(df.round(0)._to_pandas().to_numpy(), z["round0"], f"{name}:round(0)")
        assert_exact((df * 100.0).round(-1)._to_pandas().to_numpy(), z["round_m1"], f"{name}:round(-1)")
        assert_exact(df.clip(-0.5, 0.75)._to_pandas().to_numpy(), z["clip"], f"{name}:clip")
        assert_exact(df.clip(lower=0.0)._to_pandas().to_numpy(), z["clip_lower"], f"{name}:clip lower")
        for got, key in ((df.var(), "var"), (df.var(ddof=0), "var_ddof0"), (df.std(), "std")):
            assert isinstance(got, pandas.Series) and list(got.index) == list(pdf.columns)
            assert np.allclose(got.to_numpy(), z[key], rtol=1e-12, atol=0), f"{name}:{key}"
        assert np.isnan(df.var(skipna=False).to_numpy()).all() and np.isnan(z["var_noskip"]).all()
        small = m.DataFrame(pdf.iloc[:60] * 1.25)
        assert np.allclose(small.prod().to_numpy(), z["prod60"], rtol=1e-12, atol=0), f"{name}:prod"
    for name, z in _load(golden_dir, "ext_groupby_*.npz"):
        n, G, V, nan, seed, kseed = (int(x) for x in z["meta"])
        pdf = synth.host_frame(n, V, seed=seed, nan_per_64k=nan, key_modulus=G, key_seed=kseed)
        g = m.DataFrame(pdf).groupby("key")
        for agg in ("min", "max"):
            got = getattr(g, agg)()._to_pandas()
            assert_exact(got.index.to_numpy(), z["keys"], f"{name}:{agg} keys")
            assert_exact(got.to_numpy(), z[agg], f"{name}:{agg}")
    # int64 columns: round(d >= 0) is the identity, clip stays int64, var promotes to float64
    ipdf = pandas.DataFrame({"a": np.arange(-50, 50, dtype=np.int64), "b": (np.arange(100, dtype=np.int64) * 7) % 13})
    idf = m.DataFrame(ipdf)
    assert_exact(idf.round(1)._to_pandas().to_numpy(), ipdf.round(1).to_numpy(), "int round")
    assert_exact(idf.clip(-3, 9)._to_pandas().to_numpy(), ipdf.clip(-3, 9).to_numpy(), "int clip")
    assert np.allclose(idf.var().to_numpy(), ipdf.var().to_numpy(), rtol=1e-12)
    assert np.allclose(idf.std(ddof=0).to_numpy(), ipdf.std(ddof=0).to_numpy(), rtol=1e-12)


def test_groupby_dictionary_aggregation(gb_table_kind):
    """qc._groupby_dict_reduce (qc.py:3876-3970): per-column functions; results zipped on the device."""
    m = bpd()
    pdf = synth.host_frame(30_011, 4, seed=5, nan_per_64k=2500, key_modulus=4099)
    spec = {"c2": "max", "c0": "sum", "c3": "count", "c1": "min"}
    got = m.DataFrame(pdf).groupby("key").agg(spec)._to_pandas()
    want = pdf.groupby("key").agg(spec)
    assert list(got.columns) == list(want.columns)
    assert_exact(got.index.to_numpy(), want.index.to_numpy(), "keys")
    for c in ("c2", "c3", "c1"):
        assert_exact(got[c].to_numpy(dtype=np.float64), want[c].to_numpy(dtype=np.float64), f"dict agg {c}")
    abs0 = pdf["c0"].abs().groupby(pdf["key"]).sum().to_numpy()
    assert_sum_close(got["c0"].to_numpy(), want["c0"].to_numpy(), abs0, len(pdf), "dict agg sum")


def test_binary_ops_between_differently_partitioned_frames():
    """Row half of _copartition: the right operand is re-cut along the left's partition lengths; the re-cut
    blocks are unaligned views (odd row offsets), which exercises the kernels' scalar-load fallback."""
    from modin_b200 import config

    m = bpd()
    a, b = synth.host_frame(100_003, 3, seed=1), synth.host_frame(100_003, 3, seed=2, nan_per_64k=5000)
    A = m.DataFrame(a)
    config.NPartitions.put(3)
    B = m.DataFrame(b)
    config.NPartitions.put(4)
    assert_exact((A * B + B)._to_pandas().to_numpy(), (a * b + b).to_numpy(), "a*b+b re-cut")
    assert_exact((B - A)._to_pandas().to_numpy(), (b - a).to_numpy(), "b-a re-cut")
    assert_exact((A >= B)._to_pandas().to_numpy(), (a >= b).to_numpy(), "a>=b re-cut")


def test_dlpack_interchange_is_zero_copy_on_device():
    import torch

    m = bpd()
    x = torch.randn(100_000, dtype=torch.float64, device="cuda")
    k = (torch.arange(100_000, device="cuda") % 7).to(torch.int64)
    df = m.from_dlpack({"x": x, "key": k})
    v = m.to_dlpack(df)
    assert v["x"].data_ptr() == x.data_ptr() and v["key"].data_ptr() == k.data_ptr()
    got = df.groupby("key").sum()._to_pandas()
    want = pandas.DataFrame({"x": x.cpu().numpy(), "key": k.cpu().numpy()}).groupby("key").sum()
    assert_exact(got.index.to_numpy(), want.index.to_numpy(), "keys")
    assert np.allclose(got.to_numpy(), want.to_numpy(), rtol=0, atol=1e-9)
    y = torch.from_dlpack(m.to_dlpack(df[["x"]] * 2.0)["x"])  # a consumer on the same device, no host round trip
    assert torch.equal(y, x * 2.0)


def test_sort_values_stable_nan_last():
    """SURVEY 8f-2 on one GPU: order-preserving key image + stable radix sort + one gather per column; equals
    pandas' stable sort bit for bit, row labels included."""
    m = bpd()
    pdf = synth.host_frame(100_003, 3, seed=2, nan_per_64k=4000, key_modulus=1009)
    pdf.loc[5, "c1"], pdf.loc[6, "c1"], pdf.loc[7, "c1"] = np.inf, -np.inf, -0.0
    df = m.DataFrame(pdf)
    for by, asc in (("key", True), ("key", False), ("c1", True), ("c1", False)):
        got = df.sort_values(by, ascending=asc)._to_pandas()
        want = pdf.sort_values(by, ascending=asc, kind="stable")
        assert_exact(got.index.to_numpy(), want.index.to_numpy(), f"sort {by} asc={asc}: row labels")
        assert_exact(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64), f"sort {by} asc={asc}")
    got = df.sort_values("c0", ignore_index=True)._to_pandas()
    want = pdf.sort_values("c0", kind="stable", ignore_index=True)
    assert isinstance(got.index, pandas.RangeIndex) and assert_exact(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64), "ignore_index") is None


def test_series_nunique_and_value_counts():
    m = bpd()
    pdf = synth.host_frame(60_001, 1, seed=3, key_modulus=5003, key_skew=True)
    s = m.DataFrame(pdf)["key"]
    assert s.nunique() == pdf["key"].nunique()
    got = s.value_counts()._to_pandas()
    want = pdf["key"].value_counts()
    assert_exact(got.to_numpy(), want.to_numpy(), "value counts, most frequent first")
    assert dict(zip(got.index, got.to_numpy())) == dict(zip(want.index, want.to_numpy()))


def test_boolean_pipelines_on_device():
    """bool (uint8) columns through the map kernel: & | ^ ~ (32-bit packed loads), widening copy for sum / mean,
    any / all as max / min -- bit-exact against pandas, odd lengths and unaligned views included."""
    m = bpd()
    for n in (5, 4099, 100_003):
        pdf = synth.host_frame(n, 3, seed=4, nan_per_64k=2000)
        df = m.DataFrame(pdf)
        mk, pm = (df > 0.0) & (df < 1.0), (pdf > 0.0) & (pdf < 1.0)
        assert_exact(mk._to_pandas().to_numpy(), pm.to_numpy(), f"and n={n}")
        assert_exact(((df > 0.5) | (df < -0.5))._to_pandas().to_numpy(), ((pdf > 0.5) | (pdf < -0.5)).to_numpy(), "or")
        assert_exact(((df > 0.0) ^ (df > 1.0))._to_pandas().to_numpy(), ((pdf > 0.0) ^ (pdf > 1.0)).to_numpy(), "xor")
        assert_exact((~mk)._to_pandas().to_numpy(), (~pm).to_numpy(), "not")
        assert_exact(mk.sum().to_numpy(), pm.sum().to_numpy(), "sum of bools")
        assert mk.sum().dtype == np.int64
        assert np.allclose(mk.mean().to_numpy(), pm.mean().to_numpy(), rtol=1e-12)
        assert_exact(mk.any().to_numpy(), pm.any().to_numpy(), "any")
        assert_exact(mk.all().to_numpy(), pm.all().to_numpy(), "all")
        assert_exact((df > -100.0).all().to_numpy(), (pdf > -100.0).all().to_numpy(), "all with NaN")


def test_multi_key_groupby_packs_the_keys(gb_table_kind):
    """groupby([k1, k2, ...]) on int64 keys: packed into one order-preserving int64 on the device, single-key
    group table, MultiIndex unpacked from the G result keys."""
    m = bpd()
    n = 40_009
    pdf = synth.host_frame(n, 3, seed=12, nan_per_64k=2000, key_modulus=97)
    pdf["k2"] = synth.gen_i64(n, 99, 1, 11) * 10 - 20
    df = m.DataFrame(pdf)
    g, pg = df.groupby(["key", "k2"]), pdf.groupby(["key", "k2"])
    abs_by_group = pdf[["c0", "c1", "c2"]].abs().groupby([pdf["key"], pdf["k2"]]).sum().to_numpy()
    got, want = g.sum()._to_pandas(), pg.sum()
    assert got.index.equals(want.index) and list(got.index.names) == ["key", "k2"]
    assert_sum_close(got.to_numpy(), want.to_numpy(), abs_by_group, n, "multi-key sum")
    for agg in ("count", "min", "max"):
        assert_exact(getattr(g, agg)()._to_pandas().to_numpy(dtype=np.float64), getattr(pg, agg)().to_numpy(dtype=np.float64), agg)
    assert_exact(g.size()._to_pandas().to_numpy(), pg.size().to_numpy(), "size")
