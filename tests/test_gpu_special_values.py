"""Special values against exact references (``-m gpu``): signed zeros that tie, sums that overflow to +-inf, both
infinities, int64 keys at the limits, and more groups than a hash table was sized for -- placed where kernels go wrong:
the first and last row, both sides of a 4096-row tile, of a 2048-element reduce tile and of every partition cut, the
odd tail element of a block, and a view that starts one row into its buffer (``tail(n - 1)``: 8-byte aligned only).

Expected values are pandas or the exact helpers of ``tests/exact.py``; where Modin's partitioning changes the answer
(the sum of +inf and -inf within one partition) they come from the oracle.  Everything is compared bit for bit, except
float sums (the README bound around the exact value, with +-inf and NaN matched exactly) and the zero sign of min /
max, which is unspecified.
"""

import operator

import numpy as np
import pandas
import pytest

from oracle import reference_path as orc
from tests.exact import assert_bits, assert_within_sum_bound, exact_group_sums, exact_prefix_sums, exact_sum
from tests.test_gpu_parity import _four_partitions, bpd, gb_table_kind, join_table_kind  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
N = 20_011  # odd; 4 partitions of 5003 rows (odd blocks: the TMA reduce's tail element) and one of 5002
BIG = 1e308


def _hot_rows(n, nparts=4):
    """First / last row, both sides of the 2048- and 4096-row tiles of every partition, both sides of every cut."""
    chunk = -(-n // nparts)
    rows = {0, n - 1, n - 2}
    for p in range(0, n, chunk):
        rows |= {p - 1, p, p + 1, p + 2047, p + 2048, p + 4095, p + 4096, min(p + chunk, n) - 1}
    return np.array(sorted(r for r in rows if 0 <= r < n))


def _frame_with(specials, n=N, ncols=4, seed=0):
    """float64 columns of normals with ``specials`` cycled over the hot rows (a different phase per column)."""
    rng = np.random.RandomState(seed)
    hot = _hot_rows(n)
    cols = {}
    for j in range(ncols):
        x = rng.randn(n)
        x[hot] = np.resize(np.roll(np.asarray(specials, dtype=np.float64), j), len(hot))
        cols[f"c{j}"] = x
    return pandas.DataFrame(cols)


def _both_offsets(pdf):
    """(device frame, host frame) as ingested and shifted by one row."""
    m = bpd()
    df = m.DataFrame(pdf)
    return [(df, pdf), (df.tail(len(pdf) - 1), pdf.iloc[1:])]


# ------------------------------------------------------------------ Map / Binary
SPECIALS = [0.0, -0.0, np.inf, -np.inf, np.nan, -0.4, 0.4, -0.6, 2.5, -2.5, BIG, -BIG, 5e-324, -5e-324, 1.0, -1.0]


def test_map_and_binary_on_special_values():
    pdf = _frame_with(SPECIALS)
    for df, p in _both_offsets(pdf):
        tag = f"rows {len(p)}"
        get = lambda r: r._to_pandas().to_numpy()  # noqa: E731
        assert_bits(get(df.abs()), p.abs().to_numpy(), f"{tag} abs")
        assert_bits(get(-df), (-p).to_numpy(), f"{tag} neg")
        assert_bits(get(df.clip(lower=0.0)), p.clip(lower=0.0).to_numpy(), f"{tag} clip(lower=0.0) keeps -0.0")
        assert_bits(get(df.round()), p.round().to_numpy(), f"{tag} round: round(-0.4) = -0.0")
        for s in (0.0, -0.0, 3.0):
            assert_bits(get(df / s), (p / s).to_numpy(), f"{tag} / {s!r}")
        assert_bits(get(df * 0.0), (p * 0.0).to_numpy(), f"{tag} * 0.0 (inf * 0 = NaN)")
        assert_bits(get(df * -1.0 + BIG), (p * -1.0 + BIG).to_numpy(), f"{tag} fused affine")
        for name in ("eq", "lt", "le", "gt", "ge", "ne"):
            for s in (0.0, -0.0):
                cmp = getattr(operator, name)
                assert_bits(get(cmp(df, s)), cmp(p, s).to_numpy(), f"{tag} {name} {s!r}")
        # a * b + c with b, c frames: inf - inf, inf * 0, overflow of the product
        b, c = p[["c1", "c2", "c3", "c0"]].set_axis(p.columns, axis=1), p[["c3", "c0", "c1", "c2"]].set_axis(p.columns, axis=1)
        m = bpd()
        got = get(df * m.DataFrame(b) + m.DataFrame(c))
        assert_bits(got, (p * b + c).to_numpy(), f"{tag} a*b+c")
        assert_bits(get(df == m.DataFrame(b)), (p == b).to_numpy(), f"{tag} a == b (-0.0 == 0.0)")
        assert_bits(get(df < m.DataFrame(b)), (p < b).to_numpy(), f"{tag} a < b")


def test_int64_map_at_the_limits():
    m = bpd()
    rng = np.random.RandomState(1)
    hot = _hot_rows(N)
    i = rng.randint(-1000, 1000, N).astype(np.int64)
    i[hot] = np.resize(np.array([I64_MIN, I64_MAX, I64_MIN + 1, I64_MAX - 1, 0, -1, 2**53 + 1, -(2**53) - 1]), len(hot))
    pdf = pandas.DataFrame({"i": i, "j": np.roll(i, 7)})
    for df, p in _both_offsets(pdf):
        get = lambda r: r._to_pandas().to_numpy()  # noqa: E731
        assert_bits(get(df.abs()), p.abs().to_numpy(), "int abs (abs(INT64_MIN) wraps)")
        assert_bits(get(-df), (-p).to_numpy(), "int neg (-INT64_MIN wraps)")
        assert_bits(get(df.astype("float64")), p.astype("float64").to_numpy(), "int -> float64 rounds to nearest even")
        assert_bits(get(df / 0), (p / 0).to_numpy(), "int / 0")
        assert_bits(get(df + 1), (p + 1).to_numpy(), "int + 1 wraps")
        assert_bits(get(df == I64_MIN), (p == I64_MIN).to_numpy(), "int == INT64_MIN")


# ------------------------------------------------------------------ TreeReduce
def _overflow_frame():
    """Columns whose exact sum is outside the float64 range: overflow inside one CTA (rows 1, 2), only at the combine
    of one block's CTA partials (rows 1, 2049 of partition 0), only across partitions, negative overflow; and the
    infinities: +inf / -inf in different partitions (NaN everywhere) and in one partition (the reference's map phase
    gives NaN there and its skipna reduce drops it)."""
    rng = np.random.RandomState(2)
    cols = {}
    for name, rows, v in (("cta", (1, 2), BIG), ("finalize", (1, 2049), BIG), ("partitions", (5002, 5003), BIG),
                          ("negative", (N - 2, N - 1), -BIG), ("tail", (5002, 10005), BIG)):  # fmt: skip
        x = rng.randn(N)
        x[list(rows)] = v
        cols[name] = x
    x = np.round(rng.randn(N) * 8)  # integer-valued: every partial sum is exact
    x[[3, 15_009]] = [np.inf, -np.inf]
    cols["inf_across"] = x
    x = np.round(rng.randn(N) * 8)
    x[[3, 4096]] = [np.inf, -np.inf]
    cols["inf_within"] = x
    return pandas.DataFrame(cols)


@pytest.mark.parametrize("variant", [0, 1])
def test_sums_that_overflow_are_inf_not_nan(variant):
    from modin_b200 import config

    pdf = _overflow_frame()
    config.ReduceVariant.put(variant)
    try:
        df = bpd().DataFrame(pdf)
        exact = np.array([exact_sum(pdf[c].to_numpy()) for c in pdf.columns])
        assert np.isinf(exact[:5]).all() and np.isnan(exact[5:]).all()
        got = df.sum().to_numpy()
        assert_bits(got, orc.df_sum(pdf, 4).to_numpy(), f"variant {variant}: sum vs the oracle")
        assert_bits(got[:6], exact[:6], f"variant {variant}: overflowing sums are +-inf")
        assert_bits(df.mean().to_numpy(), orc.df_mean(pdf, 4).to_numpy(), f"variant {variant}: mean vs the oracle")
        # the shifted view is cut differently; overflow does not depend on the cuts
        shifted, p = df.tail(N - 1)[list(pdf.columns[:5])], pdf.iloc[1:, :5]
        exact = np.array([exact_sum(p[c].to_numpy()) for c in p.columns])
        assert_bits(shifted.sum().to_numpy(), exact, f"variant {variant}: shifted view, overflowing sums")
        assert_bits(shifted.mean().to_numpy(), exact, f"variant {variant}: shifted view, overflowing means")
    finally:
        config.ReduceVariant.put(0)


def test_var_and_std_whose_squares_overflow():
    m = bpd()
    x = np.resize(np.array([1e154, -1e154]), N)
    y = np.resize(np.array([1.5e154, -1.5e154, 0.0]), N)  # every square finite, their sum is not
    pdf = pandas.DataFrame({"x": x, "y": y, "z": np.random.RandomState(3).randn(N)})
    df = m.DataFrame(pdf)
    for ddof in (1, 0):
        assert_bits(df.var(ddof=ddof).to_numpy()[:2], pdf.var(ddof=ddof).to_numpy()[:2], f"var ddof={ddof}")
        assert_bits(df.std(ddof=ddof).to_numpy()[:2], pdf.std(ddof=ddof).to_numpy()[:2], f"std ddof={ddof}")
        assert np.isinf(df.var(ddof=ddof).to_numpy()[:2]).all()
        assert np.allclose(df.var(ddof=ddof).to_numpy()[2], pdf["z"].var(ddof=ddof), rtol=1e-12, atol=0)


@pytest.mark.parametrize("n", [1, 3, 2047, 2048, 2049, 300_007])
def test_ill_conditioned_sums_against_the_exact_sum(n):
    """Sum |x| >> |sum x|: large values that nearly cancel, so the bound is the only slack; both reduce variants."""
    from modin_b200 import config

    m = bpd()
    rng = np.random.RandomState(n % 1000)
    big = rng.randn(n) * 1e12
    x = big + rng.randn(n)
    x[1::2] = -big[:-1:2] if n > 1 else x[1::2]  # pairs cancel to ~1e-4 relative
    y = rng.randn(n) * np.exp(rng.uniform(-30, 30, n))  # magnitudes over 26 decades
    y[rng.rand(n) < 0.05] = np.nan
    pdf = pandas.DataFrame({"x": x, "y": y, "z": np.where(rng.rand(n) < 0.5, -0.0, 0.0)})
    for variant in (0, 1):
        config.ReduceVariant.put(variant)
        try:
            got = m.DataFrame(pdf).sum().to_numpy()
        finally:
            config.ReduceVariant.put(0)
        for j, c in enumerate(pdf.columns):
            v = pdf[c].to_numpy()
            assert_within_sum_bound(got[j], exact_sum(v), np.nansum(np.abs(v)), n, f"n={n} variant {variant} {c}")
        assert_bits(got[2], 0.0, "a sum of zeros is +0.0")


def test_min_max_of_signed_zeros_and_int_wrapping():
    m = bpd()
    pdf = _frame_with([0.0, -0.0, -0.0, 0.0, np.inf, -np.inf], ncols=2)
    zeros = pandas.DataFrame({"z": np.resize(np.array([-0.0, 0.0, -0.0]), N), "w": np.resize(np.array([0.0, -0.0]), N)})
    for frame in (pdf, zeros):
        for df, p in _both_offsets(frame):
            for agg in ("min", "max"):
                assert_bits(getattr(df, agg)().to_numpy(), getattr(p, agg)().to_numpy(), f"{agg}", zero_sign=False)
    i = np.full(N, 3, dtype=np.int64)
    i[_hot_rows(N)] = I64_MAX
    assert_bits(m.DataFrame(pandas.DataFrame({"i": i})).sum().to_numpy(), np.array([np.sum(i)]), "int sum wraps like numpy")
    small = pandas.DataFrame({"p": np.resize(np.array([3, -5, 7], dtype=np.int64), 200)})
    assert_bits(m.DataFrame(small).prod().to_numpy(), np.array([np.prod(small["p"].to_numpy())]), "int prod wraps like numpy")


# ------------------------------------------------------------------ Fold
def _fold_frame():
    rng = np.random.RandomState(4)
    lead = rng.randn(N)
    lead[0] = -0.0
    nan_lead = rng.randn(N)
    nan_lead[:3] = [np.nan, -0.0, -0.0]
    zeros = np.full(N, -0.0)  # -0.0 through every tile and cut, then +0.0 after a NaN and after a 0.0
    zeros[15_009] = np.nan
    zeros[[4096 + 5003]] = 0.0
    over = np.abs(rng.randn(N))
    over[[4095, 5003, 10_006]] = BIG  # inf from row 5003 on
    over[15_009] = -np.inf  # then inf + -inf
    return pandas.DataFrame({"lead": lead, "nan_lead": nan_lead, "zeros": zeros, "over": over})


def test_cumsum_signed_zeros_and_overflow_against_the_exact_prefix_sums():
    m = bpd()
    pdf = _fold_frame()
    for df, p in _both_offsets(pdf):
        got = df._query_compiler.cumsum(0).to_pandas()
        for c in p.columns:
            x = p[c].to_numpy()
            exact = exact_prefix_sums(x)
            g = got[c].to_numpy()
            assert_within_sum_bound(g, exact, np.cumsum(np.abs(np.nan_to_num(x, posinf=0, neginf=0))), len(x), f"cumsum {c}")
            z = exact == 0
            assert_bits(g[z], exact[z], f"cumsum {c}: zero signs")
            assert_bits(g[z], p[c].cumsum().to_numpy()[z], f"cumsum {c}: zero signs as pandas")
    first = m.DataFrame(pdf)._query_compiler.cumsum(0).to_pandas()
    assert_bits(first["lead"].to_numpy()[:1], np.array([-0.0]), "cumsum([-0.0, ...]) starts with -0.0")
    assert_bits(first["nan_lead"].to_numpy()[:3], np.array([np.nan, 0.0, 0.0]), "cumsum([NaN, -0.0, -0.0]) = [NaN, 0.0, 0.0]")


def test_cummin_cummax_return_the_latest_of_tied_zeros():
    """pandas' cummax / cummin return the latest of equal values (``cummax([0.0, -0.0]) = [0.0, -0.0]``)."""
    pdf = _frame_with([0.0, -0.0, -0.0, 0.0, np.nan, np.inf, -np.inf, 0.0], ncols=3)
    pdf["zeros"] = np.resize(np.array([-0.0, 0.0, np.nan, 0.0, -0.0]), N)
    for df, p in _both_offsets(pdf):
        for name in ("cummax", "cummin"):
            got = getattr(df._query_compiler, name)(0).to_pandas().to_numpy()
            assert_bits(got, getattr(p, name)().to_numpy(), f"{name} rows {len(p)}")


@pytest.mark.parametrize("op", ["sum", "max", "min"])
def test_special_values_across_three_shard_carries(op):
    """The multi-rank carry (``mb200_cum_carry``) with -0.0 runs, +-inf and NaN on both sides of the shard cuts."""
    from modin_b200 import ops
    from modin_b200.block import DeviceColumn

    t = ops.torch_mod()
    n = 30_011
    rng = np.random.RandomState(9)
    a = np.where(rng.rand(n) < 0.5, -0.0, 0.0)
    a[:10_001] = -0.0  # the whole first shard and the first row of the second
    b = rng.randn(n)
    b[[9_999, 20_000]] = [np.inf, -np.inf]
    c = rng.randn(n)
    c[[9_999, 10_000, 19_999, 20_000]] = [-0.0, np.nan, 0.0, -0.0]
    host = [a, b, c]
    cuts = [(0, 10_000), (10_000, 20_000), (20_000, n)]
    shards = [[DeviceColumn.from_numpy(np.ascontiguousarray(x[lo:hi])) for x in host] for lo, hi in cuts]
    states = [ops.cum_partials(op, s) for s in shards]
    gathered = [t.cat([st.groups[k][3] for st in states]) for k in range(len(states[0].groups))]
    pieces = [[] for _ in host]
    for r, (st, cols) in enumerate(zip(states, shards)):
        for j, o in enumerate(ops.cum_apply(st, cols, ops.cum_carry(st, gathered, r))):
            pieces[j].append(o.to_numpy())
    for x, pc in zip(host, pieces):
        got = np.concatenate(pc)
        if op == "sum":
            exact = exact_prefix_sums(x)
            assert_within_sum_bound(got, exact, np.cumsum(np.abs(np.nan_to_num(x, posinf=0, neginf=0))), n, "carried cumsum")
            assert_bits(got[exact == 0], exact[exact == 0], "carried cumsum: zero signs")
        else:
            assert_bits(got, getattr(pandas.Series(x), "cum" + op)().to_numpy(), f"carried cum{op}")


# ------------------------------------------------------------------ GroupByReduce
def _group_frame(keys_of):
    """Rows of groups with special sums / extrema, plus ordinary groups; ``keys_of`` maps group number -> key."""
    rng = np.random.RandomState(5)
    n = N
    g = rng.randint(6, 40, n)
    v = rng.randn(n, 2)
    g[[0, 1]], v[[0, 1], 0] = 0, BIG  # group 0: overflow inside partition 0
    g[[5002, 15_009]], v[[5002, 15_009], 0] = 1, -BIG  # group 1: overflow across partitions
    g[[4095, 10_006]], v[[4095, 10_006], 0] = 2, [np.inf, -np.inf]  # group 2: both infinities, different partitions
    g[[2047, 2048, 9_099]], v[[2047, 2048, 9_099], :] = 3, -0.0  # group 3: only -0.0 (sum +0.0)
    g[[100, 101, 102, 5003]], v[[100, 101, 102, 5003], :] = 4, [[0.0, -0.0], [-0.0, 0.0], [0.0, -0.0], [-0.0, -0.0]]
    g[[200, 201, N - 1]], v[[200, 201, N - 1], :] = 5, [[np.inf, -np.inf], [1.0, 2.0], [-np.inf, np.inf]]
    v[rng.rand(n) < 0.03] = np.nan
    return pandas.DataFrame({"key": np.array([keys_of(int(x)) for x in g], dtype=np.int64), "c0": v[:, 0], "c1": v[:, 1]})


def _check_groupby(pdf, what):
    m = bpd()
    g = m.DataFrame(pdf).groupby("key")
    pg = pdf.groupby("key")
    keys, exact = exact_group_sums(pdf["key"].to_numpy(), pdf[["c0", "c1"]].to_numpy())
    got = g.sum()._to_pandas()
    assert_bits(got.index.to_numpy(), keys, f"{what}: keys")
    abs_by_group = pdf[["c0", "c1"]].abs().groupby(pdf["key"]).sum().to_numpy()
    assert_within_sum_bound(got.to_numpy(), exact, abs_by_group, len(pdf), f"{what}: sums vs exact")
    assert_bits(got.to_numpy()[exact == 0], exact[exact == 0], f"{what}: zero sums are +0.0")
    for agg in ("min", "max"):
        assert_bits(getattr(g, agg)()._to_pandas().to_numpy(), getattr(pg, agg)().to_numpy(), f"{what}: {agg}", zero_sign=False)
    assert_bits(g.size()._to_pandas().to_numpy(), pg.size().to_numpy(), f"{what}: size")
    assert_bits(g.count()._to_pandas().to_numpy(), pg.count().to_numpy(), f"{what}: count")


def test_groupby_special_sums_and_extrema(gb_table_kind):
    _check_groupby(_group_frame(lambda x: x * 3 - 50), "narrow keys")


def test_groupby_keys_at_the_int64_limits(gb_table_kind):
    extremes = [I64_MIN, I64_MIN + 1, -1, 0, I64_MAX]
    _check_groupby(_group_frame(lambda x: extremes[x % 5]), "keys INT64_MIN, INT64_MIN + 1, -1, 0, INT64_MAX (hash)")
    _check_groupby(_group_frame(lambda x: I64_MAX - 999 + (x * 25) % 1000), "1000 keys ending at INT64_MAX")
    _check_groupby(_group_frame(lambda x: I64_MIN + (x * 25) % 1000), "1000 keys starting at INT64_MIN")


def test_skewed_groupby_with_special_values():
    from modin_b200 import ops
    from modin_b200.block import DeviceColumn

    pdf = _group_frame(lambda x: x)
    rng = np.random.RandomState(6)
    hot = rng.rand(N) < 0.4
    hot[[0, 1, 5002, 15_009, 4095, 10_006, 2047, 2048, 9_099]] = False
    pdf.loc[hot, "key"] = 7  # a heavy hitter: the per-CTA hot-group cache
    pdf.loc[hot & (rng.rand(N) < 0.5), "c1"] = -0.0
    lo, hi, sampled, dup = (int(v) for v in ops.key_range_device([DeviceColumn.from_numpy(pdf["key"].to_numpy())]).tolist())
    assert ops.keys_are_skewed(sampled, dup)
    _check_groupby(pdf, "skewed keys")


# ------------------------------------------------------------------ group-table growth
def _wide_keys(G, reps, seed):
    rng = np.random.RandomState(seed)
    k = (np.arange(G, dtype=np.int64) - G // 2) * 1_000_003_019  # range ~1e14: the dense table is refused
    return k[rng.permutation(np.tile(np.arange(G), reps))]


def test_hash_table_regrowth_at_the_ops_level():
    from modin_b200 import _lib, ops
    from modin_b200.block import DeviceColumn

    G = 100_003
    keys = _wide_keys(G, 2, 7)
    rng = np.random.RandomState(8)
    v = rng.randn(len(keys))
    v[rng.rand(len(keys)) < 0.1] = np.nan
    v[:2] = [-0.0, BIG]
    kd, vd = DeviceColumn.from_numpy(keys), DeviceColumn.from_numpy(v)
    assert not ops.dense_range_ok(int(keys.min()), int(keys.max()), 1024, len(keys), 1, _lib.GB_SUM)
    pg = pandas.DataFrame({"k": keys, "v": v}).groupby("k")["v"]
    want_keys = np.sort(np.unique(keys))
    for flag, out, want in ((_lib.GB_SUM, 1, None), (_lib.GB_COUNT, 2, pg.count()), (_lib.GB_MIN, 1, pg.min()),
                            (_lib.GB_MAX, 1, pg.max()), (_lib.GB_SIZE, 3, pg.size())):  # fmt: skip
        res = ops.hash_aggregate([(kd, [vd])], flag, 1024)
        assert_bits(res[0].to_numpy(), want_keys, f"flag {flag}: keys after regrowth")
        col = res[out][0] if out in (1, 2) else res[out]
        if want is None:
            _, exact = exact_group_sums(keys, v)
            assert_within_sum_bound(col.to_numpy(), exact, pandas.Series(np.abs(v)).groupby(keys).sum().to_numpy(), 2, "sum")
        else:
            assert_bits(col.to_numpy(), want.to_numpy(), f"flag {flag}", zero_sign=flag not in (_lib.GB_MIN, _lib.GB_MAX))
    # partial=True: per-partition partial results (keys repeat) merged into a table that has to grow
    pk = np.concatenate([np.unique(keys[: len(keys) // 2]), np.unique(keys[len(keys) // 2 :])])
    pv = np.random.RandomState(9).randn(len(pk))
    pc = np.random.RandomState(10).randint(0, 5, len(pk)).astype(np.int64)
    pkd, pvd, pcd = DeviceColumn.from_numpy(pk), DeviceColumn.from_numpy(pv), DeviceColumn.from_numpy(pc)
    ph = pandas.DataFrame({"k": pk, "v": pv, "c": pc}).groupby("k")
    k, s, _, _ = ops.hash_aggregate([(pkd, [pvd], None, None)], _lib.GB_SUM, 1024, partial=True)
    assert_bits(k.to_numpy(), want_keys, "partial sum keys")
    _, exact = exact_group_sums(pk, pv)
    assert_within_sum_bound(s[0].to_numpy(), exact, ph["v"].apply(lambda x: np.abs(x).sum()).to_numpy(), 2, "partial sum")
    for flag, want in ((_lib.GB_MIN, ph["v"].min()), (_lib.GB_MAX, ph["v"].max())):
        k, s, _, _ = ops.hash_aggregate([(pkd, [pvd], None, None)], flag, 1024, partial=True)
        assert_bits(s[0].to_numpy(), want.to_numpy(), f"partial flag {flag}")
    k, _, c, _ = ops.hash_aggregate([(pkd, [ops.cast_columns_f64([pcd])[0]], [pcd], None)], _lib.GB_COUNT, 1024, partial=True)
    assert_bits(c[0].to_numpy(), ph["c"].sum().to_numpy(), "partial count")
    k, _, _, z = ops.hash_aggregate([(pkd, [], None, pcd)], _lib.GB_SIZE, 1024, partial=True)
    assert_bits(z.to_numpy(), ph["c"].sum().to_numpy(), "partial size")


def test_an_overflowed_group_table_refuses_to_emit():
    from modin_b200 import _lib, ops
    from modin_b200.block import DeviceColumn

    keys = _wide_keys(5000, 1, 11)
    table = ops.GroupTable(1024, 1, _lib.GB_SUM)
    try:
        table.accumulate(DeviceColumn.from_numpy(keys), [DeviceColumn.from_numpy(np.ones(len(keys)))])
        ng, overflow = table.ngroups()
        assert overflow and ng <= 1024
        with pytest.raises(_lib.B200Error, match="overflow"):
            table.emit(ng)
    finally:
        table.close()


@pytest.mark.parametrize("nparts", [1, 4])
def test_groupby_with_more_groups_than_the_first_table(nparts):
    """3 * 2**20 distinct wide keys: G > 2**20, the first table's capacity (one partition: the table must grow)."""
    from modin_b200 import config

    config.NPartitions.put(nparts)
    n = 3 << 20
    keys = _wide_keys(n, 1, 12)
    v = np.random.RandomState(13).randn(n)
    pdf = pandas.DataFrame({"key": keys, "v": v})
    g = bpd().DataFrame(pdf).groupby("key")
    got = g.sum()._to_pandas()
    want = pdf.groupby("key").sum()
    assert len(got) == n
    assert_bits(got.index.to_numpy(), want.index.to_numpy(), "keys")
    assert_bits(got["v"].to_numpy(), want["v"].to_numpy(), "one row per group: the sum is the value")
    assert_bits(g.size()._to_pandas().to_numpy(), pdf.groupby("key").size().to_numpy(), "size")


# ------------------------------------------------------------------ Merge
def test_merge_with_keys_at_the_int64_limits(join_table_kind):
    m = bpd()
    rng = np.random.RandomState(14)
    narrow = I64_MAX - np.arange(500, dtype=np.int64)  # dense: max - min + 1 = 500, ending at INT64_MAX
    for dim_keys, fact_pool in (
        (rng.permutation(narrow)[:463], np.concatenate([I64_MAX - np.arange(580, dtype=np.int64), [I64_MIN, 0, -1]])),
        (np.array([I64_MIN, I64_MIN + 1, -1, 0, I64_MAX], dtype=np.int64), np.array([I64_MIN, I64_MIN + 1, I64_MIN + 2, -1, 0, 1, I64_MAX, I64_MAX - 1])),
        (I64_MIN + rng.permutation(500)[:450].astype(np.int64), np.concatenate([I64_MIN + np.arange(520, dtype=np.int64), [I64_MAX]])),
    ):  # fmt: skip
        fact = pandas.DataFrame({"key": fact_pool[rng.randint(0, len(fact_pool), N)], "c0": rng.randn(N)})
        dim = pandas.DataFrame({"key": dim_keys, "d0": rng.randn(len(dim_keys)), "d1": np.arange(len(dim_keys), dtype=np.int64)})
        for how in ("left", "inner"):
            got = m.DataFrame(fact).merge(m.DataFrame(dim), on="key", how=how)._to_pandas()
            want = orc.broadcast_merge(fact, dim, "key", how, 4)
            assert list(got.columns) == list(want.columns)
            assert_bits(got["key"].to_numpy(), want["key"].to_numpy(), f"merge {how}: keys")
            assert_bits(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64), f"merge {how}")


# ------------------------------------------------------------------ sort and friends
def test_sort_values_ties_signed_zeros_and_orders_infinities():
    m = bpd()
    pdf = _frame_with([0.0, -0.0, np.nan, np.inf, -np.inf, -0.0, 0.0, 1.0, -1.0], ncols=2)
    pdf["k"] = np.resize(np.array([I64_MIN, 0, I64_MAX, -1, I64_MIN + 1, I64_MAX - 1]), N)
    pdf.loc[pdf.index % 7 == 0, "c0"] = -0.0
    pdf.loc[pdf.index % 11 == 0, "c0"] = 0.0
    df = m.DataFrame(pdf)
    for by in ("c0", "c1", "k"):
        for asc in (True, False):
            got = df.sort_values(by, ascending=asc)._to_pandas()
            want = pdf.sort_values(by, ascending=asc, kind="stable")
            assert_bits(got.index.to_numpy(), want.index.to_numpy(), f"sort {by} asc={asc}: row labels")
            assert_bits(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64), f"sort {by} asc={asc}: bits")
            assert_bits(got["k"].to_numpy(), want["k"].to_numpy(), f"sort {by} asc={asc}: int64 column")


def test_distinct_values_and_membership_at_the_int64_limits():
    m = bpd()
    rng = np.random.RandomState(15)
    pool = np.array([I64_MIN, I64_MIN + 1, -1, 0, 1, I64_MAX - 1, I64_MAX], dtype=np.int64)
    k = pool[rng.randint(0, len(pool), N)]
    k[[0, N - 1]] = [I64_MAX, I64_MIN]
    pdf = pandas.DataFrame({"k": k, "v": rng.randn(N)})
    df = m.DataFrame(pdf)
    for keep in ("first", "last"):
        got = df.drop_duplicates(subset=["k"], keep=keep)._to_pandas()
        want = pdf.drop_duplicates(subset=["k"], keep=keep)
        assert_bits(got.index.to_numpy(), want.index.to_numpy(), f"drop_duplicates keep={keep}: labels")
        assert_bits(got.to_numpy(dtype=np.float64), want.to_numpy(dtype=np.float64), f"drop_duplicates keep={keep}")
    assert df["k"].nunique() == pdf["k"].nunique() == len(pool)
    got, want = df["k"].value_counts()._to_pandas(), pdf["k"].value_counts()
    assert dict(zip(got.index, got.to_numpy())) == dict(zip(want.index, want.to_numpy()))
    assert_bits(got.to_numpy(), want.to_numpy(), "value counts, most frequent first")
    for vals in ([I64_MIN, I64_MAX], [I64_MIN + 1, 0, 5], [I64_MAX - 1]):
        assert_bits(df[["k"]].isin(vals)._to_pandas().to_numpy(), pdf[["k"]].isin(vals).to_numpy(), f"isin {vals}")


def test_alignment_matches_a_negative_zero_label_to_zero():
    m = bpd()
    a = pandas.DataFrame({"c": [1.0, 2.0, 4.0, 8.0]}, index=pandas.Index([0.0, 1.0, 2.0, 5.0]))
    b = pandas.DataFrame({"c": [16.0, 32.0, 64.0]}, index=pandas.Index([-0.0, 1.0, 3.0]))
    for left, right in ((a, b), (b, a)):
        got = (m.DataFrame(left) + m.DataFrame(right))._to_pandas()
        want = left + right
        assert list(got.index) == list(want.index)
        assert_bits(got["c"].to_numpy(), want["c"].to_numpy(), "-0.0 label matched to 0.0")
