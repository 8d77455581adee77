"""Wide and mixed-dtype frames on the device (``-m gpu``), at the column counts where the kernels and their wrappers
branch: launches of at most 32 columns per dtype (``map_columns``, ``take_columns``, the join's payload gather),
8 columns per reduce launch, the group table's value stride (padded to a multiple of 4) and its 8-column TMA / hot-cache
limits, the 32-column column partitions, and ``mb200_concat``'s 64 sources per launch.

float64, int64 and bool columns are interleaved in an irregular order, so a dtype group's launch-local column index
differs from the column's position, and every column has data of its own: a column written to the wrong output, or two
columns swapped, shows up.  Float columns carry NaN and signed zeros (every second one also +inf or -inf) and int
columns INT64_MIN / INT64_MAX at the hot rows of ``test_gpu_special_values``; every case also runs on the
``tail(n - 1)`` view, which starts one row into its buffers.

Expected values come from pandas or from the exact references of ``tests/exact.py``.  Everything is compared bit for
bit, with dtypes and labels, except float sums and means (the README bound around the exact value) and var / std (the
derived bound of ``test_zzz_gpu_strict_bounds`` around an exact two-pass evaluation).
"""

import math

import numpy as np
import pandas
import pytest

from tests.exact import EPS, assert_bits, assert_within_sum_bound, exact_group_sums, exact_prefix_sums, exact_sum
from tests.test_gpu_parity import _four_partitions, bpd, gb_table_kind, join_table_kind  # noqa: F401  (fixtures)
from tests.test_gpu_special_values import I64_MAX, I64_MIN, _hot_rows
from tests.test_zzz_gpu_strict_bounds import _var_rtol

pytestmark = pytest.mark.gpu

N = 20_011  # odd, not a multiple of 256: the TMA groupby's ragged tail; 4 partitions of 5003 / 5002 rows
ORDER = "ffibfiifbfifbbfiffbi"  # the irregular cycle the column kinds follow
# one sign of infinity per column: a sum that meets both depends on where the partitions are cut (NaN inside one)
FLOAT_SPECIALS = ([np.inf, np.nan, -0.0, 0.0], [np.nan, 0.0, -0.0], [-0.0, 0.0], [np.nan, -np.inf, -0.0, np.nan])
INT_SPECIALS = [I64_MIN, I64_MAX, 0, -1, I64_MIN + 1, I64_MAX - 1]


def _kinds(nf, ni, nb):
    """Column kinds ('f', 'i', 'b') in ORDER's cycle, each kind until it has its count."""
    left, out, k = {"f": nf, "i": ni, "b": nb}, [], 0
    while len(out) < nf + ni + nb:
        c = ORDER[k % len(ORDER)]
        k += 1
        if left[c]:
            out.append(c)
            left[c] -= 1
    return out


def mixed_frame(nf, ni=0, nb=0, n=N, seed=0):
    """``nf`` float64, ``ni`` int64 and ``nb`` bool columns named ``<kind><position>``, interleaved; each column has its
    own scale and offset.  Float column k carries ``FLOAT_SPECIALS[k % 4]`` at the hot rows, int columns the int64
    limits."""
    rng = np.random.RandomState(seed)
    hot = _hot_rows(n)
    cols, nfl = {}, 0
    kinds = _kinds(nf, ni, nb)
    for j, kind in enumerate(kinds):
        if kind == "f":
            x = rng.randn(n) * (1.0 + 0.37 * j) + 0.5 * j
            sp = FLOAT_SPECIALS[nfl % 4]
            x[hot] = np.resize(np.roll(np.asarray(sp, dtype=np.float64), j), len(hot))
            nfl += 1
        elif kind == "i":
            x = rng.randint(-(10**6), 10**6, n).astype(np.int64) * (j + 1)
            x[hot] = np.resize(np.roll(np.array(INT_SPECIALS, dtype=np.int64), j), len(hot))
        else:
            x = rng.rand(n) < (j + 1.0) / (len(kinds) + 2.0)
        cols[f"{kind}{j}"] = x
    return pandas.DataFrame(cols)


def _of(pdf, kind):
    return [c for c in pdf.columns if str(c)[0] == kind]


def _views(*pdfs):
    """[(device frames, host frames)] as ingested and shifted by one row (8-byte aligned only)."""
    m = bpd()
    devs = [m.DataFrame(p) for p in pdfs]
    return [(devs, list(pdfs)), ([d.tail(len(p) - 1) for d, p in zip(devs, pdfs)], [p.iloc[1:] for p in pdfs])]


def assert_frame_bits(got, want, what, zero_sign=True):
    """Column labels, dtypes, row labels and every column's bits."""
    g = got._to_pandas() if hasattr(got, "_to_pandas") else got
    if isinstance(want, pandas.Series):  # a reduction or groupby.size(): values, dtype and row labels
        g = g.iloc[:, 0] if isinstance(g, pandas.DataFrame) else g
        assert str(g.dtype) == str(want.dtype), f"{what}: dtype {g.dtype} vs {want.dtype}"
        assert np.array_equal(np.asarray(g.index), np.asarray(want.index)), f"{what}: row labels"
        assert_bits(g.to_numpy(), want.to_numpy(), what, zero_sign=zero_sign)
        return
    assert list(g.columns) == list(want.columns), f"{what}: columns {list(g.columns)[:6]} vs {list(want.columns)[:6]}"
    gd, wd = [str(t) for t in g.dtypes], [str(t) for t in want.dtypes]
    assert gd == wd, f"{what}: dtypes {[(c, a, b) for c, a, b in zip(want.columns, gd, wd) if a != b][:4]}"
    assert g.shape == want.shape, f"{what}: shape {g.shape} vs {want.shape}"
    assert np.array_equal(np.asarray(g.index), np.asarray(want.index)), f"{what}: row labels"
    for j, c in enumerate(want.columns):
        assert_bits(g.iloc[:, j].to_numpy(), want.iloc[:, j].to_numpy(), f"{what} [{c}]", zero_sign=zero_sign)


# ------------------------------------------------------------------ Map / Binary
@pytest.mark.parametrize("counts", [(33, 31, 6), (65, 3, 2), (32, 6, 32), (4, 64, 2)], ids=lambda c: "f%d-i%d-b%d" % c)
def test_map_and_binary_on_wide_mixed_frames(counts):
    """Per-dtype group sizes 31, 32, 33, 64 and 65 in frames of 70 columns: scalar, row-vector and frame operands,
    the fused a*b+c, predicates, casts, fillna, clip, round, abs and negation."""
    m = bpd()
    pa, pb, pc = (mixed_frame(*counts, seed=s) for s in (1, 2, 3))
    num = _of(pa, "f") + _of(pa, "i")
    num = [c for c in pa.columns if c in num]
    bools = _of(pa, "b")
    row = list(np.linspace(-2.0, 3.0, len(num)))
    for (a, b, c), (qa, qb, qc) in _views(pa, pb, pc):
        tag = f"{counts} rows {len(qa)}"
        x, y, z, hx, hy, hz = a[num], b[num], c[num], qa[num], qb[num], qc[num]
        cases = {
            "abs": (x.abs(), hx.abs()), "neg": (-x, -hx), "+ 3": (x + 3, hx + 3), "* 2.5": (x * 2.5, hx * 2.5),
            "2 - x": (2 - x, 2 - hx), "/ 4": (x / 4, hx / 4), "+ row": (x + row, hx + row),
            "* Series": (x * pandas.Series(row, index=num), hx * pandas.Series(row, index=num)),
            "- frame": (x - y, hx - hy), "/ frame": (x / y, hx / hy), "a*b+c": (x * y + z, hx * hy + hz),
            "a*1.5+0.25": (x * 1.5 + 0.25, hx * 1.5 + 0.25), "> 0": (x > 0, hx > 0), "<= 0.5": (x <= 0.5, hx <= 0.5),
            "== frame": (x == y, hx == hy), "< frame": (x < y, hx < hy), "isna": (x.isna(), hx.isna()),
            "fillna": (x.fillna(0.5), hx.fillna(0.5)), "clip": (x.clip(-5, 5), hx.clip(-5, 5)),
            "round": (x.round(1), hx.round(1)), "astype": (a.astype("float64"), qa.astype("float64")),
        }  # fmt: skip
        if bools:
            u, v, hu, hv = a[bools], b[bools], qa[bools], qb[bools]
            cases.update({"~": (~u, ~hu), "&": (u & v, hu & hv), "|": (u | v, hu | hv), "^": (u ^ v, hu ^ hv),
                          "bool -> int64": (u.astype("int64"), hu.astype("int64"))})  # fmt: skip
        for name, (got, want) in cases.items():
            assert_frame_bits(got, want, f"{tag}: {name}")


# ------------------------------------------------------------------ TreeReduce
def _exact_var(x, ddof, skipna):
    """Two-pass variance with correctly rounded sums (``math.fsum``); NaN where pandas gives NaN."""
    nan = np.isnan(x)
    if nan.any() and not skipna:
        return math.nan
    v = x[~nan]
    if len(v) - ddof <= 0 or not np.isfinite(v).all():
        return math.nan
    mean = math.fsum(v.tolist()) / len(v)
    return math.fsum(((v - mean) ** 2).tolist()) / (len(v) - ddof)


def _assert_means(got, exact_sums, abs_sums, counts, n, what):
    """The mean bound of ``test_zzz_gpu_strict_bounds``: the sum bound over the count plus the division's rounding."""
    got = np.asarray(got, dtype=np.float64)
    counts = np.asarray(counts, dtype=np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        exact = np.where(counts > 0, np.asarray(exact_sums) / np.maximum(counts, 1), np.nan)
    assert_within_sum_bound(got, exact, np.asarray(abs_sums) / np.maximum(counts, 1) + np.abs(np.nan_to_num(exact)) / (
        2.0 * max(1.0, math.log2(max(n, 2)))), n, what)  # fmt: skip


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("nf", [7, 8, 9, 16, 17, 33])
def test_tree_reduce_on_mixed_frames(nf, variant):
    from modin_b200 import config

    pdf = mixed_frame(nf, 5, 3, seed=nf)
    fl, it, bl = _of(pdf, "f"), _of(pdf, "i"), _of(pdf, "b")
    config.ReduceVariant.put(variant)
    try:
        for (df,), (p,) in _views(pdf):
            tag = f"{nf} floats variant {variant} rows {len(p)}"
            x, hx = df[fl], p[fl]
            xs = [hx[c].to_numpy() for c in fl]
            n = len(p)
            exact = np.array([exact_sum(v) for v in xs])
            abs_sums = np.array([np.nansum(np.abs(v)) for v in xs])
            counts = np.array([int((~np.isnan(v)).sum()) for v in xs])
            assert_within_sum_bound(x.sum().to_numpy(), exact, abs_sums, n, f"{tag}: float sum")
            _assert_means(x.mean().to_numpy(), exact, abs_sums, counts, n, f"{tag}: float mean")
            for agg in ("min", "max", "count"):
                assert_frame_bits(getattr(x, agg)(), getattr(hx, agg)(), f"{tag}: float {agg}", zero_sign=False)
            for ddof in (0, 1):
                for skipna in (True, False):
                    want = np.array([_exact_var(v, ddof, skipna) for v in xs])
                    for name, w in (("var", want), ("std", np.sqrt(want))):
                        got = getattr(x, name)(ddof=ddof, skipna=skipna).to_numpy()
                        what = f"{tag}: {name} ddof={ddof} skipna={skipna}"
                        assert_bits(np.isnan(got), np.isnan(w), f"{what}: NaN where the exact value is NaN")
                        ok = np.isnan(w) | (np.abs(got - w) <= _var_rtol(n) * np.abs(w))
                        assert ok.all(), f"{what}: {got[~ok][:3]} vs exact {w[~ok][:3]}"
            y, hy = df[it], p[it]
            wrapped = [((int(np.sum(hy[c].to_numpy().astype(object))) + 2**63) % 2**64) - 2**63 for c in it]
            assert_bits(y.sum().to_numpy(), np.array(wrapped, dtype=np.int64), f"{tag}: int sum wraps")
            for agg in ("sum", "min", "max", "count"):
                assert_frame_bits(getattr(y, agg)(), getattr(hy, agg)(), f"{tag}: int {agg}")
            b, hb = df[bl], p[bl]
            for agg in ("any", "all", "sum", "count"):
                assert_frame_bits(getattr(b, agg)(), getattr(hb, agg)(), f"{tag}: bool {agg}")
    finally:
        config.ReduceVariant.put(0)


# ------------------------------------------------------------------ Fold
def test_fold_on_a_mixed_40_column_frame():
    pdf = mixed_frame(26, 14, seed=40)
    fl, it = _of(pdf, "f"), _of(pdf, "i")
    for (df,), (p,) in _views(pdf):
        tag = f"rows {len(p)}"
        qc = df._query_compiler
        got = qc.cumsum(0).to_pandas()
        assert [str(t) for t in got.dtypes] == [str(t) for t in p.dtypes], f"{tag}: cumsum dtypes"
        for c in it:
            assert_bits(got[c].to_numpy(), np.cumsum(p[c].to_numpy()), f"{tag}: int cumsum wraps [{c}]")
        for c in fl:
            x = p[c].to_numpy()
            bound = np.cumsum(np.abs(np.nan_to_num(x, posinf=0, neginf=0)))
            assert_within_sum_bound(got[c].to_numpy(), exact_prefix_sums(x), bound, len(x), f"{tag}: cumsum [{c}]")
        for name in ("cummax", "cummin"):
            assert_frame_bits(getattr(qc, name)(0).to_pandas(), getattr(p, name)(), f"{tag}: {name}")
        assert_frame_bits(df.fillna(method="ffill"), p.ffill(), f"{tag}: ffill (float columns; int columns unchanged)")


# ------------------------------------------------------------------ GroupByReduce
def _group_frame(nv, seed, G=97, skew=False, spread=3):
    """``nv`` float value columns and an int64 key column of G groups, keys ``g * spread - 50``, at a random position."""
    pdf = mixed_frame(nv, n=N, seed=seed)
    rng = np.random.RandomState(seed + 1000)
    key = rng.randint(0, G, N).astype(np.int64) * spread - 50
    if skew:
        key[rng.rand(N) < 0.4] = 7
    pdf.insert(int(rng.randint(0, nv + 1)), "key", key)
    return pdf


def _check_groupby(df, p, what, aggs=("min", "max", "count", "size")):
    vals = [c for c in p.columns if c != "key"]
    g, pg = df.groupby("key"), p.groupby("key")
    keys, exact = exact_group_sums(p["key"].to_numpy(), p[vals].to_numpy())
    abs_sums = p[vals].abs().groupby(p["key"]).sum().to_numpy()
    counts = pg.count().to_numpy()
    n = len(p)
    got = g.sum()._to_pandas()
    assert list(got.columns) == vals, f"{what}: sum columns"
    assert_bits(got.index.to_numpy(), keys, f"{what}: keys")
    assert_within_sum_bound(got.to_numpy(), exact, abs_sums, n, f"{what}: sums")
    got = g.mean()._to_pandas()
    assert_bits(got.index.to_numpy(), keys, f"{what}: mean keys")
    _assert_means(got.to_numpy(), exact, abs_sums, counts, n, f"{what}: means")
    for agg in aggs:
        assert_frame_bits(getattr(g, agg)(), getattr(pg, agg)(), f"{what}: {agg}", zero_sign=agg not in ("min", "max"))


@pytest.mark.parametrize("nv", [1, 2, 3, 4, 5, 6, 7, 8, 9, 12, 16, 17, 31, 32, 40])
def test_groupby_across_value_column_counts(nv, gb_table_kind):
    pdf = _group_frame(nv, seed=nv)
    for (df,), (p,) in _views(pdf):
        _check_groupby(df, p, f"{nv} values, {gb_table_kind}, rows {len(p)}")


@pytest.mark.parametrize("nv", [8, 9])
@pytest.mark.parametrize("table", ["dense", "hash"])
def test_skewed_groupby_at_the_hot_cache_width(nv, table, monkeypatch):
    """A heavy hitter on the TMA-staged accumulate: its per-CTA hot-group cache runs for sum / count / mean of at most 8
    value columns (9: the direct-load kernel).  The privatised shared-memory table would take this small dense range
    first, so it is switched off; min / max / size do not use the hot cache and are covered above."""
    from modin_b200 import config, ops
    from modin_b200.block import DeviceColumn

    monkeypatch.setenv("MB200_GB_SMEM", "0")
    old = config.GroupbyDenseKeys.get()
    config.GroupbyDenseKeys.put(table == "dense")
    try:
        pdf = _group_frame(nv, seed=100 + nv, skew=True)
        st = ops.key_range_device([DeviceColumn.from_numpy(pdf["key"].to_numpy())]).tolist()
        assert ops.keys_are_skewed(int(st[2]), int(st[3]))
        (df,), (p,) = _views(pdf)[0]  # the aligned view: the shifted one is not TMA-staged
        _check_groupby(df, p, f"skewed keys, {nv} values, {table}", aggs=())
    finally:
        config.GroupbyDenseKeys.put(old)


@pytest.mark.parametrize("nv", [1, 32])
def test_groupby_where_the_shared_memory_table_fits_at_one_column_only(nv):
    """1500 dense keys (range 1500).  The privatised shared-memory table keeps (value stride + 1) doubles per key and
    replica (groupby.cu): at one value column (stride 4) one replica of the sums is 1500 * 5 * 8 B = 60 kB and two fit
    in the H100's 227 kB; at 32 (stride 32) one replica is 1500 * 33 * 8 B = 396 kB, so the global-atomics kernel runs."""
    pdf = _group_frame(nv, seed=200 + nv, G=1500, spread=1)
    assert pdf["key"].max() - pdf["key"].min() + 1 == 1500
    (df,), (p,) = _views(pdf)[0]
    _check_groupby(df, p, f"1500 keys, {nv} values")


def test_dict_aggregation_across_the_column_partition_cut_and_two_keys():
    m = bpd()
    pdf = _group_frame(40, seed=300)
    pdf["k2"] = np.random.RandomState(301).randint(0, 3, N).astype(np.int64) * 100 - 100
    df = m.DataFrame(pdf)
    vals = [c for c in pdf.columns if c not in ("key", "k2")]
    spec = {vals[29]: "max", vals[30]: "count", vals[31]: "sum", vals[32]: "min", vals[33]: "sum", vals[0]: "count"}
    got, want = df.groupby("key").agg(spec)._to_pandas(), pdf.groupby("key").agg(spec)
    assert list(got.columns) == list(want.columns) and [str(t) for t in got.dtypes] == [str(t) for t in want.dtypes]
    assert_bits(got.index.to_numpy(), want.index.to_numpy(), "agg keys")
    for c, f in spec.items():
        if f == "sum":
            keys, exact = exact_group_sums(pdf["key"].to_numpy(), pdf[c].to_numpy())
            assert_within_sum_bound(got[c].to_numpy(), exact, pdf[c].abs().groupby(pdf["key"]).sum().to_numpy(), N, c)
        else:
            assert_bits(got[c].to_numpy(), want[c].to_numpy(), f"agg {c}: {f}", zero_sign=f == "count")
    cols = ["key", "k2"] + vals
    got, want = df[cols].groupby(["key", "k2"]).sum()._to_pandas(), pdf[cols].groupby(["key", "k2"]).sum()
    assert list(got.index) == list(want.index) and list(got.columns) == list(want.columns)
    two = pdf["key"].to_numpy() * 1000 + pdf["k2"].to_numpy()
    _, exact = exact_group_sums(two, pdf[vals].to_numpy())
    abs_sums = pdf[vals].abs().groupby([pdf["key"], pdf["k2"]]).sum().to_numpy()
    assert_within_sum_bound(got.to_numpy(), exact, abs_sums, N, "two-key sums")


# ------------------------------------------------------------------ Merge
def _dim(nf, ni, unique, seed):
    rng = np.random.RandomState(seed)
    keys = rng.permutation(520)[:450] if unique else rng.randint(0, 520, 700)
    pay = mixed_frame(nf, ni, n=len(keys), seed=seed)
    pay.columns = [f"d{c}" for c in pay.columns]
    pay.insert(0, "key", keys.astype(np.int64))
    return pay


def _fact(dim, misses, seed, n=N):
    rng = np.random.RandomState(seed)
    pool = np.arange(520, dtype=np.int64) if misses else np.unique(dim["key"].to_numpy())
    return pandas.DataFrame({"key": pool[rng.randint(0, len(pool), n)], "x": rng.randn(n),
                             "xi": rng.randint(-9, 9, n).astype(np.int64)})  # fmt: skip


@pytest.mark.parametrize("payload", [(1, 0), (7, 1), (26, 5), (32, 0), (27, 5), (33, 0), (33, 7), (5, 35)],
                         ids=lambda w: "f%d-i%d" % w)
def test_merge_across_payload_widths(payload, join_table_kind, monkeypatch):
    """Payload widths 1, 8, 31, 32, 33 and 40 of float64 and int64 columns, with more than 32 of one dtype at 33 and 40
    (int64 promoted to float64 when a left join misses) x ordered probe on / off
    x unique / repeated dim keys x left / inner x with / without misses; each dim merged twice in a row with different
    facts, so that a payload copy cached with the table for the wrong columns would show."""
    m = bpd()
    width = sum(payload)
    for ordered in ("1", "0"):
        monkeypatch.setenv("MB200_JOIN_ORDERED", ordered)
        for unique in (True, False):
            dim = _dim(*payload, unique, seed=width + 7 * unique)
            ddim = m.DataFrame(dim)
            for misses in (True, False):
                for how in ("left", "inner"):
                    for rep in range(2):
                        fact = _fact(dim, misses, seed=10 * width + rep)
                        got = m.DataFrame(fact).merge(ddim, on="key", how=how)
                        want = fact.merge(dim, on="key", how=how)
                        what = f"payload {payload} {join_table_kind} ordered={ordered} unique={unique} misses={misses} {how} #{rep}"
                        assert_frame_bits(got, want, what)
            if payload == (33, 7) and unique:
                # a merge result is ONE block of 43 columns: map and row selection see more than 32 of a dtype at once
                fact = _fact(dim, True, seed=99)
                got, want = m.DataFrame(fact).merge(ddim, on="key", how="left"), fact.merge(dim, on="key", how="left")
                assert_frame_bits(got * 1.5 + 0.25, want * 1.5 + 0.25, "merge result * 1.5 + 0.25")
                assert_frame_bits(got[got["x"] > 0.0], want[want["x"] > 0.0], "merge result [x > 0]")
                assert_frame_bits(got.sort_values("x"), want.sort_values("x", kind="stable"), "merge result sorted")


def test_bool_payload_is_gathered_or_refused_never_false(join_table_kind):
    """pandas turns a bool payload column of a left join with misses into object dtype (NaN): that is refused; without
    misses, and for inner joins, the bool column is gathered."""
    m = bpd()
    for unique in (True, False):
        dim = _dim(2, 1, unique, seed=50 + unique)
        dim["bp"] = np.random.RandomState(52).rand(len(dim)) < 0.5
        ddim = m.DataFrame(dim)
        for misses in (True, False):
            fact = _fact(dim, misses, seed=53)
            inner = m.DataFrame(fact).merge(ddim, on="key", how="inner")
            assert_frame_bits(inner, fact.merge(dim, on="key", how="inner"), f"unique={unique} misses={misses} inner")
            if misses:
                with pytest.raises(NotImplementedError, match="bool payload"):
                    m.DataFrame(fact).merge(ddim, on="key", how="left")._to_pandas()
            else:
                got = m.DataFrame(fact).merge(ddim, on="key", how="left")
                assert_frame_bits(got, fact.merge(dim, on="key", how="left"), f"unique={unique} left without misses")


# ------------------------------------------------------------------ row movement
def test_row_movement_on_a_70_column_mixed_frame():
    """Row selection, sort and drop_duplicates gather float64 / int64 columns (frames with bool columns are refused
    there); head, tail and concatenation also carry the bool columns."""
    m = bpd()
    pdf = mixed_frame(33, 31, 6, seed=70)
    pdf["key"] = np.random.RandomState(71).randint(0, 900, N).astype(np.int64)
    other = mixed_frame(2, 1, 1, seed=72)
    other.columns = [f"o{c}" for c in other.columns]
    num = [c for c in pdf.columns if c not in _of(pdf, "b")]
    f0, i0 = _of(pdf, "f")[2], _of(pdf, "i")[1]  # f0: no NaN among its specials
    for (df, do), (p, po) in _views(pdf, other):
        tag = f"rows {len(p)}"
        cases = {
            "head": (df.head(7001), p.head(7001)), "tail": (df.tail(7001), p.tail(7001)),
            "concat rows": (m.concat([df, df.tail(999)]), pandas.concat([p, p.tail(999)])),
            "concat columns": (m.concat([df, do], axis=1), pandas.concat([p, po], axis=1)),
        }  # fmt: skip
        df, p = df[num], p[num]
        cases.update({"[mask]": (df[df[f0] > 0.0], p[p[f0] > 0.0]), "dropna": (df.dropna(), p.dropna())})
        for by in (f0, i0):
            for asc in (True, False):
                cases[f"sort {by} asc={asc}"] = (df.sort_values(by, ascending=asc), p.sort_values(by, ascending=asc, kind="stable"))
        for keep in ("first", "last"):
            cases[f"drop_duplicates {keep}"] = (df.drop_duplicates(subset=["key"], keep=keep), p.drop_duplicates(subset=["key"], keep=keep))
        for name, (got, want) in cases.items():
            assert_frame_bits(got, want, f"{tag}: {name}")


# ------------------------------------------------------------------ concatenation
@pytest.mark.parametrize("npieces", [1, 63, 64, 65, 130])
def test_concat_columns_against_numpy(npieces):
    from modin_b200 import ops
    from modin_b200.block import DeviceColumn

    rng = np.random.RandomState(npieces)
    lengths = rng.randint(1, 400, npieces) * 2 + 1  # odd: later bool pieces start unaligned
    lengths[npieces // 2] = 9001  # 72 kB of float64: more than one 64 KiB chunk
    for dtype in (np.float64, np.int64, np.bool_):
        host = [rng.randn(k + 1).astype(dtype) if dtype != np.bool_ else rng.rand(k + 1) < 0.5 for k in lengths]
        for shifted in (False, True):
            # shifted: every piece is a view one element into its buffer
            pieces = [DeviceColumn.from_numpy(h).slice(1, len(h)) if shifted else DeviceColumn.from_numpy(h[1:]) for h in host]
            got = ops.concat_columns(pieces).to_numpy()
            want = np.concatenate([h[1:] for h in host])
            assert got.dtype == want.dtype
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), f"{npieces} {np.dtype(dtype)} shifted={shifted}"


def test_frames_concatenated_from_70_odd_pieces_merge_and_deduplicate():
    m = bpd()
    rng = np.random.RandomState(80)
    dim = pandas.DataFrame({"key": rng.permutation(5000).astype(np.int64), "d": rng.randn(5000),
                            "di": rng.randint(-99, 99, 5000).astype(np.int64), "db": rng.rand(5000) < 0.3})  # fmt: skip
    cuts = np.concatenate([[0], np.sort(rng.choice(np.arange(1, 2500) * 2 + 1, 69, replace=False)), [5000]])
    assert len(cuts) == 71 and (np.diff(cuts)[:-1] % 2 == 1).any()
    ddim = m.concat([m.DataFrame(dim.iloc[a:b]) for a, b in zip(cuts[:-1], cuts[1:])], ignore_index=True)
    assert_frame_bits(ddim, dim, "dim from 70 pieces")
    fact = pandas.DataFrame({"key": rng.randint(0, 5200, N).astype(np.int64), "x": rng.randn(N)})
    got = m.DataFrame(fact).merge(ddim, on="key", how="inner")
    assert_frame_bits(got, fact.merge(dim, on="key", how="inner"), "inner merge against the concatenated dim")
    got = m.DataFrame(fact).merge(ddim[["key", "d", "di"]], on="key", how="left")
    assert_frame_bits(got, fact.merge(dim[["key", "d", "di"]], on="key", how="left"), "left merge against the concatenated dim")
    frame = pandas.DataFrame({"key": rng.randint(0, 700, 5000).astype(np.int64), "v": rng.randn(5000),
                              "i": rng.randint(-99, 99, 5000).astype(np.int64)})  # fmt: skip
    dframe = m.concat([m.DataFrame(frame.iloc[a:b]) for a, b in zip(cuts[:-1], cuts[1:])], ignore_index=True)
    for keep in ("first", "last"):
        assert_frame_bits(dframe.drop_duplicates(subset=["key"], keep=keep), frame.drop_duplicates(subset=["key"], keep=keep),
                          f"drop_duplicates keep={keep} of a frame from 70 pieces")  # fmt: skip
