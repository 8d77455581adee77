"""``groupby.nunique`` on the H100, bit for bit against numpy and pandas.

The NUNIQUE table through ``ops.GroupTable``: pass 1 on the existing SIZE launch, pass 2 (``mb200_gb_accumulate_distinct``)
on the new kernel, on every table kind (dense over a small range -- the shared-memory pass-1 kernel --, dense over a
large range, hashed, and skewed keys), row counts around warp, 256-row tile and grid boundaries up to 2^25 + 3, 1 to 40
columns, value cardinalities of one, two, about sqrt(n) and all distinct, the edge values (+-0.0, NaN payloads, +-inf,
the int64 extremes and the images of the empty slot), the partial form over other tables' ``emit_distinct``, and both
front doors at the benchmark's groupby shape.  The reference counts distinct (key, image) pairs with numpy."""

import numpy as np
import pandas
import pytest

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
NAN_IMAGE = 0x7FF8000000000000
PAYLOADS = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0x7FF8DEADBEEF0001],
                    dtype=np.uint64).view(np.float64)  # fmt: skip


def _images(x, dropna):
    if x.dtype == np.int64:
        return x, np.ones(len(x), dtype=bool)
    b = x.view(np.int64)
    img = np.where(x == 0.0, 0, b ^ ((b >> 63) & np.int64(0x7FFFFFFFFFFFFFFF)))
    nan = np.isnan(x)
    return np.where(nan, NAN_IMAGE, img).astype(np.int64), ~nan | (not dropna)


def _expected(keys, cols, dropna):
    """Ascending unique keys, and per column the number of distinct images per key (numpy, exact)."""
    uk = np.unique(keys)
    out = []
    for x in cols:
        img, ok = _images(x, dropna)
        pairs = np.unique(np.stack([keys[ok], img[ok]], axis=1), axis=0) if ok.any() else np.zeros((0, 2), np.int64)
        gk, n = np.unique(pairs[:, 0], return_counts=True)
        cnt = np.zeros(len(uk), dtype=np.int64)
        cnt[np.searchsorted(uk, gk)] = n
        out.append(cnt)
    return uk, out


def _columns(n, ncols, seed):
    """Columns of cardinality one, two, ~sqrt(n) and all distinct, float64 and int64 in turn, with edge values."""
    rng = np.random.default_rng(seed)
    edges_f = np.concatenate([[0.0, -0.0, np.inf, -np.inf], PAYLOADS])
    edges_i = np.array([I64_MIN, I64_MAX, 0, -1], dtype=np.int64)
    r = max(int(np.sqrt(n)), 1)
    cols = []
    for j in range(ncols):
        kind, i64 = j % 4, (j // 4) % 2 == 1
        if kind == 0:
            x = np.full(n, 7, dtype=np.int64) if i64 else np.full(n, 0.25)
        elif kind == 1:
            x = rng.choice(edges_i[:2], n) if i64 else rng.choice(np.array([0.0, -0.0, np.nan]), n)
        elif kind == 2:
            x = rng.integers(0, r, n).astype(np.int64) if i64 else rng.integers(0, r, n) * 0.5
        else:
            x = rng.permutation(n).astype(np.int64) - n // 2 if i64 else rng.permutation(n) * 1.5 - 3.0
        if n and kind >= 2:
            m = rng.random(n) < 0.05
            x[m] = rng.choice(edges_i, m.sum()) if i64 else rng.choice(edges_f, m.sum())
        cols.append(x)
    return cols


def _keys(n, seed, kind):
    rng = np.random.default_rng(seed + 1)
    G = 40 if kind == "small" else 5000
    keys = rng.integers(0, G, n).astype(np.int64)
    if kind == "skewed":
        keys[rng.random(n) < 0.33] = 0
    if kind == "large" and n:
        keys[0] = 1 << 20  # a range far wider than shared memory holds
    return keys


def _table(keys, W, kind):
    from modin_b200 import _lib, ops

    flags = _lib.GB_SIZE | _lib.GB_NUNIQUE
    if kind in ("hashed", "skewed"):
        t = ops.GroupTable(max(1024, len(np.unique(keys))), W, flags)
    else:
        t = ops.GroupTable.dense(int(keys.min()) if len(keys) else 0, int(keys.max()) if len(keys) else 0, W, flags)
    t.hint_skew(kind == "skewed")
    return t


def _fill(keys, cols, kind, dropna):
    from modin_b200 import functors, ops
    from modin_b200.block import DeviceColumn

    t = _table(keys, len(cols), kind)
    kd = DeviceColumn.from_numpy(keys)
    t.accumulate(kd, [])
    t.reserve_distinct(functors._next_pow2(2 * max(len(keys) * len(cols), 1)))
    t.accumulate_distinct(kd, [DeviceColumn.from_numpy(x) for x in cols], dropna=dropna)
    ng, overflow = t.ngroups()
    assert not overflow
    return t, ng


def _check(keys, cols, dropna, got):
    k, sums, cnts, sizes = got
    uk, want = _expected(keys, cols, dropna)
    assert sums is None and np.array_equal(k.to_numpy(), uk)
    assert np.array_equal(sizes.to_numpy(), np.unique(keys, return_counts=True)[1])
    for j, w in enumerate(want):
        assert np.array_equal(cnts[j].to_numpy(), w), (j, np.flatnonzero(cnts[j].to_numpy() != w)[:5])


def _run(keys, cols, kind, dropna=True):
    from modin_b200 import ops

    from tests.test_gpu_groupby_var import env

    with env(MB200_GB_SMEM=1 if kind == "small" else 0):
        t, ng = _fill(keys, cols, kind, dropna)
    try:
        got = t.emit(ng, sort=True)
    finally:
        t.close()
    _check(keys, cols, dropna, got)


ROWS = [0, 1, 31, 32, 33, 255, 256, 257, 4097, 1024 * 132 + 5]


@pytest.mark.parametrize("kind", ["small", "large", "hashed", "skewed"])
@pytest.mark.parametrize("n", ROWS)
def test_tables_count_exactly(kind, n):
    keys = _keys(n, n, kind)
    cols = _columns(n, 8, n + 3)
    for dropna in (True, False):
        _run(keys, cols, kind, dropna)


@pytest.mark.parametrize("kind", ["small", "large", "hashed"])
@pytest.mark.parametrize("ncols", [1, 8, 9, 32])
def test_column_counts(kind, ncols):
    n = 256 * 61 + 13
    _run(_keys(n, ncols, kind), _columns(n, ncols, ncols), kind, dropna=ncols % 2 == 0)


@pytest.mark.parametrize("kind", ["small", "large", "hashed"])
def test_partial_rows_rebuild_the_counts(kind):
    """Three tables over three row ranges emit their distinct sets; a fresh table takes the concatenated rows (pass 1
    on their keys, pass 2 in partial form) and gives the counts of all the rows."""
    from modin_b200 import ops
    from modin_b200.block import DeviceColumn

    from tests.test_gpu_groupby_var import env

    n = 1024 * 132 + 5
    keys, cols = _keys(n, 7, kind), _columns(n, 9, 7)
    parts = []
    with env(MB200_GB_SMEM=1 if kind == "small" else 0):
        for a, b in ((0, 1000), (1000, 70_001), (70_001, n)):
            t, ng = _fill(keys[a:b], [x[a:b] for x in cols], kind, False)
            try:
                ek, ec, ei, count = t.emit_distinct(ng, ng + (b - a) * 9)
                m, overflow = count.tolist()
                assert not overflow and m >= ng
                parts.append([x.to_numpy()[:m] for x in (ek, ec, ei)])
            finally:
                t.close()
        pk, pc, pi = (np.concatenate([p[j] for p in parts]) for j in range(3))
        t = _table(pk, 9, kind)
        try:
            kd = DeviceColumn.from_numpy(pk)
            t.accumulate(kd, [])
            t.reserve_distinct(1 << int(2 * len(pk) - 1).bit_length())
            t.accumulate_distinct(kd, col_ids=DeviceColumn.from_numpy(pc), images=DeviceColumn.from_numpy(pi))
            got = ops.emit_counted(t)
        finally:
            t.close()
    k, _, cnts, _ = got
    uk, want = _expected(keys, cols, False)
    assert np.array_equal(k.to_numpy(), uk)
    for j in range(9):
        assert np.array_equal(cnts[j].to_numpy(), want[j]), j


def test_two_to_the_25_rows():
    n = (1 << 25) + 3
    cols = _columns(n, 3, 9)
    keys = np.random.default_rng(9).integers(0, 100_000, n).astype(np.int64)
    for kind in ("small", "large", "hashed"):
        _run(keys % 64 if kind == "small" else keys, cols, kind)


def test_nunique_tables_refuse_what_they_cannot_do():
    from modin_b200 import _lib, ops
    from modin_b200.block import DeviceColumn

    flags = _lib.GB_SIZE | _lib.GB_NUNIQUE
    keys = DeviceColumn.from_numpy(np.arange(8, dtype=np.int64))
    vals = [DeviceColumn.from_numpy(np.arange(8.0))]
    for dense in (False, True):
        t = ops.GroupTable.dense(0, 7, 1, flags) if dense else ops.GroupTable(64, 1, flags)
        try:
            t.accumulate(keys, [])
            with pytest.raises(_lib.B200Error):
                t.accumulate_distinct(keys, vals)  # no set reserved yet
            with pytest.raises(_lib.B200Error):
                t.reserve_distinct(3)  # not a power of two
            t.reserve_distinct(4)  # 8 entries do not fit in 4 slots: the overflow flag, never a short count
            t.accumulate_distinct(keys, vals)
            assert t.ngroups()[1]
            with pytest.raises(_lib.B200Error):
                t.accumulate(keys, [])  # no pass-1 rows after pass 2
        finally:
            t.close()
    for bad in (_lib.GB_NUNIQUE, _lib.GB_COUNT | _lib.GB_NUNIQUE, flags | _lib.GB_SUM):
        with pytest.raises(_lib.B200Error):
            ops.GroupTable(64, 1, bad)
    t = ops.GroupTable(64, 1, _lib.GB_SIZE)
    try:
        with pytest.raises(_lib.B200Error):
            t.reserve_distinct(16)  # not a NUNIQUE table
    finally:
        t.close()


@pytest.mark.parametrize("nparts", [1, 3])
def test_front_door_special_values_and_batches_match_pandas(nparts):
    import modin_b200.pandas as bpd
    from modin_b200 import config

    old, budget = config.NPartitions.get(), config.GroupbyDistinctBytes.get()
    config.NPartitions.put(nparts)
    try:
        n = 4000
        rng = np.random.default_rng(4)
        key = rng.integers(0, 50, n).astype(np.int64)
        cols = _columns(n, 12, 5)
        pdf = pandas.DataFrame({"key": key, **{f"c{j}": x for j, x in enumerate(cols)}, "b": rng.random(n) < 0.3,
                                "nan": np.where(key == 3, np.nan, 1.0)})  # fmt: skip
        for budget_bytes in (budget, 16):  # the default, then one column per batch
            config.GroupbyDistinctBytes.put(budget_bytes)
            for dropna in (True, False):
                got = bpd.DataFrame(pdf).groupby("key").nunique(dropna=dropna)._to_pandas()
                want = pdf.groupby("key").nunique(dropna=dropna)
                pandas.testing.assert_frame_equal(got, want, check_index_type=False)
    finally:
        config.NPartitions.put(old)
        config.GroupbyDistinctBytes.put(budget)


# ------------------------------------------------------------------ front doors
@pytest.fixture(scope="module")
def bench_frame():
    from modin_b200 import synth

    df = synth.device_frame(1 << 26, 8, seed=42, nan_per_64k=3000, key_modulus=1_000_000)
    pdf = df._to_pandas()
    return df, pdf, pdf.groupby("key").nunique()


@pytest.mark.parametrize("case", ["dense", "hashed"])
def test_front_door_at_the_benchmark_shape(bench_frame, case):
    from modin_b200 import config

    df, pdf, want = bench_frame
    old = config.GroupbyDenseKeys.get()
    config.GroupbyDenseKeys.put(case == "dense")
    try:
        got = df.groupby("key").nunique()._to_pandas()
        pandas.testing.assert_frame_equal(got, want, check_index_type=False)
        if case == "dense":
            got = df.groupby("key", as_index=False).agg({"c0": "nunique", "c1": "sum"})._to_pandas()
            assert np.array_equal(got["c0"].to_numpy(), want["c0"].to_numpy())
    finally:
        config.GroupbyDenseKeys.put(old)


def test_plugin_front_door_at_the_benchmark_shape(bench_frame):
    import os
    import sys
    import warnings

    ref = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "modin")):
        pytest.skip("reference Modin not installed under oracle/_ref")
    if ref not in sys.path:
        sys.path.insert(0, ref)
    warnings.filterwarnings("ignore")
    from modin_b200 import modin_plugin

    modin_plugin.register()
    import modin
    import modin.pandas as mpd

    modin.set_execution(engine="B200", storage_format="Arrow")
    _, pdf, want = bench_frame
    got = mpd.DataFrame(pdf).groupby("key").nunique()._to_pandas()
    pandas.testing.assert_frame_equal(got, want, check_index_type=False)
    s = mpd.DataFrame(pdf[["key", "c3"]]).groupby("key")["c3"].nunique(dropna=False)._to_pandas()
    pandas.testing.assert_series_equal(s, pdf.groupby("key")["c3"].nunique(dropna=False), check_index_type=False)
