"""``groupby.first`` / ``last`` on the H100, bit for bit against numpy.

The kernel through ``ops.GroupTable`` / ``ops.hash_aggregate``: every accumulate variant a FIRST / LAST table can take
(shared-memory table, TMA tiles with a ragged tail, direct loads at 9-40 columns and on shifted views and under
``MB200_GB_VARIANT=1`` / ``2``, hashed tables, skewed keys, ``MB200_GB_SMEM=0``), with winners planted at row 0, at the
last row, on both sides of 256-row tile cuts and of the TMA / tail boundary, NULL value columns, and a second
accumulate call on the same table.  Then both aggregations through the mirror at the benchmark's shape (dense, hashed,
skewed, several row partitions), run twice, and a small mixed-dtype frame against pandas."""

import contextlib
import os

import numpy as np
import pandas
import pytest

pytestmark = pytest.mark.gpu

G = 1000


@contextlib.contextmanager
def env(**kw):
    old = {k: os.environ.get(k) for k in kw}
    os.environ.update({k: str(v) for k, v in kw.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _positions(keys, col, fn):
    """numpy reference: ascending unique keys of ALL rows, and per key the first / last row whose value is not NaN
    (every row for col None), -1 when there is none."""
    uk = np.unique(keys)
    ok = np.ones(len(keys), dtype=bool) if col is None else ~np.isnan(col)
    k, rows = keys[ok], np.flatnonzero(ok)
    if fn == "last":
        k, rows = k[::-1], rows[::-1]
    u, idx = np.unique(k, return_index=True)
    out = np.full(len(uk), -1, dtype=np.int64)
    out[np.searchsorted(uk, u)] = rows[idx]
    return uk, out


def _planted(n, ncols, seed, tail_start=None):
    """Keys over [0, G) and values ~97 % NaN, with special keys (G, G + 1, ...) that occur only at planted rows: row 0
    with the last row, both sides of every 256-row tile cut, and the TMA / tail boundary; one of them has its only
    non-NaN value in the ragged tail.  Column 1 holds -0.0 / 0.0 / +-inf where it is not NaN."""
    rng = np.random.default_rng(seed)
    keys = rng.integers(0, G, n).astype(np.int64)
    vals = [np.where(rng.random(n) < 0.97, np.nan, rng.standard_normal(n)) for _ in range(ncols)]
    if ncols > 1:
        vals[1] = np.where(np.isnan(vals[1]), np.nan, rng.choice([-0.0, 0.0, np.inf, -np.inf], n))
    special = G
    pairs = [(0, n - 1)] + [(c - 1, c) for c in range(256, n, 256)]
    if tail_start is not None and 0 < tail_start < n:
        pairs.append((tail_start - 1, tail_start))
    for a, b in pairs:
        keys[[a, b]] = special
        for v in vals:
            v[a], v[b] = 1.5 + a, -2.5 - b
        special += 1
    if tail_start is not None and 0 < tail_start < n - 1:
        keys[[5, tail_start + 1]] = special  # only non-NaN value of this group is in the tail
        for v in vals:
            v[5], v[tail_start + 1] = np.nan, 3.25
    return keys, vals


def _run_table(keys, vals, fn, dense=True, skew=False, calls=1, shift=0, with_null=True):
    """Positions from a FIRST / LAST table; with ``calls`` > 1 the rows arrive in that many accumulate calls."""
    from modin_b200 import _lib, ops
    from modin_b200.block import DeviceColumn

    flag = _lib.GB_FIRST if fn == "first" else _lib.GB_LAST
    cols = list(vals) + ([None] if with_null else [])
    n = len(keys) - shift
    dk = DeviceColumn.from_numpy(keys)
    dv = [DeviceColumn.from_numpy(v) if v is not None else None for v in cols]
    if shift:  # views that start 1-3 rows into their buffers: not 16-byte aligned, so the direct-load kernel
        dk = DeviceColumn(dk.data[shift:], np.int64)
        dv = [DeviceColumn(v.data[shift:], np.float64) if v is not None else None for v in dv]
    hk = keys[shift:]
    table = ops.GroupTable.dense(int(hk.min()), int(hk.max()), len(cols), flag) if dense else ops.GroupTable(4 * G, len(cols), flag)
    table.hint_skew(skew)
    try:
        cuts = np.linspace(0, n, calls + 1).astype(int)
        for a, b in zip(cuts, cuts[1:]):
            ops.fill_table(table, [(DeviceColumn(dk.data[a:b], np.int64),
                                    [DeviceColumn(v.data[a:b], np.float64) if v is not None else None for v in dv])])  # fmt: skip
        k, pos, _, _ = ops.emit_counted(table)
    finally:
        table.close()
    got_k = k.to_numpy()
    for j, c in enumerate(cols):
        uk, want = _positions(hk, c[shift:] if c is not None else None, fn)
        assert np.array_equal(got_k, uk)
        got = pos[j].to_numpy()
        assert got.dtype == np.int64 and np.array_equal(got, want), (fn, j, np.flatnonzero(got != want)[:5])


@pytest.mark.parametrize("fn", ["first", "last"])
def test_smem_table(fn):
    keys, vals = _planted(10_000, 3, 1)
    _run_table(keys % 50, vals, fn)  # 50 keys: the per-CTA shared-memory table
    _run_table(keys % 50, vals, fn, calls=2)


@pytest.mark.parametrize("fn", ["first", "last"])
@pytest.mark.parametrize("nvals", [1, 7])
def test_tma_tiles_with_ragged_tail(fn, nvals):
    n = 256 * 301 + 77
    keys, vals = _planted(n, nvals, 2, tail_start=256 * 301)
    with env(MB200_GB_SMEM=0):
        _run_table(keys, vals, fn)  # nvals + the NULL column <= 8, aligned: TMA tiles, 77-row tail on direct loads
        _run_table(keys, vals, fn, calls=3)
        _run_table(keys, vals, fn, dense=False)


@pytest.mark.parametrize("fn", ["first", "last"])
def test_direct_loads_wide_shifted_and_variants(fn):
    n = 256 * 97 + 131
    keys, vals = _planted(n, 12, 3, tail_start=256 * 97)
    with env(MB200_GB_SMEM=0):
        _run_table(keys, vals, fn)  # 13 columns
        for shift in (1, 2, 3):
            _run_table(keys, vals[:5], fn, shift=shift, dense=shift != 2)
        for variant in (1, 2):
            with env(MB200_GB_VARIANT=variant):
                _run_table(keys, vals, fn)
                _run_table(keys, vals[:3], fn, dense=False, calls=2)


@pytest.mark.parametrize("fn", ["first", "last"])
def test_forty_columns_through_hash_aggregate(fn):
    from modin_b200 import _lib, ops
    from modin_b200.block import DeviceColumn

    keys, vals = _planted(256 * 40 + 5, 39, 4)
    cols = [DeviceColumn.from_numpy(v) for v in vals] + [None]
    flag = _lib.GB_FIRST if fn == "first" else _lib.GB_LAST
    k, pos, _, _ = ops.hash_aggregate([(DeviceColumn.from_numpy(keys), cols)], flag, G)
    for j, c in enumerate(vals + [None]):
        uk, want = _positions(keys, c, fn)
        assert np.array_equal(k.to_numpy(), uk) and np.array_equal(pos[j].to_numpy(), want), j


@pytest.mark.parametrize("fn", ["first", "last"])
def test_skewed_keys_do_not_take_the_hot_cache(fn):
    keys, vals = _planted(256 * 200 + 9, 4, 5, tail_start=256 * 200)
    rng = np.random.default_rng(6)
    hot = rng.random(len(keys)) < 0.6
    keys[hot & (keys < G)] = 7  # one key with most of the rows
    _run_table(keys, vals, fn, skew=True, dense=True)
    _run_table(keys, vals, fn, skew=True, dense=False)


def test_first_last_tables_refuse_what_they_cannot_do():
    from modin_b200 import _lib, ops
    from modin_b200.block import DeviceColumn

    keys = DeviceColumn.from_numpy(np.arange(8, dtype=np.int64))
    t = ops.GroupTable(64, 1, _lib.GB_FIRST)
    try:
        with pytest.raises(_lib.B200Error):
            t.merge_partial(keys, [DeviceColumn.from_numpy(np.zeros(8))])
    finally:
        t.close()
    with pytest.raises(_lib.B200Error):
        ops.GroupTable(64, 1, _lib.GB_FIRST | _lib.GB_SUM)
    t = ops.GroupTable(64, 1, _lib.GB_MAX)
    try:
        with pytest.raises(TypeError):
            t.accumulate(keys, [None])
    finally:
        t.close()


# ------------------------------------------------------------------ front doors
def _reference(pdf, fn):
    """numpy first / last per column (one stable sort of the keys, then per column the non-NaN rows)."""
    keys = pdf["key"].to_numpy()
    order = np.argsort(keys, kind="stable")
    ks = keys[order]
    uk = ks[np.r_[True, ks[1:] != ks[:-1]]]
    out = {}
    for c in pdf.columns.drop("key"):
        x = pdf[c].to_numpy()
        ok = ~np.isnan(x[order])
        o, k = order[ok], ks[ok]
        if fn == "first":
            sel = np.r_[True, k[1:] != k[:-1]]
        else:
            sel = np.r_[k[1:] != k[:-1], True]
        res = np.full(len(uk), np.nan)
        res[np.searchsorted(uk, k[sel])] = x[o[sel]]
        out[c] = res
    return uk, out


def _bits_equal(a, b):
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.nan_to_num(a).view(np.int64),
                                                                        np.nan_to_num(b).view(np.int64))  # fmt: skip


@pytest.mark.parametrize("case", ["dense", "hashed", "skewed", "3 partitions"])
def test_front_door_at_the_benchmark_shape(case):
    from modin_b200 import config, synth

    n, groups = 1 << 26, 1_000_000
    old = config.GroupbyDenseKeys.get()
    config.GroupbyDenseKeys.put(case != "hashed")
    try:
        df = synth.device_frame(n, 8, npartitions=3 if case == "3 partitions" else 1, seed=42, nan_per_64k=30000,
                                key_modulus=groups, key_skew=case == "skewed")  # fmt: skip
        pdf = df._to_pandas()
        for fn in ("first", "last"):
            uk, want = _reference(pdf, fn)
            a = getattr(df.groupby("key"), fn)()._to_pandas()
            b = getattr(df.groupby("key"), fn)()._to_pandas()
            assert np.array_equal(a.index.to_numpy(), uk) and np.array_equal(b.index.to_numpy(), uk)
            for c, w in want.items():
                assert _bits_equal(a[c].to_numpy(), w) and _bits_equal(b[c].to_numpy(), w), (fn, c)
    finally:
        config.GroupbyDenseKeys.put(old)


@pytest.mark.parametrize("nparts", [1, 3])
def test_front_door_mixed_dtypes_match_pandas(nparts):
    import modin_b200.pandas as bpd
    from modin_b200 import config

    old = config.NPartitions.get()
    config.NPartitions.put(nparts)
    try:
        rng = np.random.default_rng(11)
        n = 5003
        key = rng.integers(0, 97, n).astype(np.int64)
        key[:3] = 500  # a group whose float values are all NaN
        f = np.where(rng.random(n) < 0.6, np.nan, rng.choice([-0.0, 0.0, np.inf, -np.inf, 1.25], n))
        f[:3] = np.nan
        lim = np.where(np.arange(n) % 3 == 0, np.iinfo(np.int64).min, np.iinfo(np.int64).max).astype(np.int64)
        pdf = pandas.DataFrame({"key": key, "f": f, "i": lim, "b": rng.random(n) < 0.5})
        df = bpd.DataFrame(pdf)
        for fn in ("first", "last"):
            for kw in ({}, {"skipna": False}):
                got, want = getattr(df.groupby("key"), fn)(**kw)._to_pandas(), getattr(pdf.groupby("key"), fn)(**kw)
                assert list(got.dtypes) == list(want.dtypes) and np.array_equal(got.index, want.index)
                assert _bits_equal(got["f"].to_numpy(), want["f"].to_numpy())
                assert np.array_equal(got["i"], want["i"]) and np.array_equal(got["b"], want["b"])
            spec = {"f": fn, "i": "last", "b": "first"}
            got, want = df.groupby("key").agg(spec)._to_pandas(), pdf.groupby("key").agg(spec)
            assert list(got.dtypes) == list(want.dtypes) and _bits_equal(got["f"].to_numpy(), want["f"].to_numpy())
    finally:
        config.NPartitions.put(old)
