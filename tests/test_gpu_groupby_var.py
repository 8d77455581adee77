"""``groupby.var`` / ``std`` on the H100, against exact sums of squared deviations.

The VAR table through ``ops.GroupTable``: pass 1 on the existing SUM | COUNT kernels, pass 2 (``mb200_gb_accumulate_m2``)
on the new ones, on every table kind (dense over a small range -- the per-CTA shared-memory tables --, dense over a
large range and hashed on direct loads, and skewed keys whose pass 1 takes the hot-group cache), row counts around
warp, 256-row, 4096-row and grid boundaries up to 2^25 + 3, 1 to 40 columns, and partial merges.  Values are
``base + X / 1024`` with integer X, so the exact M2 of every group is an integer ratio; the result must lie within

    |M2^ - M2| <= (3n + 8) u (M2 + 5 n d^2) + 5 n d^2 + 4 d sqrt(n M2),   d = (n + 2) u max|x|,  u = 2^-53

(README, "Accuracy of groupby.var / std"), and without the last term when no partials are merged.  The mean-1e9 column
is the ill-conditioned case a one-pass sum of squares gets wrong.  Then special values and both front doors at the
benchmark's groupby shape (2^26 rows, 1e6 keys, dense and hashed) against pandas."""

import contextlib
import os

import numpy as np
import pandas
import pytest

pytestmark = pytest.mark.gpu

U = 2.0**-53


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


def _data(n, ncols, seed, G, kind):
    """Keys over [0, G) (skewed: key 0 takes a third of the rows); per column integers X in [-2^12, 2^12), ~10 % NaN,
    values base + X / 1024 with base 0 or 1e9 (every third column)."""
    rng = np.random.default_rng(seed)
    keys = rng.integers(0, G, n).astype(np.int64)
    if kind == "skewed":
        keys[rng.random(n) < 0.33] = 0
    Xs, nans, bases = [], [], []
    for j in range(ncols):
        Xs.append(rng.integers(-(1 << 12), 1 << 12, n).astype(np.int64))
        nans.append(rng.random(n) < 0.1)
        bases.append(1e9 if j % 3 == 2 else 0.0)
    return keys, Xs, nans, bases


def _values(X, nan, base):
    v = base + X.astype(np.float64) / 1024.0  # exact: |X| / 1024 < 4 sits on the 2^-22 grid of 1e9
    v[nan] = np.nan
    return v


def _exact(keys, X, nan, base):
    """Per ascending key: (n, exact sum as float, exact M2 as float, max |x|)."""
    ok = ~nan
    k, x = keys[ok], X[ok]
    order = np.argsort(k, kind="stable")
    k, x = k[order], x[order]
    uk = np.unique(keys)
    out = {int(g): (0, 0.0, 0.0, 0.0) for g in uk}
    if len(k):
        starts = np.flatnonzero(np.r_[True, k[1:] != k[:-1]])
        sx = np.add.reduceat(x, starts)
        sx2 = np.add.reduceat(x * x, starts)  # |X| < 2^12, <= 2^25 rows: < 2^49
        cnt = np.diff(np.r_[starts, len(k)])
        amax = np.maximum.reduceat(np.abs(base + x.astype(np.float64) / 1024.0), starts)
        for g, n, s, s2, a in zip(k[starts].tolist(), cnt.tolist(), sx.tolist(), sx2.tolist(), amax.tolist()):
            m2 = (n * s2 - s * s) / (n * (1 << 20))  # Python ints: exact, one rounding
            out[g] = (n, base * n + s / 1024.0, m2, a)
    return uk, out


def _bound(n, m2, a, merged):
    d = (n + 2) * U * a
    b = (3 * n + 8) * U * (m2 + 5 * n * d * d) + 5 * n * d * d
    return b + (4 * d * np.sqrt(n * m2) if merged else 0.0)


def _check(keys, Xs, nans, bases, got, merged):
    k, sums, cnts, _ = got
    W = len(Xs)
    assert len(sums) == 2 * W and len(cnts) == W
    gk = k.to_numpy()
    for j in range(W):
        uk, ex = _exact(keys, Xs[j], nans[j], bases[j])
        assert np.array_equal(gk, uk), j
        n = np.array([ex[g][0] for g in uk.tolist()], dtype=np.int64)
        s = np.array([ex[g][1] for g in uk.tolist()])
        m2 = np.array([ex[g][2] for g in uk.tolist()])
        a = np.array([ex[g][3] for g in uk.tolist()])
        assert np.array_equal(cnts[j].to_numpy(), n), j
        assert np.all(np.abs(sums[j].to_numpy() - s) <= (n + 1) * U * n * a), j
        err = np.abs(sums[W + j].to_numpy() - m2)
        lim = _bound(n.astype(np.float64), m2, a, merged)
        bad = np.flatnonzero(~(err <= lim))
        assert not len(bad), (j, bad[:5], err[bad[:5]], lim[bad[:5]], m2[bad[:5]])


def _table(keys, W, kind):
    from modin_b200 import _lib, ops

    flags = _lib.GB_SUM | _lib.GB_COUNT | _lib.GB_VAR
    if kind in ("hashed", "skewed"):
        t = ops.GroupTable(max(1024, len(np.unique(keys))), W, flags)
    else:
        t = ops.GroupTable.dense(int(keys.min()) if len(keys) else 0, int(keys.max()) if len(keys) else 0, W, flags)
    t.hint_skew(kind == "skewed")
    return t


def _run(keys, Xs, nans, bases, kind):
    from modin_b200 import ops
    from modin_b200.block import DeviceColumn

    t = _table(keys, len(Xs), kind)
    try:
        with env(MB200_GB_SMEM=1 if kind == "small" else 0):
            ops.fill_table(t, [(DeviceColumn.from_numpy(keys),
                                [DeviceColumn.from_numpy(_values(X, m, b)) for X, m, b in zip(Xs, nans, bases)])])  # fmt: skip
        got = ops.emit_counted(t)
    finally:
        t.close()
    _check(keys, Xs, nans, bases, got, merged=False)


ROWS = [0, 1, 31, 33, 255, 256, 257, 4095, 4096, 4097, 1024 * 132 + 5, 1024 * 1056 + 77]


@pytest.mark.parametrize("kind", ["small", "large", "hashed", "skewed"])
@pytest.mark.parametrize("n", ROWS)
def test_tables_within_the_bound(kind, n):
    keys, Xs, nans, bases = _data(n, 3, n + 1, 40 if kind == "small" else 5000, kind)
    if kind == "large" and n:
        keys[0] = 1 << 20  # a range far wider than shared memory holds
    _run(keys, Xs, nans, bases, kind)


@pytest.mark.parametrize("kind", ["small", "large", "hashed"])
@pytest.mark.parametrize("ncols", [1, 8, 9, 32, 40])
def test_column_counts(kind, ncols):
    from modin_b200 import _lib, ops
    from modin_b200.block import DeviceColumn

    keys, Xs, nans, bases = _data(256 * 61 + 13, ncols, ncols, 40 if kind == "small" else 3000, kind)
    if kind == "large":
        keys[0] = 1 << 20
    if ncols <= 32:
        _run(keys, Xs, nans, bases, kind)
        return
    # more columns than one table holds: hash_aggregate splits them and keeps the sums-then-M2s layout
    flags = _lib.GB_SUM | _lib.GB_COUNT | _lib.GB_VAR
    with env(MB200_GB_SMEM=1 if kind == "small" else 0):
        got = ops.hash_aggregate([(DeviceColumn.from_numpy(keys),
                                   [DeviceColumn.from_numpy(_values(X, m, b)) for X, m, b in zip(Xs, nans, bases)])],
                                 flags, 3000)  # fmt: skip
    _check(keys, Xs, nans, bases, got, merged=False)


@pytest.mark.parametrize("kind", ["small", "large", "hashed"])
def test_partial_merges_within_the_bound(kind):
    """Three tables over three row ranges, their emits concatenated and merged: pass 1 on the partial sums / counts,
    pass 2 on the partial rows (S_p, n_p, M2_p)."""
    from modin_b200 import _lib, ops
    from modin_b200.block import DeviceColumn

    n = 1024 * 132 + 5
    keys, Xs, nans, bases = _data(n, 9, 7, 40 if kind == "small" else 5000, kind)
    if kind == "large":
        keys[0] = 1 << 20
    parts = []
    for a, b in ((0, 1000), (1000, 70_001), (70_001, n)):
        t = _table(keys[a:b], 9, kind)
        try:
            ops.fill_table(t, [(DeviceColumn.from_numpy(keys[a:b]),
                                [DeviceColumn.from_numpy(_values(X[a:b], m[a:b], bb)) for X, m, bb in zip(Xs, nans, bases)])])  # fmt: skip
            parts.append(ops.emit_counted(t))
        finally:
            t.close()
    cat = lambda cols: DeviceColumn.from_numpy(np.concatenate([c.to_numpy() for c in cols]))  # noqa: E731
    pk = cat([p[0] for p in parts])
    sums = [cat([p[1][j] for p in parts]) for j in range(18)]
    cnts = [cat([p[2][j] for p in parts]) for j in range(9)]
    flags = _lib.GB_SUM | _lib.GB_COUNT | _lib.GB_VAR
    with env(MB200_GB_SMEM=1 if kind == "small" else 0):
        got = ops.hash_aggregate([(pk, sums, cnts, None)], flags, len(pk), partial=True)
    _check(keys, Xs, nans, bases, got, merged=True)


def test_two_to_the_25_rows():
    n = (1 << 25) + 3
    keys, Xs, nans, bases = _data(n, 3, 9, 100_000, "hashed")
    for kind in ("small", "large", "hashed"):
        _run(keys % 64 if kind == "small" else keys, Xs, nans, bases, kind)


def test_var_tables_refuse_what_they_cannot_do():
    from modin_b200 import _lib, ops
    from modin_b200.block import DeviceColumn

    flags = _lib.GB_SUM | _lib.GB_COUNT | _lib.GB_VAR
    keys = DeviceColumn.from_numpy(np.arange(8, dtype=np.int64))
    vals = [DeviceColumn.from_numpy(np.arange(8.0))]
    for dense in (False, True):
        t = ops.GroupTable.dense(0, 7, 1, flags) if dense else ops.GroupTable(64, 1, flags)
        try:
            t.accumulate(keys, vals)
            t.accumulate_m2(keys, vals)
            with pytest.raises(_lib.B200Error):
                t.accumulate(keys, vals)  # the means are final once pass 2 has run
            with pytest.raises(_lib.B200Error):
                t.merge_partial(keys, vals, [DeviceColumn.from_numpy(np.ones(8, dtype=np.int64))])
            t.accumulate_m2(keys, vals)  # pass 2 may run again
            _, s, c, _ = ops.emit_counted(t)
            assert s[1].to_numpy().tolist() == [0.0] * 8
        finally:
            t.close()
    for bad in (_lib.GB_VAR, _lib.GB_SUM | _lib.GB_VAR, flags | _lib.GB_SIZE, _lib.GB_COUNT | _lib.GB_VAR,
                _lib.GB_MIN | _lib.GB_COUNT | _lib.GB_VAR):  # fmt: skip
        with pytest.raises(_lib.B200Error):
            ops.GroupTable(64, 1, bad)
    t = ops.GroupTable(64, 1, _lib.GB_SUM | _lib.GB_COUNT)
    try:
        with pytest.raises(_lib.B200Error):
            t.accumulate_m2(keys, vals)  # not a VAR table
    finally:
        t.close()


@pytest.mark.parametrize("nparts", [1, 3])
def test_special_values_match_pandas(nparts):
    """Infinities give NaN, squares that overflow inf, -0.0 is a zero, int64 values above 2^53 go through float64, and
    a constant 0.1 group is within the bound of pandas' exact 0.0."""
    import modin_b200.pandas as bpd
    from modin_b200 import config

    old = config.NPartitions.get()
    config.NPartitions.put(nparts)
    try:
        key = np.repeat(np.arange(6, dtype=np.int64), 4)
        x = np.array([2.0, 3.0, np.inf, 1.0, 1e300, -1e300, np.nan, np.nan, -0.0, 0.0, -0.0, np.nan,
                      0.1, 0.1, 0.1, 0.1, np.inf, np.inf, 5.0, np.nan, np.nan, np.nan, np.nan, np.nan])  # fmt: skip
        big = np.array([2**53 + 1, 2**60, -(2**62), 7] * 6, dtype=np.int64)
        pdf = pandas.DataFrame({"key": key, "x": x, "big": big, "b": np.arange(24) % 3 == 0})
        for fn in ("var", "std"):
            for ddof in (0, 1, -1):
                got = getattr(bpd.DataFrame(pdf).groupby("key"), fn)(ddof=ddof)._to_pandas()
                want = getattr(pdf.groupby("key"), fn)(ddof=ddof)
                assert list(got.dtypes) == list(want.dtypes) and np.array_equal(got.index, want.index)
                for c in want.columns:
                    a, b = got[c].to_numpy(), want[c].to_numpy()
                    assert np.array_equal(np.isnan(a), np.isnan(b)), (fn, ddof, c, a, b)
                    ok = ~np.isnan(b)
                    np.testing.assert_allclose(a[ok], b[ok], rtol=1e-12, atol=1e-15)
        got = bpd.DataFrame(pdf).groupby("key").var()._to_pandas()
        assert got.loc[0, "x"] != got.loc[0, "x"] and got.loc[1, "x"] == np.inf and got.loc[2, "x"] == 0.0
        assert abs(got.loc[3, "x"]) <= _bound(4, 0.0, 0.1, nparts > 1) / 3
    finally:
        config.NPartitions.put(old)


# ------------------------------------------------------------------ front doors
@pytest.mark.parametrize("case", ["dense", "hashed"])
def test_front_door_at_the_benchmark_shape(case):
    from modin_b200 import config, synth

    n, groups = 1 << 26, 1_000_000
    old = config.GroupbyDenseKeys.get()
    config.GroupbyDenseKeys.put(case == "dense")
    try:
        df = synth.device_frame(n, 8, seed=42, nan_per_64k=3000, key_modulus=groups)
        pdf = df._to_pandas()
        for fn, ddof in (("var", 1), ("std", 0)):
            want = getattr(pdf.groupby("key"), fn)(ddof=ddof)
            got = getattr(df.groupby("key"), fn)(ddof=ddof)._to_pandas()
            assert np.array_equal(got.index.to_numpy(), want.index.to_numpy())
            assert list(got.dtypes) == list(want.dtypes)
            for c in want.columns:
                a, b = got[c].to_numpy(), want[c].to_numpy()
                assert np.array_equal(np.isnan(a), np.isnan(b)), (fn, c)
                np.testing.assert_allclose(a[~np.isnan(a)], b[~np.isnan(b)], rtol=1e-10, atol=1e-13)
    finally:
        config.GroupbyDenseKeys.put(old)
