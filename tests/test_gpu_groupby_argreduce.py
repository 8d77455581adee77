"""``groupby.idxmax`` / ``idxmin`` on the H100, bit for bit against numpy.

The two-pass ARGMAX / ARGMIN kernels through ``ops.GroupTable``: every table kind (dense over a small range -- the
per-CTA shared-memory tables --, dense over a large range and hashed, both on direct loads), row counts around warp,
256-row, 4096-row and grid boundaries up to 2^25 + 3, winners planted on both sides of those boundaries and at the
tail, ``-0.0`` before ``0.0`` and the reverse, int64 extremes, and 1 to 40 columns mixing float64 / int64 / bool.
Then both aggregations through the mirror at the benchmark's groupby shape (2^26 rows, 1e6 keys, dense and hashed)
against pandas."""

import contextlib
import os

import numpy as np
import pandas
import pytest

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max


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


def _image(x):
    if x.dtype != np.float64:
        return x.astype(np.int64)
    b = np.where(x == 0.0, 0.0, x).view(np.int64)  # -0.0 and 0.0 tie
    return b ^ ((b >> 63) & np.int64(0x7FFFFFFFFFFFFFFF))


def _reference(keys, col, fn):
    """Ascending unique keys of all rows and, per key, the first row holding the extreme non-NaN value (-1: none)."""
    uk = np.unique(keys)
    ok = ~np.isnan(col) if col.dtype == np.float64 else np.ones(len(col), dtype=bool)
    rows, k, img = np.flatnonzero(ok), keys[ok], _image(col[ok])
    order = np.lexsort((rows, img if fn == "idxmin" else ~img, k))  # ~ reverses the int64 order exactly
    ks = k[order]
    first = np.r_[True, ks[1:] != ks[:-1]] if len(ks) else np.zeros(0, dtype=bool)
    out = np.full(len(uk), -1, dtype=np.int64)
    out[np.searchsorted(uk, ks[first])] = rows[order][first]
    return uk, out


def _planted(n, ncols, seed, G):
    """Keys over [0, G); columns cycle float64 (NaN, signed zeros, infinities) / int64 (limits) / bool (0 / 1 int64).
    Special keys G, G + 1, ... occur only at planted row pairs that hold EQUAL extremes -- row 0 with the last row, and
    both sides of every warp (32), 256-, 1024- and 4096-row cut -- so the earlier row must win."""
    rng = np.random.default_rng(seed)
    keys = rng.integers(0, G, n).astype(np.int64)
    cols = []
    for j in range(ncols):
        if j % 3 == 0:
            v = rng.choice([-0.0, 0.0, np.inf, -np.inf, 1.5, -2.5, np.nan], n)
        elif j % 3 == 1:
            v = rng.choice(np.array([I64_MIN, I64_MAX, 0, -7, 7], dtype=np.int64), n)
        else:
            v = (rng.random(n) < 0.5).astype(np.int64)
        cols.append(v)
    cuts = sorted({c for step in (32, 256, 1024, 4096, 1 << 17) for r in (range(step, n, step),)
                   for c in list(r[:300]) + list(r[-100:])})  # fmt: skip
    pairs = ([(0, n - 1)] if n > 1 else []) + [(c - 1, c) for c in cuts]
    special = G
    for a, b in pairs:
        keys[[a, b]] = special
        for j, v in enumerate(cols):
            v[a] = v[b] = (-0.0 if special % 2 else 0.0) if j % 3 == 0 else (I64_MIN if special % 2 else I64_MAX)
            if j % 3 == 0 and special % 3 == 0:
                v[b] = -v[a]  # -0.0 before 0.0 and the reverse
        special += 1
    return keys, cols


def _run(keys, cols, fn, kind):
    from modin_b200 import _lib, ops
    from modin_b200.block import DeviceColumn

    flag = _lib.GB_ARGMAX if fn == "idxmax" else _lib.GB_ARGMIN
    dk = DeviceColumn.from_numpy(keys)
    dv = [DeviceColumn.from_numpy(v) for v in cols]
    if kind == "hashed":
        table = ops.GroupTable(max(1024, len(np.unique(keys))), len(cols), flag)
    else:
        table = ops.GroupTable.dense(int(keys.min()) if len(keys) else 0, int(keys.max()) if len(keys) else 0,
                                     len(cols), flag)  # fmt: skip
    try:
        with env(MB200_GB_SMEM=1 if kind == "small" else 0):
            table.accumulate(dk, dv)
        k, pos, _, _ = ops.emit_counted(table)
    finally:
        table.close()
    got_k = k.to_numpy()
    for j, c in enumerate(cols):
        uk, want = _reference(keys, c, fn)
        assert np.array_equal(got_k, uk), (fn, kind)
        got = pos[j].to_numpy()
        assert got.dtype == np.int64 and np.array_equal(got, want), (fn, kind, j, np.flatnonzero(got != want)[:5])


@pytest.mark.parametrize("fn", ["idxmax", "idxmin"])
@pytest.mark.parametrize("kind", ["small", "large", "hashed"])
@pytest.mark.parametrize("n", [0, 1, 31, 33, 255, 256, 257, 4095, 4096, 4097, 1024 * 132 + 5, 1024 * 1056 + 77])
def test_tables_bit_for_bit(fn, kind, n):
    G = 40 if kind == "small" else 5000
    keys, cols = _planted(n, 5, n + 1, G)
    if kind == "large" and n:
        keys[0] = 1 << 20  # a range far wider than shared memory holds
    _run(keys, cols, fn, kind)


@pytest.mark.parametrize("kind", ["small", "large", "hashed"])
@pytest.mark.parametrize("ncols", [1, 2, 8, 9, 17, 32])
def test_column_counts(kind, ncols):
    keys, cols = _planted(256 * 61 + 13, ncols, ncols, 40 if kind == "small" else 3000)
    if kind == "large":
        keys[0] = 1 << 20
    for fn in ("idxmax", "idxmin"):
        _run(keys, cols, fn, kind)


def test_forty_columns_and_two_to_the_25_rows():
    from modin_b200 import _lib, ops
    from modin_b200.block import DeviceColumn

    keys, cols = _planted(256 * 40 + 5, 40, 4, 1000)
    for fn, flag in (("idxmax", _lib.GB_ARGMAX), ("idxmin", _lib.GB_ARGMIN)):
        k, pos, _, _ = ops.hash_aggregate([(DeviceColumn.from_numpy(keys), [DeviceColumn.from_numpy(v) for v in cols])],
                                          flag, 1000)  # fmt: skip
        for j, c in enumerate(cols):
            uk, want = _reference(keys, c, fn)
            assert np.array_equal(k.to_numpy(), uk) and np.array_equal(pos[j].to_numpy(), want), (fn, j)
    n = (1 << 25) + 3
    keys, cols = _planted(n, 3, 9, 100_000)
    for kind in ("small", "large", "hashed"):
        kk = keys % 64 if kind == "small" else keys
        _run(kk, cols, "idxmax", kind)


def test_arg_tables_refuse_what_they_cannot_do():
    from modin_b200 import _lib, ops
    from modin_b200.block import DeviceColumn

    keys = DeviceColumn.from_numpy(np.arange(8, dtype=np.int64))
    vals = [DeviceColumn.from_numpy(np.zeros(8))]
    t = ops.GroupTable(64, 1, _lib.GB_ARGMAX)
    try:
        t.accumulate(keys, vals)
        with pytest.raises(_lib.B200Error):
            t.accumulate(keys, vals)  # one fill per table
        with pytest.raises(_lib.B200Error):
            t.merge_partial(keys, vals)
    finally:
        t.close()
    for bad in (_lib.GB_ARGMAX | _lib.GB_SIZE, _lib.GB_ARGMAX | _lib.GB_ARGMIN, _lib.GB_ARGMIN | _lib.GB_MIN):
        with pytest.raises(_lib.B200Error):
            ops.GroupTable(64, 1, bad)
    lib = _lib.load()
    t = ops.GroupTable(64, 1, _lib.GB_ARGMIN)
    try:
        with pytest.raises(_lib.B200Error):
            _lib.check(lib.mb200_gb_accumulate(t.handle, keys.ptr, _lib.ptr_array([vals[0].ptr]), 8, None))
    finally:
        t.close()


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
        for fn in ("idxmax", "idxmin"):
            want = getattr(pdf.groupby("key"), fn)()
            got = getattr(df.groupby("key"), fn)()._to_pandas()
            assert np.array_equal(got.index.to_numpy(), want.index.to_numpy())
            assert list(got.dtypes) == list(want.dtypes)
            for c in want.columns:
                assert np.array_equal(got[c].to_numpy(), want[c].to_numpy()), (fn, c)
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
        f = np.where(rng.random(n) < 0.6, np.nan, rng.choice([-0.0, 0.0, np.inf, -np.inf, 1.25], n))
        f[np.unique(key, return_index=True)[1]] = -np.inf  # every group has a value
        lim = np.where(np.arange(n) % 3 == 0, I64_MIN, I64_MAX).astype(np.int64)
        pdf = pandas.DataFrame({"key": key, "f": f, "i": lim, "b": rng.random(n) < 0.5},
                               index=pandas.RangeIndex(10, 10 + n))  # fmt: skip
        df = bpd.DataFrame(pdf)
        for fn in ("idxmax", "idxmin"):
            got, want = getattr(df.groupby("key"), fn)()._to_pandas(), getattr(pdf.groupby("key"), fn)()
            pandas.testing.assert_frame_equal(got, want)
        nan = pdf.assign(f=np.where(pdf["key"] == 5, np.nan, pdf["f"]))
        with pytest.raises(ValueError, match="all NA values in a group"):
            bpd.DataFrame(nan).groupby("key").idxmax()
    finally:
        config.NPartitions.put(old)
