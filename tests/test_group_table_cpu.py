"""The group-table driver of ``ops.hash_aggregate`` and the fused dense groupby -- dense-or-hashed choice, regrowth of
an overflowed hash table, the split of more than MAX_COLS value columns, host round trips -- on the numpy device
double (tests/cpu_double.py), which stands in for the table only.  Results are compared with pandas."""

import numpy as np
import pandas
import pytest

from modin_b200 import _lib, config, ops, synth
from tests import cpu_double
from tests.cpu_double import _col, _np

FLAGS = {"sum": _lib.GB_SUM, "count": _lib.GB_COUNT, "min": _lib.GB_MIN, "max": _lib.GB_MAX, "size": _lib.GB_SIZE}


@pytest.fixture
def tables(cpu_device):
    """The double's table log and round-trip counter, cleared; the groupby switches restored afterwards."""
    saved = [(p, p.get()) for p in (config.NPartitions, config.GroupbyDenseKeys, config.GroupbyAsyncEmit)]
    cpu_double.GroupTable.created.clear()
    cpu_double.GroupTable.round_trips = 0
    yield cpu_double.GroupTable
    for p, v in saved:
        p.put(v)


def _reset(log):
    log.created.clear()
    log.round_trips = 0


def _wide_keys(G, reps, seed):
    k = (np.arange(G, dtype=np.int64) - G // 2) * 1_000_003_019  # range ~5e12: the dense table is refused
    return k[np.random.RandomState(seed).permutation(np.tile(np.arange(G), reps))]


def _values(n, seed):
    v = np.random.RandomState(seed).randn(n)
    v[np.random.RandomState(seed + 1).rand(n) < 0.1] = np.nan
    return v


def _emitted(res, agg):
    """The one result column of ``agg`` out of hash_aggregate's (keys, sums, cnts, sizes)."""
    return _np(res[3]) if agg == "size" else _np((res[2] if agg == "count" else res[1])[0])


def _check(got, want, agg):
    if agg == "sum":
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
    else:
        np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("agg", list(FLAGS))
def test_hash_table_regrowth(tables, agg):
    keys = _wide_keys(5000, 2, 7)
    v = _values(len(keys), 8)
    assert not ops.dense_range_ok(int(keys.min()), int(keys.max()), 1024, len(keys), 1, FLAGS[agg])
    want = pandas.DataFrame({"k": keys, "v": v}).groupby("k")["v"].agg(agg)
    res = ops.hash_aggregate([(_col(keys), [_col(v)])], FLAGS[agg], 1024)
    np.testing.assert_array_equal(_np(res[0]), want.index.to_numpy())
    _check(_emitted(res, agg), want.to_numpy(), agg)
    # 1024 -> 4096 groups overflow; the third table holds all 10000 rows: one round trip per attempt
    assert tables.created == ["hashed"] * 3 and tables.round_trips == 3


@pytest.mark.parametrize("agg", list(FLAGS))
def test_hash_table_regrowth_merging_partials(tables, agg):
    keys = _wide_keys(5000, 2, 9)
    pk = np.concatenate([np.unique(keys[: len(keys) // 2]), np.unique(keys[len(keys) // 2 :])])
    pv = np.random.RandomState(10).randn(len(pk))
    pc = np.random.RandomState(11).randint(0, 5, len(pk)).astype(np.int64)
    part = pandas.DataFrame({"k": pk, "v": pv, "c": pc}).groupby("k")
    if agg == "count":
        item, want = (_col(pk), [_col(pc.astype(np.float64))], [_col(pc)], None), part["c"].sum()
    elif agg == "size":
        item, want = (_col(pk), [], None, _col(pc)), part["c"].sum()
    else:
        item, want = (_col(pk), [_col(pv)], None, None), part["v"].agg(agg)
    res = ops.hash_aggregate([item], FLAGS[agg], 1024, partial=True)
    np.testing.assert_array_equal(_np(res[0]), want.index.to_numpy())
    _check(_emitted(res, agg), want.to_numpy(), agg)
    assert tables.created == ["hashed"] * 3 and tables.round_trips == 3


@pytest.mark.parametrize("wide", [False, True])
def test_more_value_columns_than_a_table_holds(tables, wide):
    W = _lib.MAX_COLS + 8
    keys = _wide_keys(700, 3, 12) if wide else np.random.RandomState(12).randint(-50, 650, 2100).astype(np.int64)
    vals = [_values(len(keys), 20 + j) for j in range(W)]
    pdf = pandas.DataFrame({f"c{j}": v for j, v in enumerate(vals)})
    for agg, flags in (("sum", _lib.GB_SUM), ("max", _lib.GB_MAX), ("mean", _lib.GB_SUM | _lib.GB_COUNT)):
        _reset(tables)
        k, s, c, _ = ops.hash_aggregate([(_col(keys), [_col(v) for v in vals])], flags, 1024)
        assert tables.created == ["hashed" if wide else "dense"] * 2  # 32 + 8 value columns
        g = pdf.groupby(keys)
        np.testing.assert_array_equal(_np(k), np.unique(keys))
        if agg == "mean":
            np.testing.assert_allclose(np.column_stack([_np(x) for x in s]), g.sum().to_numpy(), rtol=1e-12, atol=1e-12)
            np.testing.assert_array_equal(np.column_stack([_np(x) for x in c]), g.count().to_numpy())
        else:
            _check(np.column_stack([_np(x) for x in s]), g.agg(agg).to_numpy(), agg)
    # through the front door: the fused path leaves frames this wide to the per-partition tables
    import modin_b200.pandas as bpd

    config.NPartitions.put(4)
    src = pdf.assign(key=keys)
    got = bpd.DataFrame(src).groupby("key").sum()._to_pandas()
    want = src.groupby("key").sum()
    assert list(got.columns) == list(want.columns)
    np.testing.assert_allclose(got.to_numpy(), want.to_numpy(), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("nparts", [1, 4])
@pytest.mark.parametrize("keys", ["narrow", "wide", "dense off"])
def test_which_tables_a_query_creates(tables, keys, nparts):
    import modin_b200.pandas as bpd

    config.NPartitions.put(nparts)
    config.GroupbyDenseKeys.put(keys != "dense off")
    pdf = synth.host_frame(6000, 3, seed=5, nan_per_64k=3000, key_modulus=300)
    if keys == "wide":
        pdf["key"] = pdf["key"] * 1_000_003_019
    df = bpd.DataFrame(pdf)
    _reset(tables)
    got = df.groupby("key").sum()._to_pandas()
    want = pdf.groupby("key").sum()
    np.testing.assert_array_equal(got.index.to_numpy(), want.index.to_numpy())
    np.testing.assert_allclose(got.to_numpy(), want.to_numpy(), rtol=1e-12, atol=1e-12)
    if keys == "narrow":
        # one dense table for every row partition, emitted without a round trip
        assert tables.created == ["dense"] and tables.round_trips == 0
    else:
        # one hash table per row partition, plus one that regroups their partial tables when there are several
        n = nparts + (nparts > 1)
        assert tables.created == ["hashed"] * n and tables.round_trips == n


@pytest.mark.parametrize("agg", ["sum", "count", "size", "min", "max", "mean"])
def test_host_round_trips_of_a_dense_query(tables, agg):
    import modin_b200.pandas as bpd

    config.NPartitions.put(4)
    pdf = synth.host_frame(6000, 3, seed=6, nan_per_64k=3000, key_modulus=300)
    df = bpd.DataFrame(pdf)
    for async_emit in (True, False):
        config.GroupbyAsyncEmit.put(async_emit)
        _reset(tables)
        got = getattr(df.groupby("key"), agg)()._to_pandas()
        want = getattr(pdf.groupby("key"), agg)()
        np.testing.assert_array_equal(got.index.to_numpy(), want.index.to_numpy())
        np.testing.assert_allclose(np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64), rtol=1e-12,
                                   atol=1e-12)  # fmt: skip
        assert tables.created == ["dense"]
        # the count is read back before the emit unless the emit leaves it on the device; mean always counts first
        assert tables.round_trips == (0 if async_emit and agg != "mean" else 1)
