"""Odd frame SHAPES through the API on the CPU device double: frames made of several unequal row partitions whose
range labels restart (what a row-wise concat produces), empty frames (a filter nothing passes) and one-row frames,
flowing into the other operations.  Values, row labels and column labels against pandas.  The case tables live in
``tests/shape_cases.py``; ``test_gpu_shape_cases.py`` runs the same tables on the kernels, bit for bit.

Found with this sweep and fixed: comparisons of an EMPTY frame kept the input dtype instead of giving an empty bool
frame (so ``empty[empty.x > 0]`` and ``(empty > 0).any()`` were refused), and row-wise concatenation demoted restarting
numeric labels to a host index (so ``sort_values`` of a concatenated frame was refused as "non-numeric labels").
"""

import numpy as np
import pandas
import pytest

from modin_b200 import config
from tests import shape_cases


@pytest.fixture(autouse=True)
def _np4():
    old = config.NPartitions.get()
    config.NPartitions.put(4)
    yield
    config.NPartitions.put(old)


def _compare(cases, check_dtypes=False):
    bad = {}
    for name, (dev, host) in cases.items():
        want = host()
        g = dev()
        g = g._to_pandas() if hasattr(g, "_to_pandas") else g
        labels_ok = list(g.index) == list(want.index) and g.index.name == want.index.name
        cols_ok = not hasattr(want, "columns") or list(g.columns) == list(want.columns)
        vals_ok = g.shape == want.shape and np.allclose(np.asarray(g, dtype=np.float64), np.asarray(want, dtype=np.float64),
                                                        rtol=1e-12, atol=1e-9, equal_nan=True)  # fmt: skip
        gd = [str(t) for t in (g.dtypes if hasattr(g, "columns") else [g.dtype])]
        wd = [str(t) for t in (want.dtypes if hasattr(want, "columns") else [want.dtype])]
        dtypes_ok = gd == wd or not check_dtypes
        if not (labels_ok and cols_ok and vals_ok and dtypes_ok):
            bad[name] = (f"values {vals_ok}, labels {labels_ok}, columns {cols_ok}, shape {g.shape} vs {want.shape}, "
                         f"dtypes {gd} vs {wd}")  # fmt: skip
    assert not bad, bad


@pytest.fixture
def frames(cpu_device):
    import modin_b200.pandas as bpd

    return (bpd,) + shape_cases.frames()


def test_concatenated_frames_flow_into_the_other_operations(frames):
    _compare(shape_cases.concatenated(*frames))


def test_empty_and_one_row_frames(frames):
    _compare(shape_cases.empty_and_one_row(*frames))


def test_int64_bool_and_mixed_value_columns(cpu_device):
    """The synthetic frames are float64; int64 and bool VALUE columns take the promotion / widening paths.  Values,
    labels and the result dtypes against pandas; what is not on the path is refused, never approximated."""
    import modin_b200.pandas as bpd

    cases, refused = shape_cases.int64_bool_and_mixed(bpd)
    _compare(cases, check_dtypes=True)
    for call in refused:
        with pytest.raises(NotImplementedError):
            call()
    with pytest.raises(NotImplementedError, match="groupby.min"):
        refused[2]()


def test_wide_frames_use_the_2d_grid_everywhere(frames):
    """More than 32 columns: several column partitions, so every operation sees a 2-D grid of blocks."""
    bpd, pa, pb, dim = frames
    cases, reductions = shape_cases.wide(bpd, pa, dim)
    _compare(cases)
    _compare(reductions, check_dtypes=True)


def test_frames_whose_labels_are_not_a_plain_range(frames):
    bpd, pa, pb, dim = frames
    cases, ds = shape_cases.non_range_labels(bpd, pa, dim)
    _compare(cases)
    with pytest.raises(NotImplementedError, match="numeric / range row labels"):
        ds[ds["c0"] > 0.0]._to_pandas()  # string labels cannot ride through the device compaction: refused, not dropped



def test_sort_values_treats_the_two_zeros_as_a_tie(cpu_device):
    """pandas sorts ``-0.0`` and ``0.0`` as a tie: rows keep their order.  The device sort key folds ``-0.0`` into
    ``0.0`` before it orders the bits; the gathered values keep theirs."""
    import modin_b200.pandas as bpd

    x = np.array([0.0, -0.0, 1.0, -0.0, 0.0, np.nan, -1.0, -0.0, np.inf, 0.0, -np.inf] * 37)
    pdf = pandas.DataFrame({"x": x, "v": np.arange(len(x), dtype=np.float64)})
    df = bpd.DataFrame(pdf)
    for asc in (True, False):
        got = df.sort_values("x", ascending=asc)._to_pandas()
        want = pdf.sort_values("x", ascending=asc, kind="stable")
        assert list(got.index) == list(want.index), f"sort ascending={asc}: row order"
        assert np.array_equal(got.to_numpy().view(np.int64), want.to_numpy().view(np.int64)), f"sort ascending={asc}: bits"


def test_alignment_matches_a_negative_zero_label_to_zero(cpu_device):
    """Frames with different float row labels are re-indexed onto the joined labels; pandas matches a ``-0.0`` label
    in one frame to the ``0.0`` of the other."""
    import modin_b200.pandas as bpd

    a = pandas.DataFrame({"c": [1.0, 2.0, 4.0, 8.0]}, index=pandas.Index([0.0, 1.0, 2.0, 5.0]))
    b = pandas.DataFrame({"c": [16.0, 32.0, 64.0]}, index=pandas.Index([-0.0, 1.0, 3.0]))
    for left, right in ((a, b), (b, a)):
        got = (bpd.DataFrame(left) + bpd.DataFrame(right))._to_pandas()
        want = left + right
        assert list(got.index) == list(want.index)
        assert np.array_equal(got["c"].to_numpy(), want["c"].to_numpy(), equal_nan=True), (got, want)


def test_binary_template_operand_shapes_are_bit_exact(cpu_device):
    """The Binary template's operand shapes on plain, wide (two column partitions), filtered and int64 frames: values
    bit for bit, labels and dtypes as pandas.  Found with this sweep and fixed: a positional row vector (list) on a
    frame with several column partitions reached every partition whole."""
    import modin_b200.pandas as bpd

    cases, dw, roww = shape_cases.binary_operand_shapes(bpd)
    bad = {}
    for name, (dev, host) in cases.items():
        want = host()
        g = dev()
        g = g._to_pandas() if hasattr(g, "_to_pandas") else g
        gv, wv = np.asarray(g, dtype=np.float64), np.asarray(want, dtype=np.float64)
        exact = g.shape == want.shape and bool(((gv == wv) | (np.isnan(gv) & np.isnan(wv))).all())
        if name == "round then sum":  # a reduction: summation order, not bit-exact
            exact = g.shape == want.shape and np.allclose(gv, wv, rtol=0, atol=1e-9)
        gd = [str(t) for t in (g.dtypes if hasattr(g, "columns") else [g.dtype])]
        wd = [str(t) for t in (want.dtypes if hasattr(want, "columns") else [want.dtype])]
        cols_ok = not hasattr(want, "columns") or list(g.columns) == list(want.columns)
        if not (exact and list(g.index) == list(want.index) and cols_ok and gd == wd):
            bad[name] = (exact, gd[:3], wd[:3])
    assert not bad and len(cases) >= 60, bad
    with pytest.raises(ValueError, match="length must be 40"):
        (dw + roww[:-1])._to_pandas()


@pytest.mark.parametrize("dense", [True, False])
def test_groupby_aggregations_across_key_kinds_and_shapes(cpu_device, dense):
    """Every aggregation x key kind x input kind, through the dense-table path and the hash / regroup path; plus
    dictionary and multi-key aggregation.  Keys, columns, dtypes and values against pandas."""
    import modin_b200.pandas as bpd

    config.GroupbyDenseKeys.put(dense)
    try:
        _compare(shape_cases.groupby_kinds(bpd), check_dtypes=True)
    finally:
        config.GroupbyDenseKeys.put(True)


def test_broadcast_merge_across_dim_and_fact_kinds(cpu_device):
    """fact.merge(dim) across dim, fact and input kinds, bit for bit, with dtypes, against pandas.  (The dense and the
    hashed dim table differ only below the C ABI; the ``gpu`` merge tests cover both.)"""
    import modin_b200.pandas as bpd

    bad = {}
    for name, (dev, host) in shape_cases.merge_kinds(bpd).items():
        want, g = host(), dev()._to_pandas()
        gv, wv = np.asarray(g, dtype=np.float64), np.asarray(want, dtype=np.float64)
        ok = (list(g.columns) == list(want.columns) and list(g.index) == list(want.index) and gv.shape == wv.shape
              and bool(((gv == wv) | (np.isnan(gv) & np.isnan(wv))).all())
              and [str(t) for t in g.dtypes] == [str(t) for t in want.dtypes])  # fmt: skip
        if not ok:
            bad[name] = (gv.shape, wv.shape)
    assert not bad, bad


def test_left_merge_never_fills_a_bool_payload_with_false(cpu_device):
    """A left join whose bool payload column meets an unmatched left row: pandas gives object dtype (NaN for the miss),
    which is refused, with unique and with repeated dim keys.  Without misses the bool column is gathered."""
    import modin_b200.pandas as bpd

    fact = pandas.DataFrame({"key": np.array([0, 1, 2, 3, 9], dtype=np.int64), "x": np.arange(5.0)})
    for keys in ([0, 1, 2, 3], [0, 1, 1, 2, 3, 3]):
        dim = pandas.DataFrame({"key": np.array(keys, dtype=np.int64), "b": np.arange(len(keys)) % 2 == 0})
        with pytest.raises(NotImplementedError, match="bool payload"):
            bpd.DataFrame(fact).merge(bpd.DataFrame(dim), on="key", how="left")._to_pandas()
        hit = fact[fact["key"] < 4]
        _compare({"left without misses": (lambda: bpd.DataFrame(hit).merge(bpd.DataFrame(dim), on="key", how="left"),
                                          lambda: hit.merge(dim, on="key", how="left")),
                  "inner": (lambda: bpd.DataFrame(fact).merge(bpd.DataFrame(dim), on="key", how="inner"),
                            lambda: fact.merge(dim, on="key", how="inner"))}, check_dtypes=True)  # fmt: skip


def test_int64_cumsum_stays_exact_and_wraps(cpu_device):
    """int64 cumulative sums are exact and wrap like numpy's (the double once ran them through float64)."""
    import modin_b200.pandas as bpd

    i = np.array([2**62 + 1, 2**62 + 3, 2**62, -7, 2**53 + 1, -(2**63)], dtype=np.int64)
    pdf = pandas.DataFrame({"i": np.tile(i, 50)})
    got = bpd.DataFrame(pdf)._query_compiler.cumsum(0).to_pandas()
    assert got["i"].dtype == np.int64 and np.array_equal(got["i"].to_numpy(), np.cumsum(pdf["i"].to_numpy()))
