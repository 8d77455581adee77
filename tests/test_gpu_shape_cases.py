"""The odd-frame-shape tables of ``tests/shape_cases.py`` on the kernels (``-m gpu``): the same cases the CPU device
double runs with ``rtol=1e-12`` (``test_host_shapes_cpu.py``), here compared strictly.

Row labels, column labels and dtypes as pandas; values bit for bit (NaN == NaN), except the cases ``shape_cases.rounded``
names.  A float sum or mean is within ``4 * log2(n) * 2**-53 * sum|x|`` of the exact value on the device and in pandas,
so the two differ by at most twice that; results computed from a group table (``g + g``, ``g.c0 - g.c1``) by at most
twice that again.  ``sum|x|`` is the table's ``abs_sum``.  var / std are within ``test_zzz_gpu_strict_bounds``' relative
bound of pandas.
"""

import math

import numpy as np
import pandas
import pytest

from modin_b200 import config
from tests import shape_cases
from tests.exact import EPS, assert_bits
from tests.test_gpu_parity import _four_partitions, bpd  # noqa: F401  (fixture)
from tests.test_zzz_gpu_strict_bounds import _var_rtol

pytestmark = pytest.mark.gpu


def _values(x):
    """[(label, 1-D array)] of a frame's columns or of a Series."""
    if isinstance(x, pandas.Series):
        return [(x.name, x.to_numpy())]
    return [(c, x.iloc[:, j].to_numpy()) for j, c in enumerate(x.columns)]


def _strict(cases, check_dtypes=True):
    tol = 4.0 * 4.0 * max(1.0, math.log2(max(cases.rows, 2))) * EPS * cases.abs_sum
    checked = 0
    for name, (dev, host) in cases.items():
        want = host()
        got = dev()
        got = got._to_pandas() if hasattr(got, "_to_pandas") else got
        assert type(got) is type(want), f"{name}: {type(got).__name__} vs {type(want).__name__}"
        assert got.shape == want.shape, f"{name}: shape {got.shape} vs {want.shape}"
        assert list(got.index) == list(want.index) and got.index.names == want.index.names, f"{name}: row labels"
        if isinstance(want, pandas.DataFrame):
            assert list(got.columns) == list(want.columns), f"{name}: columns"
        if check_dtypes:
            gd = [str(t) for t in (got.dtypes if isinstance(got, pandas.DataFrame) else [got.dtype])]
            wd = [str(t) for t in (want.dtypes if isinstance(want, pandas.DataFrame) else [want.dtype])]
            assert gd == wd, f"{name}: dtypes {gd[:4]} vs {wd[:4]}"
        for (label, g), (_, w) in zip(_values(got), _values(want)):
            what = f"{name} [{label}]"
            if not shape_cases.rounded(name) or w.dtype.kind != "f":
                assert_bits(g, w, what)
                continue
            g = g.astype(np.float64)
            special = ~np.isfinite(w)
            assert_bits(g[special], w[special], f"{what}: NaN / inf where pandas has them")
            err = np.abs(g[~special] - w[~special])
            if any(k in name for k in ("var", "std")):
                bound = _var_rtol(cases.rows) * np.abs(w[~special])
            else:
                bound = np.full(err.shape, tol)
            assert (err <= bound).all(), f"{what}: max error {err.max()} over the bound {bound.max()}"
        checked += 1
    assert checked == len(cases)


@pytest.fixture
def frames():
    return (bpd(),) + shape_cases.frames()


def test_concatenated_frames(frames):
    _strict(shape_cases.concatenated(*frames), check_dtypes=False)


def test_empty_and_one_row_frames(frames):
    _strict(shape_cases.empty_and_one_row(*frames), check_dtypes=False)


def test_int64_bool_and_mixed_value_columns():
    cases, refused = shape_cases.int64_bool_and_mixed(bpd())
    _strict(cases)
    for call in refused:
        with pytest.raises(NotImplementedError):
            call()


def test_wide_frames(frames):
    m, pa, _, dim = frames
    cases, reductions = shape_cases.wide(m, pa, dim)
    _strict(cases, check_dtypes=False)
    _strict(reductions)


def test_frames_whose_labels_are_not_a_plain_range(frames):
    m, pa, _, dim = frames
    cases, ds = shape_cases.non_range_labels(m, pa, dim)
    _strict(cases, check_dtypes=False)
    with pytest.raises(NotImplementedError, match="numeric / range row labels"):
        ds[ds["c0"] > 0.0]._to_pandas()


def test_binary_operand_shapes():
    cases, dw, roww = shape_cases.binary_operand_shapes(bpd())
    _strict(cases)
    with pytest.raises(ValueError, match="length must be 40"):
        (dw + roww[:-1])._to_pandas()


@pytest.mark.parametrize("dense", [True, False])
def test_groupby_across_key_kinds(dense):
    old = config.GroupbyDenseKeys.get()
    config.GroupbyDenseKeys.put(dense)
    try:
        _strict(shape_cases.groupby_kinds(bpd()))
    finally:
        config.GroupbyDenseKeys.put(old)


def test_merge_across_dim_and_fact_kinds():
    _strict(shape_cases.merge_kinds(bpd()))
