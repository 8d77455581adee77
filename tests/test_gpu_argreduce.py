"""``idxmax`` / ``idxmin`` on the H100 (``-m gpu``), bit for bit against numpy / pandas, under both reduce variants
(0 = TMA-staged tiles, 1 = direct 128-bit loads).

The kernel (``ops.arg_reduce_columns``) is checked at the row counts its tiling branches on -- the 2048-element TMA
tile, the 4096-element LDG tile and 2^25 + 3 rows (many CTAs per column) -- on views shifted by 1-3 rows (the unaligned
fallback and the odd TMA tail element), with winners planted at the first and last row, on both sides of every tile cut
and with equal extremes in two CTAs, in two tiles of one CTA and in two accumulator lanes of one thread: the first
occurrence must win every time.  Special values: a +-0.0 tie, +-inf and all -inf, the int64 limits, NaN at the
would-be winner and an all-False bool column.  Then 1 to 40 columns through both front doors."""

import os
import sys

import numpy as np
import pandas
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
TMA_TILE, LDG_TILE = 2048, 4096


def _expect(x, op):
    """(value, first row holding it or -1, #non-NaN): the exact answer."""
    ok = ~np.isnan(x) if x.dtype == np.float64 else np.ones(len(x), dtype=bool)
    n = int(ok.sum())
    if n == 0:
        return None, -1, 0
    best = x[ok].max() if op == "max" else x[ok].min()
    return best, int(np.flatnonzero(ok & (x == best))[0]), n


def _device(arrays, shift):
    """Device columns that start ``shift`` elements into their buffers."""
    import torch

    from modin_b200.block import DeviceColumn

    out = []
    for x in arrays:
        buf = torch.from_numpy(np.concatenate([np.zeros(shift, dtype=x.dtype), x])).cuda()
        out.append(DeviceColumn(buf[shift:], x.dtype))
    return out


def _check_kernel(arrays, variant, shift=0):
    from modin_b200 import ops

    cols = _device(arrays, shift)
    for op in ("max", "min"):
        vals, poss, cnts = ops.arg_reduce_columns(op, cols, variant)
        for j, x in enumerate(arrays):
            best, pos, n = _expect(x, op)
            got_pos, got_n = int(poss[j].item()), int(cnts[j].item())
            assert (got_pos, got_n) == (pos, n), (op, j, len(x), variant, shift, got_pos, pos)
            if pos >= 0:
                v = vals[j].cpu().numpy()
                assert v.view(np.uint64)[0] == np.asarray([best], dtype=x.dtype).view(np.uint64)[0], (op, j)


def _noise(n, seed, nan_every=0):
    rng = np.random.default_rng(seed)
    f = rng.standard_normal(n)
    if nan_every:
        f[::nan_every] = np.nan
    return f, rng.integers(-1000, 1000, n)


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("n", [0, 1, 2, 2047, 2048, 2049, 4095, 4096, 4097])
def test_row_counts_and_shifted_views(variant, n):
    f, i = _noise(n, n, nan_every=7)
    ends_f, ends_i = f.copy(), i.copy()
    if n:
        ends_f[-1], ends_i[-1] = 99.0, 10**6  # the maximum on the last row ...
        ends_f[0], ends_i[0] = -99.0, -10**6  # ... and the minimum on the first
    for shift in (0, 1, 2, 3):
        _check_kernel([f, i, ends_f, ends_i], variant, shift)


@pytest.mark.parametrize("variant", [0, 1])
def test_many_ctas_per_column(variant):
    n = (1 << 25) + 3
    f, i = _noise(n, 5, nan_every=1001)
    f[n // 3] = f[n - 2] = 50.0  # equal maxima far apart: the first must win over every CTA cut
    f[7] = f[n - 1] = -50.0
    i[LDG_TILE * 100 + 1] = i[n - 1] = 5000
    _check_kernel([f, i], variant)
    _check_kernel([f], variant, shift=1)


def _planted_columns(n):
    """One column per set of equal extremes; the first position of each set must win."""
    sets = [
        (0,), (n - 1,), (n - 2, n - 1),
        (TMA_TILE - 1, TMA_TILE), (TMA_TILE, TMA_TILE + 1), (LDG_TILE - 1, LDG_TILE), (LDG_TILE, 3 * LDG_TILE - 1),
        (5, TMA_TILE + 5), (TMA_TILE + 5, 2 * TMA_TILE + 5),  # two tiles, two CTAs
        tuple(7 + TMA_TILE * k for k in range(0, n // TMA_TILE, 3)),  # one per third TMA tile: tiles of one CTA
        tuple(9 + LDG_TILE * k for k in range(1, n // LDG_TILE, 2)),
        (10, 11), (11, 522), (10, 11, 522, 523),  # one thread's TMA accumulator lanes (2 tid, 2 tid + 1, 512 + 2 tid)
        (4, 5, 6, 7), (5, 1029), (1028, 1029, 2052),  # one thread's LDG lanes (4 tid + k, 1024 u + 4 tid)
    ]  # fmt: skip
    rng = np.random.default_rng(11)
    out = []
    for s in sets:
        for dt in (np.float64, np.int64):
            x = (rng.random(n) * 100).astype(dt)
            x[list(s)] = 1000
            x[[(p + 3) % n for p in s]] = -1000
            out.append(x)
    return out


@pytest.mark.parametrize("variant", [0, 1])
def test_equal_extremes_first_occurrence_wins(variant):
    n = 64 * LDG_TILE + 3
    cols = _planted_columns(n)
    _check_kernel(cols, variant)
    _check_kernel(cols, variant, shift=1)


def _specials(n=6 * TMA_TILE + 1):
    z = np.zeros(n)
    z[1::2] = -0.0  # 0.0 and -0.0 tie: the first row wins both ways
    nz = -z
    pinf = np.zeros(n)
    pinf[[3, TMA_TILE, n - 1]] = np.inf
    pinf[[2, TMA_TILE + 1]] = -np.inf
    ninf = np.full(n, -np.inf)
    allpinf = np.full(n, np.inf)
    lim = np.where(np.arange(n) % 5 == 0, I64_MAX, np.where(np.arange(n) % 5 == 1, I64_MIN, 3))
    allmin = np.full(n, I64_MIN)
    nanwin = np.arange(n, dtype=np.float64)
    nanwin[[n - 1, 0]] = np.nan  # NaN where the maximum / minimum would be
    allnan = np.full(n, np.nan)
    return pandas.DataFrame({"z": z, "nz": nz, "pinf": pinf, "ninf": ninf, "allpinf": allpinf, "lim": lim,
                             "allmin": allmin, "nanwin": nanwin, "false": np.zeros(n, dtype=bool),
                             "bools": np.arange(n) % 997 == 996, "allnan": allnan})  # fmt: skip


@pytest.mark.parametrize("variant", [0, 1])
def test_special_values(variant):
    pdf = _specials()
    arrays = [pdf[c].to_numpy() for c in pdf.columns if pdf[c].dtype != bool]
    _check_kernel(arrays, variant)
    _check_kernel(arrays, variant, shift=3)


@pytest.fixture
def reduce_variant(request):
    from modin_b200 import config

    old = config.ReduceVariant.get()
    config.ReduceVariant.put(request.param)
    yield request.param
    config.ReduceVariant.put(old)


def _front_door_cases():
    sp = _specials().drop(columns="allnan")
    rng = np.random.default_rng(4)
    wide = {}
    for j in range(40):
        k = j % 3
        if k == 0:
            x = np.round(rng.standard_normal(9001), 1)
            x[rng.random(9001) < 0.1] = np.nan
        elif k == 1:
            x = rng.integers(-50, 50, 9001)
        else:
            x = rng.random(9001) < 0.01 * (j % 5)
        wide[f"c{j}"] = x
    wide = pandas.DataFrame(wide)
    cases = {"specials": sp, "float labels": sp.set_axis(pandas.Index(np.arange(len(sp)) * 0.25 + 1.0)),
             "range offset": sp.set_axis(pandas.RangeIndex(1000, 1000 + len(sp)))}  # fmt: skip
    for w in (1, 7, 8, 9, 31, 32, 33, 40):
        cases[f"{w} columns"] = wide.iloc[:, :w]
    rep = pandas.concat([wide.iloc[:5000, :9], wide.iloc[2000:, :9]])
    cases["repeated labels"] = rep
    return cases


@pytest.mark.parametrize("reduce_variant", [0, 1], indirect=True)
def test_mirror_front_door_matches_pandas(reduce_variant):
    import modin_b200.pandas as bpd
    from modin_b200 import config

    old = config.NPartitions.get()
    config.NPartitions.put(4)
    try:
        for name, pdf in _front_door_cases().items():
            df = bpd.DataFrame(pdf)
            for op in ("idxmax", "idxmin"):
                got, want = getattr(df, op)(), getattr(pdf, op)()
                pandas.testing.assert_series_equal(got, want, check_index_type=False, obj=f"{name} {op}")
        masked = _front_door_cases()["9 columns"].drop(columns=["c2", "c5", "c8"])
        keep = masked["c1"] > 0
        dm = bpd.DataFrame(masked)
        dm = dm[dm["c1"] > 0]
        pandas.testing.assert_series_equal(dm.idxmax(), masked[keep].idxmax(), check_index_type=False)
        s, ps = bpd.DataFrame(masked)["c0"], masked["c0"]
        assert (s.idxmax(), s.idxmin(), s.argmax(), s.argmin()) == (ps.idxmax(), ps.idxmin(), ps.argmax(), ps.argmin())
        with pytest.raises(ValueError, match="Encountered all NA values"):
            bpd.DataFrame(_specials()[["z", "allnan"]]).idxmax()
    finally:
        config.NPartitions.put(old)


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "modin")), reason="reference Modin not installed under oracle/_ref")
def test_modin_front_door_matches_pandas():
    if REF not in sys.path:
        sys.path.insert(0, REF)
    import warnings

    warnings.filterwarnings("ignore")
    from modin_b200 import _lib, config, modin_plugin

    modin_plugin.register()
    import modin
    import modin.config as cfg
    import modin.pandas as mpd

    modin.set_execution(engine="B200", storage_format="Arrow")
    cfg.NPartitions.put(4)
    old = config.NPartitions.get()
    config.NPartitions.put(4)
    lib = _lib.load()
    before = lib.mb200_launch_count()
    try:
        for name, pdf in _front_door_cases().items():
            df = mpd.DataFrame(pdf)
            for op in ("idxmax", "idxmin"):
                got, want = getattr(df, op)()._to_pandas(), getattr(pdf, op)()
                pandas.testing.assert_series_equal(got, want, check_index_type=False, obj=f"{name} {op}")
        ps = _specials()["nanwin"]
        s = mpd.DataFrame(_specials())["nanwin"]
        assert (s.idxmax(), s.argmax(), s.argmin()) == (ps.idxmax(), ps.argmax(), ps.argmin())
    finally:
        config.NPartitions.put(old)
    assert lib.mb200_launch_count() > before
