"""Exact references and bit-level comparisons for the GPU suite (no GPU needed).

The README promises bit-exact elementwise ops, predicates, min / max, counts, sizes, keys and merges, and float sums
within ``4 * log2(n) * 2**-53 * sum|x|`` of the true sum.  The references here make those statements checkable as
written: sums are computed exactly (``math.fsum`` / Python integers) and rounded once, so the whole bound is left to the
kernel; comparisons look at float64 bit patterns, so a flipped zero sign or a NaN where ``inf`` belongs is an error.

IEEE overflow is part of every reference: an exact sum outside the float64 range is ``+-inf``, and a sum that has seen
both infinities is NaN.
"""

from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

EPS = 2.0**-53


def assert_bits(got, want, what, zero_sign=True):
    """Float64 bit patterns equal (any NaN equals any NaN); integers and bools exactly equal.  ``zero_sign=False`` lets
    ``-0.0`` and ``0.0`` compare equal -- only for min / max, whose zero sign is unspecified."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, f"{what}: shape {got.shape} vs {want.shape}"
    if want.dtype.kind == "f" or got.dtype.kind == "f":
        g, w = got.astype(np.float64), want.astype(np.float64)
        same = (g.view(np.uint64) == w.view(np.uint64)) | (np.isnan(g) & np.isnan(w))
        if not zero_sign:
            same |= (g == 0) & (w == 0)
        bad = np.flatnonzero(~same.ravel())
        assert bad.size == 0, (f"{what}: {bad.size} elements differ (bit-exact, NaN==NaN"
                               f"{'' if zero_sign else ', -0.0==0.0'}); first at {bad[0]}: "
                               f"got {g.ravel()[bad[0]]!r} want {w.ravel()[bad[0]]!r}")  # fmt: skip
    else:
        assert np.array_equal(got, want), f"{what}: integer/bool mismatch"


assert_exact = assert_bits  # the name the parity tests grew up with


def sum_tolerance(abs_sum, n):
    return 4.0 * max(1.0, math.log2(max(n, 2))) * EPS * abs_sum + 1e-300


def assert_sum_close(got, want, abs_sums, n, what):
    """Float sums within the README bound of ``want`` (per element; NaN == NaN, equal infinities equal)."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, f"{what}: shape"
    tol = np.array([sum_tolerance(a, n) for a in np.asarray(abs_sums, dtype=np.float64).ravel()]).reshape(got.shape)
    both_nan = np.isnan(got) & np.isnan(want)
    ok = both_nan | (np.abs(got - want) <= tol) | (got == want)
    assert ok.all(), f"{what}: max err {np.nanmax(np.abs(got - want))} vs tol {tol.max()}"


def _round_exact(total: Fraction, pos_inf: bool, neg_inf: bool) -> float:
    if pos_inf and neg_inf:
        return math.nan
    if pos_inf or neg_inf:
        return math.inf if pos_inf else -math.inf
    try:
        return float(total)  # int / int true division: correctly rounded
    except OverflowError:
        return math.inf if total > 0 else -math.inf


def _fsum(v: np.ndarray) -> float:
    """Correctly rounded sum of finite and infinite float64 values (no NaN)."""
    pos, neg = bool(np.isposinf(v).any()), bool(np.isneginf(v).any())
    if pos or neg:
        return _round_exact(Fraction(0), pos, neg)
    try:
        return math.fsum(v.tolist())
    except OverflowError:  # fsum raises when the correctly rounded value is out of range
        return _round_exact(sum((Fraction(x) for x in v.tolist()), Fraction(0)), False, False)


def exact_sum(x) -> float:
    """The float64 nearest to the exact sum of the non-NaN values of ``x``.  A zero sum is +0.0 (pandas' column and
    group sums start from +0.0, so even an all ``-0.0`` column sums to +0.0)."""
    x = np.asarray(x, dtype=np.float64).ravel()
    return _fsum(x[~np.isnan(x)]) + 0.0


def exact_group_sums(keys, x):
    """(sorted unique keys, exact per-group sum of the non-NaN values of each column) -- ``x`` is 1-D or [n, W]."""
    keys = np.asarray(keys)
    x = np.asarray(x, dtype=np.float64)
    x2 = x.reshape(len(x), -1)
    uk, inv = np.unique(keys, return_inverse=True)
    order = np.argsort(inv, kind="stable")
    bounds = np.searchsorted(inv[order], np.arange(len(uk) + 1))
    out = np.empty((len(uk), x2.shape[1]), dtype=np.float64)
    for g in range(len(uk)):
        rows = order[bounds[g] : bounds[g + 1]]
        for j in range(x2.shape[1]):
            out[g, j] = exact_sum(x2[rows, j])
    return uk, out.reshape((len(uk),) + x.shape[1:])


def exact_prefix_sums(x) -> np.ndarray:
    """pandas' ``cumsum`` computed exactly: NaN rows stay NaN and add +0.0 to the running sum, every other prefix is
    its exact sum rounded once.  A prefix that overflows stays +-inf from there on, as a running float64 sum does (a
    later infinity of the other sign makes it NaN).  Exact zeros carry IEEE's sign: ``-0.0`` while every row so far is
    ``-0.0``.  The running sum is a Python integer in units of 2**-1074 (every float64 is a whole number of those).
    Meant for n up to a few 10^5."""
    x = np.asarray(x, dtype=np.float64).ravel()
    out = np.empty_like(x)
    acc = 0
    pos_inf = neg_inf = False
    neg_zero_only = True
    scale = Fraction(1, 1 << 1074)
    for i, v in enumerate(x.tolist()):
        if v != v:
            out[i] = math.nan
            neg_zero_only = False
            continue
        if v == math.inf:
            pos_inf = True
        elif v == -math.inf:
            neg_inf = True
        else:
            num, den = v.as_integer_ratio()
            acc += num * ((1 << 1074) // den)
        if not (v == 0.0 and math.copysign(1.0, v) < 0):
            neg_zero_only = False
        if acc == 0 and not (pos_inf or neg_inf):
            out[i] = -0.0 if neg_zero_only else 0.0
        else:
            out[i] = _round_exact(acc * scale, pos_inf, neg_inf)
            pos_inf, neg_inf = pos_inf or out[i] == math.inf, neg_inf or out[i] == -math.inf
    return out


def assert_within_sum_bound(got, exact, abs_sum, n, what):
    """``|got - exact| <= 4 * log2(n) * 2**-53 * abs_sum`` element by element (the README bound around the exact
    value); where the exact value is +-inf or NaN, ``got`` must be the same bits class: the same infinity, or NaN."""
    got, exact = np.atleast_1d(np.asarray(got, dtype=np.float64)), np.atleast_1d(np.asarray(exact, dtype=np.float64))
    abs_sum = np.broadcast_to(np.asarray(abs_sum, dtype=np.float64), exact.shape)
    assert got.shape == exact.shape, f"{what}: shape {got.shape} vs {exact.shape}"
    special = ~np.isfinite(exact)
    same_special = (np.isnan(got) & np.isnan(exact)) | (got == exact)
    bad_special = special & ~same_special
    assert not bad_special.any(), (f"{what}: got {got[bad_special][:4]} where the exact value is "
                                   f"{exact[bad_special][:4]}")  # fmt: skip
    tol = 4.0 * max(1.0, math.log2(max(n, 2))) * EPS * abs_sum
    with np.errstate(invalid="ignore", over="ignore"):
        err = np.abs(got - exact)
    bad = ~special & ~(err <= tol)
    assert not bad.any(), (f"{what}: {int(bad.sum())} values outside the bound; first got {got[bad][0]!r} exact "
                           f"{exact[bad][0]!r} tol {tol[bad][0]!r}")  # fmt: skip
