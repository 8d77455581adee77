"""The two query compilers share one definition of their device operations (``query_compiler.device_operations``):
every shared name resolves to it on both classes except the declared overrides, and every shared operation gives the
same answer through both front doors -- the Modin-free ``modin_b200.pandas`` and real ``modin.pandas`` with the
plug-in -- on the numpy device double.  "The same" is bit for bit: values, dtypes, row and column labels, and the
error type of each refusal."""

import os
import sys

import numpy as np
import pandas
import pytest

from modin_b200 import config
from modin_b200.query_compiler import B200QueryCompiler

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")

needs_modin = pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "modin")),
                                 reason="reference Modin not installed under oracle/_ref")  # fmt: skip

# names each query compiler defines itself, in front of the shared definition
MIRROR_OVERRIDES = {"var", "std"}  # host Series for the mirror's API layer
PLUGIN_OVERRIDES = {"add", "radd", "sub", "rsub", "mul", "rmul", "truediv", "rtruediv"} | {  # scalar fast path
    f"groupby_{agg}" for agg in ("sum", "count", "size", "mean", "min", "max")  # groupby(level=)
}
_CLASS_ATTRS = {"__module__", "__qualname__", "__doc__", "__dict__", "__weakref__", "__firstlineno__",
                "__static_attributes__"}  # fmt: skip


@pytest.fixture(scope="module")
def plugin():
    if REF not in sys.path:
        sys.path.insert(0, REF)
    import warnings

    warnings.filterwarnings("ignore")
    from modin_b200 import modin_plugin

    ns = modin_plugin.register()
    import modin
    import modin.config as cfg
    import modin.pandas as mpd

    modin.set_execution(engine="B200", storage_format="Arrow")
    old = cfg.NPartitions.get(), config.NPartitions.get()
    cfg.NPartitions.put(3)
    config.NPartitions.put(3)
    yield ns, mpd
    cfg.NPartitions.put(old[0])
    config.NPartitions.put(old[1])


def _shared_base(cls):
    return next(c for c in cls.__mro__ if c.__name__ == "DeviceOperations")


def _owner(cls, name):
    return next(c for c in cls.__mro__ if name in vars(c))


@needs_modin
def test_shared_names_resolve_to_the_shared_definition(plugin):
    ns, _ = plugin
    mirror, plug = _shared_base(B200QueryCompiler), _shared_base(ns.QueryCompiler)
    names = set(vars(mirror)) - _CLASS_ATTRS
    assert names == set(vars(plug)) - _CLASS_ATTRS
    assert {"fillna", "astype", "merge", "groupby_agg", "groupby_sum", "count", "idxmax", "cumsum"} <= names
    for cls, base, overrides in ((B200QueryCompiler, mirror, MIRROR_OVERRIDES), (ns.QueryCompiler, plug, PLUGIN_OVERRIDES)):
        assert overrides <= names, cls
        wrong = {n for n in names - overrides if _owner(cls, n) is not base}
        assert not wrong, (cls.__name__, wrong)
        assert all(_owner(cls, n) is cls for n in overrides), cls.__name__
    # the methods written in the shared definition are one piece of code for both
    for n in names:
        fm, fp = vars(mirror)[n], vars(plug)[n]
        if callable(fm) and getattr(fm, "__qualname__", "").startswith("device_operations."):
            assert fm.__code__ is fp.__code__, n


# ------------------------------------------------------------------ the sweep
def _frames():
    rng = np.random.RandomState(5)
    n = 301
    vals = pandas.DataFrame({"a": rng.randn(n), "b": rng.randn(n) * 3.0, "c": np.round(rng.randn(n), 1)})
    vals.loc[rng.rand(n) < 0.2, "a"] = np.nan
    vals.loc[rng.rand(n) < 0.1, "c"] = np.nan
    vals.loc[::37, "b"] = -0.0
    other = pandas.DataFrame({c: rng.randn(n) for c in vals.columns})
    other.loc[rng.rand(n) < 0.3, "a"] = np.nan
    keyed = vals.assign(key=rng.randint(-3, 9, n).astype(np.int64), k2=(rng.randint(0, 4, n) * 5 - 7).astype(np.int64))
    mixed = pandas.DataFrame({"i": rng.randint(-50, 50, n).astype(np.int64), "t": rng.rand(n) < 0.4, "f": vals["a"]})
    wide = pandas.DataFrame({f"w{j}": rng.randn(n) for j in range(40)})
    wide.iloc[::7, 3] = np.nan
    wide.insert(0, "key", rng.randint(0, 11, n).astype(np.int64))
    wide.insert(20, "k2", rng.randint(-2, 2, n).astype(np.int64))
    dim = pandas.DataFrame({"key": rng.permutation(12)[:9].astype(np.int64) - 3, "d0": rng.randn(9)})
    return dict(vals=vals, other=other, keyed=keyed, mixed=mixed, wide=wide, dim=dim)


def _cases():
    """(name, frames used, call) -- or (name, frames, mirror call, plug-in call) where the two APIs spell it apart."""
    aggs = ("sum", "count", "mean", "min", "max")
    cases = [
        ("abs", ("vals",), lambda d: d.abs()),
        ("neg", ("vals",), lambda d: -d),
        ("isna", ("vals",), lambda d: d.isna()),
        ("notna", ("mixed",), lambda d: d.notna()),
        ("round", ("vals",), lambda d: d.round(1)),
        ("clip", ("vals",), lambda d: d.clip(-0.5, 0.75)),
        ("invert", ("vals",), lambda d: ~(d > 0.0)),
        ("scalar add / rsub / rtruediv", ("vals",), lambda d: ((d + 1.5) - (2.0 - d)) / (1.0 / d)),
        ("frame arithmetic", ("vals", "other"), lambda d, o: (d * o + o) / (d - o)),
        ("int64 with a float scalar", ("mixed",), lambda d: d[["i"]] * 0.5 + 1),
        ("radd / rmul", ("vals",), lambda d: d.radd(2.0).rmul(3.0)),
        ("comparisons", ("vals", "other"), lambda d, o: (d < o) | (d >= 0.25) ^ (d == o) & (d != 0.0)),
        ("le / gt", ("vals", "other"), lambda d, o: (d <= o) & (d > -0.5)),
        ("count int64 / bool / float64", ("mixed",), lambda d: d.count()),
        ("sum", ("vals",), lambda d: d.sum()),
        ("sum int64", ("mixed",), lambda d: d[["i"]].sum()),
        ("prod", ("vals",), lambda d: d.prod()),
        ("max / min", ("vals",), lambda d: d.max() - d.min()),
        ("mean", ("vals",), lambda d: d.mean()),
        ("any / all", ("vals",), lambda d: (d > 1.0).any() & (d > -9.0).all()),
        ("idxmax", ("vals",), lambda d: d.idxmax()),
        ("idxmin", ("vals",), lambda d: d.idxmin()),
        ("var", ("vals",), lambda d: d.var()),
        ("std ddof=0", ("vals",), lambda d: d.std(ddof=0)),
        ("var(axis=1) refused", ("vals",), lambda d: d.var(axis=1)),
        ("cumsum / cummax / cummin", ("vals",), lambda d: _folds(d, lambda q: (q.cumsum(0), q.cummax(0), q.cummin(0))),
         lambda d: (d.cumsum(), d.cummax(), d.cummin())),
        ("forward fill", ("vals",), lambda d: d.fillna(method="ffill"), lambda d: d.ffill()),
        ("fillna scalar", ("vals",), lambda d: d.fillna(0.5)),
        ("fillna dict", ("vals",), lambda d: d.fillna({"a": 1.0, "c": -2.0})),
        ("fillna frame", ("vals", "other"), lambda d, o: d.fillna(o)),
        ("fillna limit refused", ("vals",), lambda d: d.fillna(0.5, limit=2)),
        ("astype one dtype", ("mixed",), lambda d: d.astype("float64")),
        ("astype mapping", ("mixed",), lambda d: d.astype({"t": "int64", "i": "float64"})),
        ("astype refused", ("vals",), lambda d: d.astype("int64")),
        ("merge left", ("keyed", "dim"), lambda d, m: d.merge(m, on="key", how="left")),
        ("merge inner", ("keyed", "dim"), lambda d, m: d.merge(m, on="key", how="inner")),
    ]
    for agg in aggs + ("size",):
        cases.append((f"groupby.{agg}", ("keyed",), lambda d, agg=agg: getattr(d.drop(columns="k2").groupby("key"), agg)()))
        cases.append((f"groupby(two keys).{agg}", ("keyed",), lambda d, agg=agg: getattr(d.groupby(["key", "k2"]), agg)()))
        cases.append((f"40 values groupby.{agg}", ("wide",), lambda d, agg=agg: getattr(d.drop(columns="k2").groupby("key"), agg)()))
        cases.append((f"40 values groupby(two keys).{agg}", ("wide",), lambda d, agg=agg: getattr(d.groupby(["key", "k2"]), agg)()))
    for agg in aggs:
        cases.append((f"groupby(as_index=False).{agg}", ("keyed",),
                      lambda d, agg=agg: getattr(d.drop(columns="k2").groupby("key", as_index=False), agg)()))
        cases.append((f"groupby(two keys, as_index=False).{agg}", ("keyed",),
                      lambda d, agg=agg: getattr(d.groupby(["key", "k2"], as_index=False), agg)()))
    spec = {"c": "mean", "a": "sum", "b": "max"}
    cases += [
        ("groupby.agg(dict)", ("keyed",), lambda d: d.drop(columns="k2").groupby("key").agg(spec)),
        ("groupby(two keys).agg(dict)", ("keyed",), lambda d: d.groupby(["key", "k2"]).agg(spec)),
        ("groupby(as_index=False).agg(dict)", ("keyed",), lambda d: d.groupby(["key", "k2"], as_index=False).agg(spec)),
        ("40 values groupby.agg(dict)", ("wide",), lambda d: d.groupby("key").agg({f"w{j}": ("sum", "max")[j % 2] for j in range(40)})),
        ("groupby.agg(dict) on a key refused", ("keyed",), lambda d: d.groupby(["key", "k2"]).agg({"key": "sum"})),
        ("groupby(two keys) over a float key refused", ("keyed",), lambda d: d.groupby(["key", "a"]).sum()),
    ]
    return cases


def _folds(df, calls):
    """The Fold registrations through the mirror's query compiler: its API layer has no cumulative methods."""
    return tuple(type(df)(query_compiler=qc) for qc in calls(df._query_compiler))


def _host(x):
    if isinstance(x, tuple):
        return pandas.concat([_host(y) for y in x], axis=1)
    return x._to_pandas() if hasattr(x, "_to_pandas") else x


def _outcome(call, args):
    try:
        return _host(call(*args)), None
    except Exception as e:  # the error type is part of the answer
        return None, type(e)


def _differences(got, want):
    """What differs between two host results, bit for bit: values, dtypes, row and column labels."""
    if type(got) is not type(want):
        return f"{type(got).__name__} vs {type(want).__name__}"
    if isinstance(got, pandas.DataFrame) and not got.columns.equals(want.columns):
        return f"columns {list(got.columns)} vs {list(want.columns)}"
    if not (got.index.equals(want.index) and got.index.names == want.index.names and got.index.dtype == want.index.dtype):
        return f"index {got.index[:4]} vs {want.index[:4]}"
    pairs = [(got.iloc[:, j], want.iloc[:, j]) for j in range(got.shape[1])] if got.ndim == 2 else [(got, want)]
    for a, b in pairs:
        a, b = a.to_numpy(), b.to_numpy()
        if a.dtype != b.dtype or a.tobytes() != b.tobytes():
            return f"values / dtype {a.dtype} vs {b.dtype}"
    if isinstance(got, pandas.Series) and got.name != want.name:
        return f"name {got.name!r} vs {want.name!r}"
    return None


@needs_modin
def test_every_shared_operation_agrees_across_the_front_doors(plugin, cpu_device):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present: host-logic sweep, runs on the double only")
    import modin_b200.pandas as bpd

    _, mpd = plugin
    frames = _frames()
    bad = {}
    for case in _cases():
        name, used, mirror_call = case[:3]
        plugin_call = case[3] if len(case) > 3 else mirror_call
        got, err = _outcome(mirror_call, [bpd.DataFrame(frames[f]) for f in used])
        want, want_err = _outcome(plugin_call, [mpd.DataFrame(frames[f]) for f in used])
        if err or want_err:
            if err is None or want_err is None or not (issubclass(err, want_err) or issubclass(want_err, err)):
                bad[name] = f"mirror raised {err}, plug-in raised {want_err}"
            continue
        diff = _differences(got, want)
        if diff:
            bad[name] = diff
    assert not bad, "\n".join(f"{k}: {v}" for k, v in bad.items())
