"""The odd-frame-shape sweeps as plain case tables, shared by the CPU device double (``test_host_shapes_cpu.py``) and
the kernels (``test_gpu_shape_cases.py``).

Every builder takes the front door ``bpd`` (``modin_b200.pandas``, with or without the double installed) and returns
``{name: (device thunk, pandas thunk)}``; a few also return calls that must be refused.  The thunks are only called by
the comparison, so a builder runs no device work besides ingest.

``rounded(name)`` says which cases carry a float sum, mean, var or std (or something computed from one, like a group
table): those are compared within a bound on the device, everything else bit for bit.  For that bound every table
carries ``rows`` (the most rows any of its sums adds up) and ``abs_sum`` (an upper bound of the sum of |x| over the
values such a sum sees: ``rows`` times the largest |x| of the summed columns).
"""

import re

import numpy as np
import pandas

from modin_b200 import synth

_ROUNDED = re.compile(r"\b(sum|mean|var|std)\b|^group table|: dict$|: two keys$|^groupby$")


def rounded(name):
    return bool(_ROUNDED.search(name))


class Cases(dict):
    def __init__(self, cases, rows, *host):
        super().__init__(cases)
        big = max(float(np.nanmax(np.abs(h.drop(columns=[c for c in ("key", "k2") if c in h.columns])
                                           .to_numpy(dtype=np.float64)), initial=0.0)) for h in host)  # fmt: skip
        self.rows, self.abs_sum = int(rows), rows * big


def frames():
    """(pa, pb, dim): two synthetic frames of 1003 and 517 rows and a 9-row dim table over their 11 keys."""
    pa = synth.host_frame(1003, 3, seed=1, nan_per_64k=3000, key_modulus=11)
    pb = synth.host_frame(517, 3, seed=2, nan_per_64k=3000, key_modulus=11)
    rng = np.random.RandomState(3)
    dim = pandas.DataFrame({"key": rng.permutation(11)[:9].astype(np.int64), "d0": rng.randn(9)})
    return pa, pb, dim


def concatenated(bpd, pa, pb, dim):
    a, b, dd = bpd.DataFrame(pa), bpd.DataFrame(pb), bpd.DataFrame(dim)
    cat, wcat = bpd.concat([a, b, a]), pandas.concat([pa, pb, pa])  # labels restart: 0..1002, 0..516, 0..1002
    cati, wcati = bpd.concat([a, b, a], ignore_index=True), pandas.concat([pa, pb, pa], ignore_index=True)
    f = ["c0", "c1", "c2"]
    return Cases({
        "filter": (lambda: cat[cat["c0"] > 0.0], lambda: wcat[wcat["c0"] > 0.0]),
        "dropna": (lambda: cat.dropna(), lambda: wcat.dropna()),
        "head": (lambda: cat.head(1200), lambda: wcat.head(1200)),
        "tail": (lambda: cat.tail(1200), lambda: wcat.tail(1200)),
        "sort": (lambda: cat.sort_values("c0"), lambda: wcat.sort_values("c0", kind="stable")),
        "sort ignore_index": (lambda: cat.sort_values("c0", ignore_index=True),
                              lambda: wcat.sort_values("c0", kind="stable", ignore_index=True)),
        "merge left": (lambda: cat.merge(dd, on="key", how="left"), lambda: wcat.merge(dim, on="key", how="left")),
        "merge inner": (lambda: cat.merge(dd, on="key", how="inner"), lambda: wcat.merge(dim, on="key", how="inner")),
        "groupby": (lambda: cat.groupby("key").mean(), lambda: wcat.groupby("key").mean()),
        "binary with itself": (lambda: cat[f] + cat[f], lambda: wcat[f] + wcat[f]),
        "a*b+c": (lambda: cati[f] * cati[f] + cati[f], lambda: wcati[f] * wcati[f] + wcati[f]),
        "assign": (lambda: cat.assign(d=cat["c0"] * 2.0), lambda: wcat.assign(d=wcat["c0"] * 2.0)),
        "drop_duplicates": (lambda: cat.drop_duplicates(subset=["key"]), lambda: wcat.drop_duplicates(subset=["key"])),
        "drop_duplicates ignore_index": (lambda: cat.drop_duplicates(subset=["key"], ignore_index=True),
                                         lambda: wcat.drop_duplicates(subset=["key"], ignore_index=True)),
        "drop_duplicates last": (lambda: cati.drop_duplicates(subset=["key"], keep="last"),
                                 lambda: wcati.drop_duplicates(subset=["key"], keep="last")),
        "astype": (lambda: cat.astype({"key": "float64"}), lambda: wcat.astype({"key": "float64"})),
        "concat of concats": (lambda: bpd.concat([cat, cati]), lambda: pandas.concat([wcat, wcati])),
        "var": (lambda: cat[f].var(), lambda: wcat[f].var()),
        "sum": (lambda: cat[f].sum(), lambda: wcat[f].sum()),
    }, len(wcat), pa, pb)  # fmt: skip


def empty_and_one_row(bpd, pa, pb, dim):
    a, b, dd = bpd.DataFrame(pa), bpd.DataFrame(pb), bpd.DataFrame(dim)
    emp, wemp = a[a["c0"] > 100.0], pa[pa["c0"] > 100.0]
    assert len(emp) == 0
    f = ["c0", "c1", "c2"]
    # an empty comparison is an empty BOOL frame, an empty true division is float64, int (op) float promotes
    assert list((emp[f] > 0.0).dtypes) == [np.dtype("bool")] * 3 and list((emp[f] >= emp[f]).dtypes) == [np.dtype("bool")] * 3
    assert list((emp[["key"]] / 2).dtypes) == [np.dtype("float64")] and list((emp[["key"]] * 2).dtypes) == [np.dtype("int64")]
    assert list((emp[["key"]] * 0.5).dtypes) == [np.dtype("float64")] and list((emp[["key"]] == 3).dtypes) == [np.dtype("bool")]
    return Cases({
        "to_pandas": (lambda: emp, lambda: wemp),
        "sum": (lambda: emp[f].sum(), lambda: wemp[f].sum()),
        "mean": (lambda: emp[f].mean(), lambda: wemp[f].mean()),
        "count": (lambda: emp[f].count(), lambda: wemp[f].count()),
        "min": (lambda: emp[f].min(), lambda: wemp[f].min()),
        "var": (lambda: emp[f].var(), lambda: wemp[f].var()),
        "abs": (lambda: emp[f].abs(), lambda: wemp[f].abs()),
        "affine": (lambda: emp[f] * 2.0 + 1.0, lambda: wemp[f] * 2.0 + 1.0),
        "any": (lambda: (emp[f] > 0.0).any(), lambda: (wemp[f] > 0.0).any()),
        "all": (lambda: (emp[f] > 0.0).all(), lambda: (wemp[f] > 0.0).all()),
        "filter again": (lambda: emp[emp["c1"] > 0.0], lambda: wemp[wemp["c1"] > 0.0]),
        "groupby": (lambda: emp.groupby("key").sum(), lambda: wemp.groupby("key").sum()),
        "merge": (lambda: emp.merge(dd, on="key", how="left"), lambda: wemp.merge(dim, on="key", how="left")),
        "sort": (lambda: emp.sort_values("c0"), lambda: wemp.sort_values("c0")),
        "head": (lambda: emp.head(5), lambda: wemp.head(5)),
        "drop_duplicates": (lambda: emp.drop_duplicates(subset=["key"]), lambda: wemp.drop_duplicates(subset=["key"])),
        "astype": (lambda: emp.astype({"key": "float64"}), lambda: wemp.astype({"key": "float64"})),
        "nunique": (lambda: emp[["key"]].nunique(), lambda: wemp[["key"]].nunique()),
        "concat with an empty frame": (lambda: bpd.concat([a, emp, b]), lambda: pandas.concat([pa, wemp, pb])),
        "concat of empties": (lambda: bpd.concat([emp, emp]), lambda: pandas.concat([wemp, wemp])),
        "head(0) sum": (lambda: a.head(0)[f].sum(), lambda: pa.head(0)[f].sum()),
        "one row drop_duplicates": (lambda: a.head(1).drop_duplicates(subset=["key"]), lambda: pa.head(1).drop_duplicates(subset=["key"])),
        "one row sort": (lambda: a.head(1).sort_values("c0"), lambda: pa.head(1).sort_values("c0")),
        "one row groupby": (lambda: a.head(1).groupby("key").sum(), lambda: pa.head(1).groupby("key").sum()),
    }, len(pa), pa)  # fmt: skip


def int64_bool_and_mixed(bpd):
    """int64 and bool VALUE columns (the synthetic frames are float64): the promotion / widening paths.  Returns
    ``(cases, refused)``; ``refused`` are calls that must raise NotImplementedError, never approximate."""
    rng = np.random.RandomState(11)
    n = 803
    pdf = pandas.DataFrame({
        "key": rng.randint(0, 9, n).astype(np.int64), "i": rng.randint(-1000, 1000, n).astype(np.int64),
        "j": rng.randint(1, 50, n).astype(np.int64), "x": rng.randn(n), "b": rng.rand(n) > 0.5, "c": rng.rand(n) > 0.2,
    })  # fmt: skip
    pdf.loc[::37, "x"] = np.nan
    df = bpd.DataFrame(pdf)
    ints, wints = df[["i", "j"]], pdf[["i", "j"]]
    bools, wbools = df[["b", "c"]], pdf[["b", "c"]]
    mixed, wmixed = df[["i", "x"]], pdf[["i", "x"]]
    as_i = {"columns": {"x": "i", "j": "i", "c": "b"}}  # a second operand under the first one's label
    cases = {
        "int abs": (lambda: ints.abs(), lambda: wints.abs()),
        "int neg": (lambda: -ints, lambda: -wints),
        "int + int scalar": (lambda: ints + 3, lambda: wints + 3),
        "int * float scalar": (lambda: ints * 2.5, lambda: wints * 2.5),
        "int / int scalar": (lambda: ints / 4, lambda: wints / 4),
        "int / int frame": (lambda: ints / ints, lambda: wints / wints),
        "int * int frame": (lambda: ints * ints, lambda: wints * wints),
        "int - float frame": (lambda: df[["i"]] - df[["x"]].rename(**as_i), lambda: pdf[["i"]] - pdf[["x"]].rename(**as_i)),
        "int == int scalar": (lambda: ints == 3, lambda: wints == 3),
        "int > int frame": (lambda: df[["i"]] > df[["j"]].rename(**as_i), lambda: pdf[["i"]] > pdf[["j"]].rename(**as_i)),
        "float > int scalar": (lambda: df[["x"]] > 0, lambda: pdf[["x"]] > 0),
        "int isna": (lambda: ints.isna(), lambda: wints.isna()),
        "int fillna": (lambda: ints.fillna(0), lambda: wints.fillna(0)),
        "int round": (lambda: ints.round(1), lambda: wints.round(1)),
        "int clip": (lambda: ints.clip(-10, 10), lambda: wints.clip(-10, 10)),
        "int isin": (lambda: ints.isin([1, 2, 3]), lambda: wints.isin([1, 2, 3])),
        "sort by int": (lambda: df.sort_values("i"), lambda: pdf.sort_values("i", kind="stable")),
        "sort by int, descending": (lambda: df.sort_values("i", ascending=False),
                                    lambda: pdf.sort_values("i", ascending=False, kind="stable")),
        "mixed frame": (lambda: mixed, lambda: wmixed),
        "mixed * int scalar": (lambda: mixed * 2, lambda: wmixed * 2),
        "mixed * float scalar": (lambda: mixed * 2.0, lambda: wmixed * 2.0),
        "mixed round": (lambda: mixed.round(1), lambda: wmixed.round(1)),
        "mixed abs": (lambda: mixed.abs(), lambda: wmixed.abs()),
        "mixed dropna": (lambda: mixed.dropna(), lambda: wmixed.dropna()),
        "mixed fillna": (lambda: mixed.fillna(0.5), lambda: wmixed.fillna(0.5)),
        "bool frame": (lambda: bools, lambda: wbools),
        "bool and": (lambda: df[["b"]] & df[["c"]].rename(**as_i), lambda: pdf[["b"]] & pdf[["c"]].rename(**as_i)),
        "bool not": (lambda: ~bools, lambda: ~wbools),
        "bool -> int64": (lambda: bools.astype("int64"), lambda: wbools.astype("int64")),
        "bool -> float64": (lambda: bools.astype("float64"), lambda: wbools.astype("float64")),
        "rows where a bool column holds": (lambda: df[["key", "i", "x"]][df["b"]], lambda: pdf[["key", "i", "x"]][pdf["b"]]),
        "rows where a float column is positive": (lambda: df[["key", "i", "j", "x"]][df["x"] > 0],
                                                  lambda: pdf[["key", "i", "j", "x"]][pdf["x"] > 0]),
        "groupby count of ints": (lambda: df[["key", "i"]].groupby("key").count(), lambda: pdf[["key", "i"]].groupby("key").count()),
        "groupby mean of ints": (lambda: df[["key", "i"]].groupby("key").mean(), lambda: pdf[["key", "i"]].groupby("key").mean()),
        "groupby mean, mixed": (lambda: df[["key", "i", "x"]].groupby("key").mean(), lambda: pdf[["key", "i", "x"]].groupby("key").mean()),
        "head of all dtypes": (lambda: df.head(9), lambda: pdf.head(9)),
    }  # fmt: skip
    for red in ("sum", "mean", "min", "max", "count", "var", "std"):
        cases[f"int {red}"] = ((lambda r=red: getattr(ints, r)()), (lambda r=red: getattr(wints, r)()))
    for red in ("sum", "mean", "min", "var"):
        cases[f"mixed {red}"] = ((lambda r=red: getattr(mixed, r)()), (lambda r=red: getattr(wmixed, r)()))
    for red in ("sum", "mean", "any", "all", "count", "var"):
        cases[f"bool {red}"] = ((lambda r=red: getattr(bools, r)()), (lambda r=red: getattr(wbools, r)()))
    cases["int prod"] = (lambda: ints.head(5).prod(), lambda: wints.head(5).prod())
    # an int64 column against a FLOAT scalar is compared in float64 like numpy / pandas do -- including the rounding
    # of the converted column above 2**53, where exact integer arithmetic would answer differently
    for opname in ("gt", "ge", "lt", "le", "eq", "ne"):
        for s in (0.5, -3.0, 7.0, float("nan"), float("inf")):
            cases[f"int {opname} {s}"] = ((lambda o=opname, v=s: getattr(ints, o)(v)), (lambda o=opname, v=s: getattr(wints, o)(v)))
    edge = pandas.DataFrame({"e": np.array([2**53 - 1, 2**53, 2**53 + 1, 2**53 + 2, -(2**53) - 1, 0], dtype=np.int64)})
    dedge = bpd.DataFrame(edge)
    for opname in ("gt", "ge", "lt", "le", "eq", "ne"):
        for s in (float(2**53), float(-(2**53)), 9007199254740993.0):
            cases[f"2**53 edge {opname} {s}"] = ((lambda o=opname, v=s: getattr(dedge, o)(v)), (lambda o=opname, v=s: getattr(edge, o)(v)))
    assert bool((edge["e"] > float(2**53)).iloc[2]) is False  # pandas: 2**53 + 1 rounds to 2**53; exact math says True
    cases["filter by int > float"] = (lambda: df[["key", "i"]][df["i"] > 0.5], lambda: pdf[["key", "i"]][pdf["i"] > 0.5])
    refused = [
        lambda: bools.min(),  # any / all / sum cover bool columns
        lambda: df[["key", "i"]].groupby("key").sum()._to_pandas(),  # group tables accumulate float64 values
        lambda: df[["key", "i"]].groupby("key").min()._to_pandas(),
    ]
    return Cases(cases, n, pdf.drop(columns=["b", "c"])), refused


def wide(bpd, pa, dim):
    """More than 32 columns: several column partitions, so every operation sees a 2-D grid of blocks.  Returns
    ``(cases, reductions)``; the reductions run on a frame that IS two column partitions (ingested with 40 columns;
    selecting 40 columns on the device can come back as one partition), so the second pass of var / std has to find
    ITS columns' means by label."""
    rng = np.random.RandomState(7)
    W = 40
    fcols = [f"w{i}" for i in range(W)]
    wide = pandas.DataFrame(rng.randn(300, W), columns=fcols)
    wide.iloc[::17, 3] = np.nan
    wide.iloc[::29, 35] = np.nan
    wide.insert(0, "key", rng.randint(0, 7, 300).astype(np.int64))
    dw, dd, a = bpd.DataFrame(wide), bpd.DataFrame(dim), bpd.DataFrame(pa)
    assert dw._query_compiler._modin_frame._partitions.shape[1] == 2
    cases = {
        "to_pandas": (lambda: dw, lambda: wide),
        "filter": (lambda: dw[dw["w0"] > 0.0], lambda: wide[wide["w0"] > 0.0]),
        "dropna": (lambda: dw.dropna(), lambda: wide.dropna()),
        "head": (lambda: dw.head(77), lambda: wide.head(77)),
        "tail": (lambda: dw.tail(77), lambda: wide.tail(77)),
        "sum": (lambda: dw[fcols].sum(), lambda: wide[fcols].sum()),
        "var": (lambda: dw[fcols].var(), lambda: wide[fcols].var()),
        "a*b+c": (lambda: dw[fcols] * dw[fcols] + dw[fcols], lambda: wide[fcols] * wide[fcols] + wide[fcols]),
        "comparison": (lambda: dw[fcols] < 0.0, lambda: wide[fcols] < 0.0),
        "round": (lambda: dw[fcols].round(1), lambda: wide[fcols].round(1)),
        "sort": (lambda: dw.sort_values("w5"), lambda: wide.sort_values("w5", kind="stable")),
        "groupby": (lambda: dw.groupby("key").sum(), lambda: wide.groupby("key").sum()),
        "merge": (lambda: dw.merge(dd, on="key", how="left"), lambda: wide.merge(dim, on="key", how="left")),
        "drop_duplicates": (lambda: dw.drop_duplicates(subset=["key"]), lambda: wide.drop_duplicates(subset=["key"])),
        "astype": (lambda: dw.astype({"key": "float64"}), lambda: wide.astype({"key": "float64"})),
        "concat rows": (lambda: bpd.concat([dw, dw]), lambda: pandas.concat([wide, wide])),
        "concat columns": (lambda: bpd.concat([dw, a.head(300)[["c0"]]], axis=1),
                           lambda: pandas.concat([wide, pa.head(300)[["c0"]]], axis=1)),
        "assign": (lambda: dw.assign(z=dw["w1"] * 2.0), lambda: wide.assign(z=wide["w1"] * 2.0)),
        "columns from both partitions": (lambda: dw[["w39", "w2"]], lambda: wide[["w39", "w2"]]),
    }  # fmt: skip
    vals = wide[fcols]
    dv = bpd.DataFrame(vals)
    assert dv._query_compiler._modin_frame._partitions.shape[1] == 2
    reductions = {}
    for name, kw in (("sum", {}), ("sum", {"skipna": False}), ("sum", {"min_count": 1}), ("mean", {}), ("mean", {"skipna": False}),
                     ("min", {}), ("max", {"skipna": False}), ("count", {}), ("var", {}), ("var", {"ddof": 0}),
                     ("var", {"skipna": False}), ("std", {}), ("std", {"ddof": 0})):  # fmt: skip
        reductions[f"{name} {kw}"] = ((lambda n=name, k=kw: getattr(dv, n)(**k)), (lambda n=name, k=kw: getattr(vals, n)(**k)))
    return Cases(cases, 2 * len(wide), wide), Cases(reductions, len(vals), vals)


def non_range_labels(bpd, pa, dim):
    """Group tables and filtered frames carry their labels as device index columns; inputs may come with a named
    integer index, a float index or (small frames) a string index.  Returns ``(cases, string-labelled frame)``."""
    a, dd = bpd.DataFrame(pa), bpd.DataFrame(dim)
    g, wg = a.groupby("key").sum(), pa.groupby("key").sum()
    fl, wfl = a[a["c0"] > 0.0], pa[pa["c0"] > 0.0]
    named = pa.set_axis(pandas.Index(np.arange(len(pa))[::-1] * 2, name="rid"), axis=0)
    fidx = pa.set_axis(pandas.Index(np.linspace(0.0, 1.0, len(pa))), axis=0)
    sidx = pa.head(40).set_axis(pandas.Index([f"r{i}" for i in range(40)]), axis=0)
    dn, df_, ds = bpd.DataFrame(named), bpd.DataFrame(fidx), bpd.DataFrame(sidx)
    cases = {
        "group table * 2": (lambda: g * 2.0, lambda: wg * 2.0),
        "group table head": (lambda: g.head(3), lambda: wg.head(3)),
        "group table filter": (lambda: g[g["c0"] > 0.0], lambda: wg[wg["c0"] > 0.0]),
        "group table sort": (lambda: g.sort_values("c1"), lambda: wg.sort_values("c1", kind="stable")),
        "group table sum": (lambda: g.sum(), lambda: wg.sum()),
        "group table + itself": (lambda: g + g, lambda: wg + wg),
        "group table assign": (lambda: g.assign(z=g["c0"] - g["c1"]), lambda: wg.assign(z=wg["c0"] - wg["c1"])),
        "filter twice": (lambda: fl[fl["c1"] > 0.0], lambda: wfl[wfl["c1"] > 0.0]),
        "filter -> sort": (lambda: fl.sort_values("c2"), lambda: wfl.sort_values("c2", kind="stable")),
        "filter -> merge": (lambda: fl.merge(dd, on="key", how="inner"), lambda: wfl.merge(dim, on="key", how="inner")),
        "filter -> square": (lambda: fl[["c0"]] * fl[["c0"]], lambda: wfl[["c0"]] * wfl[["c0"]]),
        "filter -> assign": (lambda: fl.assign(z=fl["c0"] + 1.0), lambda: wfl.assign(z=wfl["c0"] + 1.0)),
        "filter -> tail": (lambda: fl.tail(13), lambda: wfl.tail(13)),
        "filter -> drop_duplicates": (lambda: fl.drop_duplicates(subset=["key"], keep="last"),
                                      lambda: wfl.drop_duplicates(subset=["key"], keep="last")),
        "concat of filtered": (lambda: bpd.concat([fl, fl]), lambda: pandas.concat([wfl, wfl])),
        "concat of plain and filtered": (lambda: bpd.concat([a, fl]), lambda: pandas.concat([pa, wfl])),
        "named int index": (lambda: dn, lambda: named),
        "named int index filter": (lambda: dn[dn["c0"] > 0.0], lambda: named[named["c0"] > 0.0]),
        "named int index sort": (lambda: dn.sort_values("c0"), lambda: named.sort_values("c0", kind="stable")),
        "named int index head": (lambda: dn.head(5), lambda: named.head(5)),
        "named int index * 2": (lambda: dn * 2, lambda: named * 2),
        "float index filter": (lambda: df_[df_["c0"] > 0.0], lambda: fidx[fidx["c0"] > 0.0]),
        "float index tail": (lambda: df_.tail(5), lambda: fidx.tail(5)),
        "string index": (lambda: ds, lambda: sidx),
        "string index * 2": (lambda: ds[["c0"]] * 2.0, lambda: sidx[["c0"]] * 2.0),
        "string index head": (lambda: ds.head(5), lambda: sidx.head(5)),
        "string index sum": (lambda: ds[["c0", "c1"]].sum(), lambda: sidx[["c0", "c1"]].sum()),
        "string index sort, ignore_index": (lambda: ds.sort_values("c0", ignore_index=True),
                                            lambda: sidx.sort_values("c0", kind="stable", ignore_index=True)),
    }  # fmt: skip
    return Cases(cases, len(pa), pa), ds


def binary_operand_shapes(bpd):
    """The Binary template's operand shapes -- scalars on either side, positional and labelled row vectors, a column
    Series along axis 0, co-partitioned frames, fused x*s+t chains -- on plain, wide (two column partitions), filtered
    and int64 frames.  Returns ``(cases, the wide device frame, its row vector)``."""
    rng = np.random.RandomState(5)
    pa = synth.host_frame(1003, 3, seed=1, nan_per_64k=3000, key_modulus=11)
    f = ["c0", "c1", "c2"]
    v, dv = pa[f], bpd.DataFrame(pa)[f]
    other = synth.host_frame(1003, 3, seed=2, nan_per_64k=2000, key_modulus=11)[f]
    do = bpd.DataFrame(other)
    W = 40
    fc = [f"w{i}" for i in range(W)]
    wide = pandas.DataFrame(rng.randn(200, W), columns=fc); wide.iloc[::13, 33] = np.nan
    dw = bpd.DataFrame(wide)
    ints = pandas.DataFrame({"i": rng.randint(-50, 50, 300).astype(np.int64), "j": rng.randint(1, 9, 300).astype(np.int64)})
    di = bpd.DataFrame(ints)
    fl, dfl = v[v["c0"] > 0.0], dv[dv["c0"] > 0.0]
    row3 = [0.5, -1.0, 2.0]; srow = pandas.Series(row3, index=f)
    roww = list(np.linspace(-1, 1, W)); sroww = pandas.Series(roww, index=fc)
    cases = {
        "2 - df": (lambda: 2.0 - dv, lambda: 2.0 - v), "1 / df": (lambda: 1.0 / dv, lambda: 1.0 / v),
        "2 + df": (lambda: 2.0 + dv, lambda: 2.0 + v), "3 * df": (lambda: 3 * dv, lambda: 3 * v),
        "df - 2": (lambda: dv - 2, lambda: v - 2), "df / 4": (lambda: dv / 4, lambda: v / 4),
        "df.rsub(1)": (lambda: dv.rsub(1.0), lambda: v.rsub(1.0)), "df.rtruediv(2)": (lambda: dv.rtruediv(2.0), lambda: v.rtruediv(2.0)),
        "df + list": (lambda: dv + row3, lambda: v + row3), "df * Series": (lambda: dv * bpd.Series(srow), lambda: v * srow),
        "df * pandas Series": (lambda: dv * srow, lambda: v * srow),
        "df - list": (lambda: dv - row3, lambda: v - row3), "df / list": (lambda: dv / row3, lambda: v / row3),
        "df < list": (lambda: dv < row3, lambda: v < row3),
        "df.mul(col, 0)": (lambda: dv.mul(dv["c1"], axis=0), lambda: v.mul(v["c1"], axis=0)),
        "df.sub(col, 0)": (lambda: dv.sub(dv["c1"], axis=0), lambda: v.sub(v["c1"], axis=0)),
        "df.rsub(col, 0)": (lambda: dv.rsub(dv["c1"], axis=0), lambda: v.rsub(v["c1"], axis=0)),
        "df.truediv(col, 0)": (lambda: dv.truediv(dv["c1"], axis=0), lambda: v.truediv(v["c1"], axis=0)),
        "df.add(col, 0)": (lambda: dv.add(dv["c1"], axis=0), lambda: v.add(v["c1"], axis=0)),
        "df.lt(col, 0)": (lambda: dv.lt(dv["c1"], axis=0), lambda: v.lt(v["c1"], axis=0)),
        "df - other": (lambda: dv - do, lambda: v - other), "df / other": (lambda: dv / do, lambda: v / other),
        "other.rsub(df)": (lambda: do.rsub(dv), lambda: other.rsub(v)), "df.rtruediv(other)": (lambda: dv.rtruediv(do), lambda: v.rtruediv(other)),
        "df >= other": (lambda: dv >= do, lambda: v >= other), "df != other": (lambda: dv != do, lambda: v != other),
        "a*b+c frames": (lambda: dv * do + do, lambda: v * other + other),
        "a*s+t": (lambda: dv * 1.5 + 0.25, lambda: v * 1.5 + 0.25), "a*s-t": (lambda: dv * 1.5 - 0.25, lambda: v * 1.5 - 0.25),
        "(a+s)*t": (lambda: (dv + 1.0) * 2.0, lambda: (v + 1.0) * 2.0), "a*s*t": (lambda: dv * 2.0 * 3.0, lambda: v * 2.0 * 3.0),
        "a*list+list": (lambda: dv * row3 + row3, lambda: v * row3 + row3),
        "-(a*2)": (lambda: -(dv * 2.0), lambda: -(v * 2.0)), "abs(a-1)": (lambda: (dv - 1.0).abs(), lambda: (v - 1.0).abs()),
        "fillna dict": (lambda: dv.fillna({"c0": 1.0, "c2": -1.0}), lambda: v.fillna({"c0": 1.0, "c2": -1.0})),
        "fillna frame": (lambda: dv.fillna(do), lambda: v.fillna(other)),
        "fillna then mul": (lambda: dv.fillna(0.0) * 2.0, lambda: v.fillna(0.0) * 2.0),
        "clip lower": (lambda: dv.clip(lower=0.0), lambda: v.clip(lower=0.0)), "clip upper": (lambda: dv.clip(upper=0.0), lambda: v.clip(upper=0.0)),
        "round then sum": (lambda: dv.round(1).sum(), lambda: v.round(1).sum()),
        "wide + list": (lambda: dw + roww, lambda: wide + roww), "wide * Series": (lambda: dw * sroww, lambda: wide * sroww),
        "wide.mul(col,0)": (lambda: dw.mul(dw["w3"], axis=0), lambda: wide.mul(wide["w3"], axis=0)),
        "wide a*s+t": (lambda: dw * 1.5 + 0.25, lambda: wide * 1.5 + 0.25), "2 - wide": (lambda: 2.0 - dw, lambda: 2.0 - wide),
        "wide - wide": (lambda: dw - dw, lambda: wide - wide), "wide fillna": (lambda: dw.fillna(0.5), lambda: wide.fillna(0.5)),
        "filtered * 2": (lambda: dfl * 2.0, lambda: fl * 2.0), "filtered + list": (lambda: dfl + row3, lambda: fl + row3),
        "filtered.mul(col,0)": (lambda: dfl.mul(dfl["c1"], axis=0), lambda: fl.mul(fl["c1"], axis=0)),
        "filtered - filtered": (lambda: dfl - dfl, lambda: fl - fl), "2 - filtered": (lambda: 2.0 - dfl, lambda: 2.0 - fl),
        "int - 2": (lambda: di - 2, lambda: ints - 2), "2 - int": (lambda: 2 - di, lambda: 2 - ints), "2.5 - int": (lambda: 2.5 - di, lambda: 2.5 - ints),
        "1 / int": (lambda: 1 / di, lambda: 1 / ints), "int + list": (lambda: di + [1, 2], lambda: ints + [1, 2]),
        "int * flist": (lambda: di * [0.5, 2.0], lambda: ints * [0.5, 2.0]), "int.mul(col,0)": (lambda: di.mul(di["j"], axis=0), lambda: ints.mul(ints["j"], axis=0)),
        "int / int col": (lambda: di.truediv(di["j"], axis=0), lambda: ints.truediv(ints["j"], axis=0)),
        "int*2+1": (lambda: di * 2 + 1, lambda: ints * 2 + 1), "int*2.0+1": (lambda: di * 2.0 + 1, lambda: ints * 2.0 + 1),
    }  # fmt: skip
    return Cases(cases, len(pa), pa, wide), dw, roww


def groupby_kinds(bpd):
    """Every aggregation x (40 value columns, narrow, keys with gaps, one group, keys over the whole int64 range) x
    (plain, filtered, concatenated input); plus dictionary and multi-key aggregation."""
    rng = np.random.RandomState(5)
    n = 907
    wide = pandas.DataFrame(rng.randn(n, 40), columns=[f"w{i}" for i in range(40)])
    wide.iloc[::13, 33] = np.nan
    wide.iloc[::7, 2] = np.nan
    wide.insert(0, "key", rng.randint(-4, 5, n).astype(np.int64))
    wide.insert(1, "k2", (rng.randint(0, 3, n) * 100 - 100).astype(np.int64))
    narrow = wide[["key", "k2", "w0", "w2", "w33"]]
    frames = {
        "wide": wide, "narrow": narrow, "keys with gaps": narrow.assign(key=narrow["key"] * 1000003),
        "one group": narrow.assign(key=np.int64(7)),
        "keys over the int64 range": narrow.assign(key=rng.randint(-(2**62), 2**62, n).astype(np.int64)),
    }  # fmt: skip
    spec = {"w2": "max", "w0": "sum", "w33": "count"}
    cases = {}
    for fname, p in frames.items():
        d = bpd.DataFrame(p)
        cols = ["key"] + [c for c in p.columns if c not in ("key", "k2")]
        variants = {
            "plain": (d, p),
            "filtered": (d[d["w0"] > 0.0], p[p["w0"] > 0.0]),
            "concatenated": (bpd.concat([d, d.head(100)], ignore_index=True), pandas.concat([p, p.head(100)], ignore_index=True)),
        }  # fmt: skip
        for vname, (dd, pp) in variants.items():
            for agg in ("sum", "count", "mean", "min", "max", "size"):
                cases[f"{fname} / {vname}: {agg}"] = ((lambda x=dd, a=agg: getattr(x[cols].groupby("key"), a)()),
                                                      (lambda x=pp, a=agg: getattr(x[cols].groupby("key"), a)()))  # fmt: skip
            if fname in ("wide", "narrow"):
                mk = ["key", "k2", "w0", "w2", "w33"]
                cases[f"{fname} / {vname}: dict"] = ((lambda x=dd: x.groupby("key").agg(spec)), (lambda x=pp: x.groupby("key").agg(spec)))
                cases[f"{fname} / {vname}: two keys"] = ((lambda x=dd: x[mk].groupby(["key", "k2"]).sum()),
                                                         (lambda x=pp: x[mk].groupby(["key", "k2"]).sum()))  # fmt: skip
    assert len(cases) == 5 * 3 * 6 + 2 * 3 * 2
    return Cases(cases, n + 100, wide)


def merge_kinds(bpd):
    """fact.merge(dim, on="key", how=left | inner): dim tables holding every key / some keys / one row / no key of the
    fact / no rows at all, with a float payload that overlaps a fact column (suffixes) and an int64 payload (promoted
    to float64 when a left join misses); facts plain, wider than one column partition, with gappy keys and keys near
    the int64 range; inputs plain, filtered, concatenated."""
    rng = np.random.RandomState(5)
    n = 907
    fact = pandas.DataFrame({"key": rng.randint(-4, 12, n).astype(np.int64), "x": rng.randn(n), "d0": rng.randn(n),
                             "i": rng.randint(0, 9, n).astype(np.int64)})  # fmt: skip
    fact.loc[::11, "x"] = np.nan
    wide = pandas.concat([fact, pandas.DataFrame(rng.randn(n, 36), columns=[f"w{i}" for i in range(36)])], axis=1)

    def dim_of(keys):
        k = np.asarray(keys, dtype=np.int64)
        return pandas.DataFrame({"key": k, "d0": rng.randn(len(k)), "p": np.arange(len(k), dtype=np.int64) * 3})

    dims = {"every key": dim_of(rng.permutation(np.arange(-4, 12))), "some keys": dim_of(rng.permutation(np.arange(-4, 12))[:9]),
            "one row": dim_of([3]), "no key of the fact": dim_of([100, 200]), "no rows": dim_of([])}  # fmt: skip
    scale = {"plain": 1, "wide": 1, "keys with gaps": 1000003, "keys near the int64 range": 2**58}
    facts = {"plain": fact, "wide": wide, "keys with gaps": fact.assign(key=fact["key"] * 1000003),
             "keys near the int64 range": fact.assign(key=fact["key"] * (2**58))}  # fmt: skip
    cases = {}
    for fname, p in facts.items():
        d = bpd.DataFrame(p)
        variants = {"plain": (d, p), "filtered": (d[d["x"] > 0.0], p[p["x"] > 0.0]),
                    "concatenated": (bpd.concat([d, d.head(50)], ignore_index=True), pandas.concat([p, p.head(50)], ignore_index=True))}  # fmt: skip
        for vname, (dd, pp) in variants.items():
            for dname, dim in dims.items():
                dim = dim.assign(key=dim["key"] * scale[fname])
                for how, suffixes in (("left", ("_x", "_y")), ("inner", ("_x", "_y")), ("left", ("_l", "_r"))):
                    cases[f"{fname} / {vname} x {dname}, {how} {suffixes}"] = (
                        lambda x=dd, y=dim, h=how, s=suffixes: x.merge(bpd.DataFrame(y), on="key", how=h, suffixes=s),
                        lambda x=pp, y=dim, h=how, s=suffixes: x.merge(y, on="key", how=h, suffixes=s))
    return Cases(cases, 1, fact)
