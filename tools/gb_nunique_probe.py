"""``groupby('key').nunique()`` against ``.size()`` on the benchmark's groupby shape, on one GPU.

    python tools/gb_nunique_probe.py [--rows 1e8] [--groups 1000000] [--steps 5] [--warmup 1] [--out DIR]

The frame is ``bench.py``'s groupby frame (``synth.device_frame``: int64 keys uniform or Zipf-like over ``--groups``
values, 8 float64 values that are all distinct in practice), driven through the Modin-free mirror.  Cases: dense table,
hash table forced (``GroupbyDenseKeys`` off), skewed keys, 8 low-cardinality int64 columns (16 values each), and 8
all-distinct float64 columns over 1000 keys (a dense range small enough for the shared-memory pass-1 kernel).
``nunique`` and ``size`` run alternately, one step each per round, each step timed with CUDA events around the launched
work; then ``ops.KernelTimer`` times the two passes of one more step apart: pass 1 (``gb_accumulate``, the SIZE launch
``size`` runs, once per column batch) and pass 2 (``gb_accumulate_distinct``, the distinct-set inserts).  The set's
bytes per batch are ``functors.distinct_batches``' plan.  Sampled groups are checked against pandas on the rows a
boolean row selection returns, outside the timed region.  The card's name, power limit and maximum SM clock are printed
with the numbers; one JSON line per case goes to stdout (and to DIR/gb_nunique_probe.jsonl with ``--out``)."""

from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import pandas

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.gb_var_probe import _card  # noqa: E402

W = 8


def _int_frame(rows, groups, modulus):
    """The groupby frame with 8 int64 value columns of ``modulus`` values each."""
    from modin_b200 import ops, synth
    from modin_b200.block import DeviceBlock
    from modin_b200.dataframe import B200Dataframe
    from modin_b200.pandas import DataFrame
    from modin_b200.query_compiler import B200QueryCompiler

    key = synth.device_blocks(rows, 0, key_modulus=groups)[0].cols[0]
    cols = [key] + [ops.gen_i64(rows, 42, j + 1, modulus) for j in range(W)]
    blk = DeviceBlock(cols, pandas.Index(["key"] + [f"c{j}" for j in range(W)]), nrows=rows, range_start=0)
    return DataFrame(query_compiler=B200QueryCompiler(B200Dataframe.from_blocks([blk])))


def _check(df, res):
    """Three sampled groups of ``res`` against pandas' nunique on the group's rows; keys must ascend."""
    keys = res.index.to_numpy()
    ok = bool(len(keys) and (np.diff(keys) > 0).all())
    for k in (keys[0], keys[len(keys) // 2], keys[-1]):
        rows = df[df["key"] == int(k)]._to_pandas()
        ok = ok and np.array_equal(res.loc[k].to_numpy(), rows.groupby("key").nunique().iloc[0].to_numpy())
    return ok


def run_case(label, df, steps, warmup, dense):
    import torch

    from modin_b200 import config, functors, ops

    config.GroupbyDenseKeys.put(dense)
    try:
        gb = df.groupby("key")
        fns = ("nunique", "size")
        for _ in range(warmup):
            for fn in fns:
                getattr(gb, fn)()._query_compiler.execute()
        torch.cuda.synchronize()
        per = {fn: [] for fn in fns}
        events = []
        for _ in range(steps):  # alternate the aggregations, one step each per round
            for fn in fns:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                getattr(gb, fn)()._query_compiler.finalize()
                b.record()
                events.append((fn, a, b))
        torch.cuda.synchronize()
        for fn, a, b in events:
            per[fn].append(a.elapsed_time(b))
        with ops.KernelTimer() as kt:
            gb.nunique()._query_compiler.execute()
            p1, p2 = kt.mean_ms("gb_accumulate"), kt.mean_ms("gb_accumulate_distinct")
        checked = _check(df, gb.nunique()._to_pandas())
        rows = len(df)
        batches = functors.distinct_batches(rows, W)
        set_bytes = [16 * functors._next_pow2(2 * rows * (hi - lo)) for lo, hi in batches]
        out = []
        for fn in fns:
            ms = float(np.median(per[fn]))
            r = {"case": label, "agg": fn, "rows": rows, "ms_per_step_median": ms, "rows_per_s": rows / (ms / 1e3)}
            if fn == "nunique":
                r.update({"column_batches": len(batches), "pass1_gb_accumulate_ms_per_batch": p1,
                          "pass2_gb_accumulate_distinct_ms_per_batch": p2, "set_bytes_per_batch": set_bytes,
                          "checked": checked})  # fmt: skip
            out.append(r)
        return out
    finally:
        config.GroupbyDenseKeys.put(True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1e8)
    ap.add_argument("--groups", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("gb_nunique_probe needs a CUDA device: nothing here is measured on the CPU")
    torch.cuda.set_device(0)
    from modin_b200 import synth

    rows, G = int(args.rows), args.groups
    card = _card()
    print(f"# card (name, power limit, max SM clock): {card}", flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)

    def report(results):
        for r in results:
            r["card"] = card
            line = json.dumps(r)
            print(line, flush=True)
            if args.out:
                with open(os.path.join(args.out, "gb_nunique_probe.jsonl"), "a") as fh:
                    fh.write(line + "\n")

    cases = (("dense", False, True, G), ("hash table forced", False, False, G), ("skewed keys", True, True, G),
             ("8 all-distinct float64, 1000 keys", False, True, 1000))  # fmt: skip
    for label, skew, dense, groups in cases:
        df = synth.device_frame(rows, W, npartitions=1, seed=42, key_modulus=groups, key_skew=skew)
        df._query_compiler.execute()
        report(run_case(label, df, args.steps, args.warmup, dense))
        del df
        torch.cuda.empty_cache()
    report(run_case("8 int64 columns of 16 values", _int_frame(rows, G, 16), args.steps, args.warmup, True))


if __name__ == "__main__":
    main()
