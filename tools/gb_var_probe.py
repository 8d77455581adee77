"""``groupby('key').var()`` / ``.std()`` against ``.mean()`` on the benchmark's groupby shape, on one GPU.

    python tools/gb_var_probe.py [--rows 5e8] [--groups 1000000] [--steps 10] [--warmup 2] [--out DIR]

The frame is ``bench.py``'s groupby frame (``synth.device_frame``: int64 keys uniform or Zipf-like over ``--groups``
values, 8 float64 values), driven through the Modin-free mirror.  Cases: dense table, hash table forced
(``GroupbyDenseKeys`` off), skewed keys, 1000 keys (a dense range small enough for the per-CTA shared-memory tables),
and a frame whose 8 value columns are int64 (cast to float64 first, as ``mean`` does).  ``var``, ``std`` and ``mean``
run alternately, one step each per round, and each step is timed with CUDA events around the launched work; then
``ops.KernelTimer`` times the two passes of a few more steps apart: pass 1 (``gb_accumulate``, the same SUM | COUNT
kernels ``mean`` runs) and pass 2 (``gb_accumulate_m2``, the centred pass).  Each pass's rate is given against the data
sheet's 3.35 TB/s of HBM3 (H100 SXM) from the algorithmic bytes of one sweep: 8 B per key plus 8 B per value per row.
Sampled groups are checked against pandas on the rows a boolean row selection returns, outside the timed region.  The
card's name and power limit are printed with the numbers; one JSON line per case goes to stdout (and to
DIR/gb_var_probe.jsonl with ``--out``)."""


from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import pandas

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet (700 W card)
W = 8


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)  # fmt: skip
        return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    except Exception as exc:  # the numbers still need a name next to them
        return f"nvidia-smi unavailable ({type(exc).__name__})"


def _int_frame(rows, groups):
    """The groupby frame with 8 int64 value columns (uniform in [0, 2^31))."""
    from modin_b200 import ops, synth
    from modin_b200.block import DeviceBlock
    from modin_b200.dataframe import B200Dataframe
    from modin_b200.pandas import DataFrame
    from modin_b200.query_compiler import B200QueryCompiler

    key = synth.device_blocks(rows, 0, key_modulus=groups)[0].cols[0]
    cols = [key] + [ops.gen_i64(rows, 42, j + 1, 1 << 31) for j in range(W)]
    blk = DeviceBlock(cols, pandas.Index(["key"] + [f"c{j}" for j in range(W)]), nrows=rows, range_start=0)
    return DataFrame(query_compiler=B200QueryCompiler(B200Dataframe.from_blocks([blk])))


def _check(df, res, fn, keys_to_check):
    """Sampled groups of ``res`` (a var / std result) against pandas on the group's rows."""
    keys = res.index.to_numpy()
    ok = bool(len(keys) and (np.diff(keys) > 0).all())
    for k in keys_to_check(keys):
        rows = df[df["key"] == int(k)]._to_pandas()
        want = getattr(rows.groupby("key"), fn)().iloc[0].to_numpy()
        got = res.loc[k].to_numpy()
        ok = ok and np.array_equal(np.isnan(got), np.isnan(want)) and np.allclose(got, want, rtol=1e-10, equal_nan=True)
    return ok


def run_case(label, df, fns, steps, warmup, dense, float_vals):
    import torch

    from modin_b200 import config, ops

    config.GroupbyDenseKeys.put(dense)
    try:
        gb = df.groupby("key")
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
        kern = {}
        for fn in fns:
            with ops.KernelTimer() as kt:
                for _ in range(3):
                    getattr(gb, fn)()._query_compiler.execute()
                kern[fn] = (kt.mean_ms("gb_accumulate"), kt.mean_ms("gb_accumulate_m2"))
        rows = len(df)
        checks = {}
        for fn in fns:
            if fn in ("var", "std") and float_vals:  # row selection takes the float frame
                res = getattr(gb, fn)()._to_pandas()
                checks[fn] = _check(df, res, fn, lambda k: [k[0], k[len(k) // 2], k[-1]])
        out = []
        nbytes = rows * (8 + 8 * W)  # one sweep
        share = lambda ms: (nbytes / (ms / 1e3)) / HBM_BYTES_PER_S if ms else None  # noqa: E731
        for fn in fns:
            ms = float(np.median(per[fn]))
            p1, p2 = kern[fn]
            out.append({"case": label, "agg": fn, "rows": rows, "ms_per_step_median": ms, "rows_per_s": rows / (ms / 1e3),
                        "pass1_gb_accumulate_ms": p1, "pass2_gb_accumulate_m2_ms": p2, "algorithmic_bytes_per_pass": nbytes,
                        "pass1_share_of_hbm_datasheet": share(p1), "pass2_share_of_hbm_datasheet": share(p2),
                        "checked": checks.get(fn)})  # fmt: skip
        return out
    finally:
        config.GroupbyDenseKeys.put(True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=5e8)
    ap.add_argument("--groups", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("gb_var_probe needs a CUDA device: nothing here is measured on the CPU")
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
                with open(os.path.join(args.out, "gb_var_probe.jsonl"), "a") as fh:
                    fh.write(line + "\n")

    cases = (("dense", False, True, G), ("hash table forced", False, False, G), ("skewed keys", True, True, G),
             ("1000 keys (shared-memory tables)", False, True, 1000))  # fmt: skip
    for label, skew, dense, groups in cases:
        df = synth.device_frame(rows, W, npartitions=1, seed=42, key_modulus=groups, key_skew=skew)
        df._query_compiler.execute()
        report(run_case(label, df, ("var", "std", "mean"), args.steps, args.warmup, dense, True))
        del df
        torch.cuda.empty_cache()
    report(run_case("8 int64 values", _int_frame(rows, G), ("var", "std", "mean"), args.steps, args.warmup, True, False))


if __name__ == "__main__":
    main()
