"""Arg-reduction probe: ``df.idxmax()`` against ``df.max()`` on the TreeReduce leg's shape (rows x 16 float64,
generated in HBM), through the front door and at the kernel.

    python tools/argreduce_probe.py [--rows 5e8] [--cols 16] [--reps 7] [--warmup 2]

Prints one JSON line per case with the median and range of ``--reps`` timings, taken after ``--warmup`` untimed runs
and alternating the two operations: the algorithmic bytes (8 B per element read; both read every element once) over
the median time, their share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s) and G rows/s, with the card's
name and power limit read in the same run.  Cases:
  frontdoor  ``df.max()`` / ``df.idxmax()`` of ``modin_b200.pandas`` (default ReduceVariant): host clock around the
             call, which returns a host Series (so it ends in a device synchronise)
  kernel_vK  ``ops.reduce_columns("max")`` / ``ops.arg_reduce_columns("max")`` under ReduceVariant K, CUDA events
The idxmax result is checked: the value at every returned row is the column's maximum.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from map_probe import PEAK_GBS, card  # noqa: E402

from modin_b200 import _lib, ops, synth  # noqa: E402


def alternate(fns, reps, warmup, timer):
    """Times of each fn, run in alternation ``reps`` times after ``warmup`` rounds."""
    for _ in range(warmup):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    out = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            out[k].append(timer(fn))
    return out


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=5e8)
    ap.add_argument("--cols", type=int, default=16)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    n, W = int(args.rows), args.cols
    lib = _lib.load()
    _lib.check(lib.mb200_device_check(0))
    torch.cuda.set_device(0)
    info = card()
    import modin_b200.pandas as bpd
    from modin_b200.dataframe import B200Dataframe

    blocks = synth.device_blocks(n, W, seed=42, npartitions=1)
    df = bpd.DataFrame(query_compiler=bpd.B200QueryCompiler(B200Dataframe.from_blocks(blocks)))
    cols = blocks[0].cols
    nbytes = n * W * 8

    def report(case, op, ms, checked=None):
        med = statistics.median(ms)
        gbs = nbytes / (med / 1e3) / 1e9
        row = {"case": case, "op": op, "rows": n, "cols": W, "bytes": nbytes, "ms": round(med, 3),
               "ms_min": round(min(ms), 3), "ms_max": round(max(ms), 3), "reps": len(ms),
               "Grows_s": round(n / (med / 1e3) / 1e9, 3), "GBs": round(gbs, 1), "frac_of_3350": round(gbs / PEAK_GBS, 3),
               **info}  # fmt: skip
        if checked is not None:
            row["checked"] = checked
        print(json.dumps(row), flush=True)

    res = {}
    t = alternate({"max": lambda: res.__setitem__("max", df.max()), "idxmax": lambda: res.__setitem__("idx", df.idxmax())},
                  args.reps, args.warmup, host_ms)  # fmt: skip
    at = torch.tensor(res["idx"].to_numpy(), dtype=torch.int64, device=cols[0].data.device)
    picked = torch.stack([cols[j].data[at[j]] for j in range(W)]).cpu().numpy()
    ok = bool((picked == res["max"].to_numpy()).all())
    report("frontdoor", "max", t["max"])
    report("frontdoor", "idxmax", t["idxmax"], ok)
    for variant in (0, 1):
        t = alternate({"max": lambda: ops.reduce_columns("max", cols, variant=variant),
                       "idxmax": lambda: ops.arg_reduce_columns("max", cols, variant)}, args.reps, args.warmup, event_ms)
        report(f"kernel_v{variant}", "max", t["max"])
        report(f"kernel_v{variant}", "idxmax", t["idxmax"])


if __name__ == "__main__":
    main()
