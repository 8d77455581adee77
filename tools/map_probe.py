"""Map-kernel probe: ``mb200_map`` at the bench shape against a device-to-device copy of the same bytes.

    python tools/map_probe.py [--rows 5e8] [--cols 8] [--reps 15] [--warmup 3]

Prints one JSON line per case: the median of ``--reps`` launches timed with CUDA events after ``--warmup``
untimed ones, the algorithmic bytes over that time, and their share of the H100 SXM data-sheet HBM3 bandwidth
(3.35 TB/s), with the card's name and power limit.  Cases:
  affine   ``df * b + c`` (AFFINE, f64), rows x cols: 8 B read + 8 B written per element -- the bench headline
  copy     torch ``copy_`` over the same bytes as ``affine``: the 1:1 read:write rate the map kernel can aim at
  gt_s     ``df > s`` (f64 in, uint8 predicate out): 8 B read + 1 B written
  and      ``p & q`` on bool columns (uint8 in, uint8 out)
  fma3     ``a * b + c`` on three frames (FMA3, f64) of rows / 4, as the bench's three-frame leg
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from modin_b200 import _lib  # noqa: E402

PEAK_GBS = 3350.0  # H100 SXM data sheet, HBM3; not a measured figure


def card():
    """Name and power limit of GPU 0, read in the same run as the measurement."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()  # fmt: skip
        name, limit, sm_max = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit_w": float(limit), "sm_max_mhz": float(sm_max)}
    except Exception as exc:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None, "error": f"nvidia-smi: {exc}"[:200]}


def time_launches(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(2 * reps)]
    for i in range(reps):
        evs[2 * i].record()
        fn()
        evs[2 * i + 1].record()
    torch.cuda.synchronize()
    return [evs[2 * i].elapsed_time(evs[2 * i + 1]) for i in range(reps)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=5e8)
    ap.add_argument("--cols", type=int, default=8)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    n, W = int(args.rows), args.cols
    lib = _lib.load()
    _lib.check(lib.mb200_device_check(0))
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream().cuda_stream
    info = card()

    def report(case, rows, nbytes, ms):
        med = statistics.median(ms)
        gbs = nbytes / (med / 1e3) / 1e9
        print(json.dumps({"case": case, "rows": rows, "cols": W, "bytes": nbytes, "ms": round(med, 3),
                          "ms_min": round(min(ms), 3), "ms_max": round(max(ms), 3), "reps": len(ms), "GBs": round(gbs, 1),
                          "frac_of_3350": round(gbs / PEAK_GBS, 3), **info}), flush=True)  # fmt: skip

    def cols(t):
        return _lib.ptr_array([t[j].data_ptr() for j in range(W)])

    def run_map(op, dtype, ins, out, rows, s0=None, s1=None):
        ptrs = [cols(t) if t is not None else None for t in ins] + [None] * (3 - len(ins))
        a0 = _lib.u64_array(s0) if s0 else None
        a1 = _lib.u64_array(s1) if s1 else None
        oc = cols(out)

        def fn():
            _lib.check(lib.mb200_map(_lib.OP[op], dtype, W, ptrs[0], ptrs[1], ptrs[2], oc, rows, a0, a1, st))

        return fn

    def bits(x):
        return [int(torch.tensor([x], dtype=torch.float64).view(torch.int64).item()) & (2**64 - 1)] * W

    # one column per row of a (W, n) tensor: every column starts 4 KiB-aligned when n is a multiple of 512
    a = torch.empty((W, n), dtype=torch.float64, device=dev).uniform_(-1.0, 1.0)
    out = torch.empty_like(a)
    fn = run_map("affine", _lib.F64, [a], out, n, bits(1.000000119), bits(0.5))
    report("affine", n, n * W * 16, time_launches(fn, args.reps, args.warmup))
    report("copy", n, n * W * 16, time_launches(lambda: out.copy_(a), args.reps, args.warmup))
    del out
    pred = torch.empty((W, n), dtype=torch.uint8, device=dev)
    fn = run_map("gt_s", _lib.F64, [a], pred, n, bits(0.0))
    report("gt_s", n, n * W * 9, time_launches(fn, args.reps, args.warmup))
    del a
    torch.cuda.empty_cache()
    q = torch.empty_like(pred).random_(0, 2)
    p2 = torch.empty_like(pred).random_(0, 2)
    fn = run_map("and", _lib.U8, [p2, q], pred, n)
    report("and", n, n * W * 3, time_launches(fn, args.reps, args.warmup))
    del pred, q, p2
    torch.cuda.empty_cache()
    n3 = n // 4
    fa, fb, fc = (torch.empty((W, n3), dtype=torch.float64, device=dev).uniform_(-1.0, 1.0) for _ in range(3))
    fo = torch.empty_like(fa)
    fn = run_map("fma3", _lib.F64, [fa, fb, fc], fo, n3)
    report("fma3", n3, n3 * W * 32, time_launches(fn, args.reps, args.warmup))


if __name__ == "__main__":
    main()
