"""Cost of n frames of one pair at arbitrary times (film_interpolate_times) against n ordinary calls.

    python tools/times_rate.py [--n 1 2 4 7] [--rounds 3] [--calls 10] [--json PATH]

One process, one GPU, one engine, a 1088x1920 frame pair resident in HBM (torch tensors):
1. For each n: `interpolate_at_device` with the n evenly spaced times k / (n + 1), against n calls of
   `interpolate_device` (what the midpoint-only engine costs for n frames).  Both are timed with CUDA events around
   --calls repetitions, alternating in every round so that clock and co-tenant drift hit both alike; the median over
   the rounds is reported with the spread (min - max of the round values).
2. The head / tail split of one call with option time_ops = 1 (eager, one event pair per op): the head is every op
   before fusion_warp@L0 (padding, pyramids, features, flows), the tail the rest (fusion warps, side tensors, decoder).
3. arena_bytes of the ordinary plan and of the times plan.

Prints the card name and power limit with the numbers.  Needs a GPU: there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

H, W = 1088, 1920


def card_info() -> str:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip() or r.stderr.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        return f"nvidia-smi unavailable ({e})"


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--n", type=int, nargs="+", default=[1, 2, 4, 7])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--json", default=None, help="also write the result as JSON to this path")
    a = ap.parse_args(argv)

    import torch
    from frame_interpolation_b200 import synthetic
    from frame_interpolation_b200.interpolator import Interpolator

    if not torch.cuda.is_available():
        raise SystemExit("times_rate.py needs a GPU")
    card = card_info()
    print("card:", card, flush=True)
    x0, x1 = synthetic.frame_pair(H, W, seed=1)
    d0 = torch.from_numpy(x0[0]).cuda()
    d1 = torch.from_numpy(x1[0]).cuda()
    out = torch.empty((max(a.n), H, W, 3), dtype=torch.float32, device="cuda")
    eng = Interpolator("synthetic", align=64)
    stream = torch.cuda.Stream()
    sp = stream.cuda_stream

    def times_call(n):
        eng.interpolate_at_device(d0.data_ptr(), d1.data_ptr(), [k / (n + 1) for k in range(1, n + 1)], H, W,
                                  out.data_ptr(), stream=sp)

    def ordinary_calls(n):
        for i in range(n):
            eng.interpolate_device(d0.data_ptr(), d1.data_ptr(), 1, H, W, out[i].data_ptr(), stream=sp)

    def timed(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record(stream)
            for _ in range(a.calls):
                fn(n)
            e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / a.calls

    for n in a.n:   # warm-up: both plans built, graphs instantiated, modules loaded
        times_call(n)
        ordinary_calls(n)
    torch.cuda.synchronize()
    arena = {}
    eng.interpolate_device(d0.data_ptr(), d1.data_ptr(), 1, H, W, out.data_ptr())
    eng.synchronize()
    arena["ordinary"] = eng.profile()["arena_bytes"]
    times_call(1)
    torch.cuda.synchronize()
    arena["times"] = eng.profile()["arena_bytes"]

    samples = {n: {"times": [], "ordinary": []} for n in a.n}
    for r in range(a.rounds):
        for n in a.n:
            samples[n]["times"].append(timed(times_call, n))
            samples[n]["ordinary"].append(timed(ordinary_calls, n))
        print(f"round {r}: " + ", ".join(f"n={n} {samples[n]['times'][-1]:.2f}/{samples[n]['ordinary'][-1]:.2f} ms"
                                         for n in a.n), flush=True)

    # head / tail split: one eager call with one event pair per op
    eng.set_option("time_ops", 1)
    eng.interpolate_at_device(d0.data_ptr(), d1.data_ptr(), [0.5], H, W, out.data_ptr())
    eng.synchronize()
    table = eng.op_table()
    cut = [r["name"] for r in table].index("fusion_warp@L0")
    head_ms = sum(r["ms"] for r in table[:cut])
    tail_ms = sum(r["ms"] for r in table[cut:])
    eng.set_option("time_ops", 0)
    eng.close()

    rows = []
    print(f"\n{H}x{W}, frames in HBM, {a.rounds} rounds x {a.calls} calls; card: {card}")
    print(f"{'n':>3} {'times call ms':>22} {'n ordinary calls ms':>24} {'ms/frame times':>15} {'ms/frame ordinary':>18} "
          f"{'speed-up':>9}")
    for n in a.n:
        t, o = samples[n]["times"], samples[n]["ordinary"]
        mt, mo = statistics.median(t), statistics.median(o)
        rows.append(dict(n=n, times_ms=mt, times_spread=[min(t), max(t)], ordinary_ms=mo, ordinary_spread=[min(o), max(o)],
                         speedup=mo / mt))
        print(f"{n:>3} {mt:9.2f} ({min(t):.2f}-{max(t):.2f}) {mo:10.2f} ({min(o):.2f}-{max(o):.2f}) {mt / n:15.2f} "
              f"{mo / n:18.2f} {mo / mt:8.2f}x")
    share = tail_ms / (head_ms + tail_ms)
    print(f"\nhead / tail of one eager (time_ops) call: {head_ms:.2f} / {tail_ms:.2f} ms, tail share {share:.3f}; "
          f"n frames cost {1 - share:.2f} + {share:.2f} n calls by these times")
    print(f"arena_bytes: ordinary plan {arena['ordinary'] / 2**30:.2f} GiB, times plan {arena['times'] / 2**30:.2f} GiB "
          f"(+{(arena['times'] - arena['ordinary']) / 1e9:.2f} GB)")
    result = dict(card=card, size=[H, W], rounds=a.rounds, calls=a.calls, rows=rows, head_ms=head_ms, tail_ms=tail_ms,
                  arena_bytes=arena)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
