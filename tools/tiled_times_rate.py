"""Cost of n frames of one 4K pair at arbitrary times in 2x2 tiles (parallel.interpolate_at_tiled_device) against n tiled
calls (parallel.interpolate_tiled_device).

    python tools/tiled_times_rate.py [--n 1 2 4 7] [--overlaps 0 32] [--rounds 3] [--calls 3] [--json PATH]

One process, one GPU, one engine, a 2160x3840 frame pair resident in HBM (torch tensors).  For each overlap and each n:
the n evenly spaced times k / (n + 1) through `interpolate_at_tiled_device` (per window one head and n tails, then one
stitch per time), against n calls of `interpolate_tiled_device` at the same overlap (what the midpoint-only engine costs
for n frames).  Both are timed with CUDA events around --calls repetitions, alternating in every round so that clock and
co-tenant drift hit both alike; the median over the rounds is reported with the spread (min - max of the round values).
Also reported: the padded window and the arena of the ordinary and of the times plan at that window.

Prints the card name and power limit with the numbers.  Needs a GPU: there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

H, W = 2160, 3840
BLOCK = [2, 2]


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
    ap.add_argument("--overlaps", type=int, nargs="+", default=[0, 32])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the result as JSON to this path")
    a = ap.parse_args(argv)

    import torch
    from frame_interpolation_b200 import parallel, spec, synthetic
    from frame_interpolation_b200.interpolator import Interpolator

    if not torch.cuda.is_available():
        raise SystemExit("tiled_times_rate.py needs a GPU")
    card = card_info()
    print("card:", card, flush=True)
    x0, x1 = synthetic.frame_pair(H, W, seed=1, n_waves=8)
    d0, d1 = torch.from_numpy(x0).cuda(), torch.from_numpy(x1).cuda()
    out = torch.empty((max(a.n), H, W, 3), dtype=torch.float32, device="cuda")
    eng = Interpolator("synthetic", align=64)     # untiled handle: the tiles are the parallel functions'
    dev = parallel.device_engine(eng)
    stream = torch.cuda.Stream()

    res = dict(card=card, frame=[H, W], block_shape=BLOCK, rounds=a.rounds, calls=a.calls, by_overlap={})
    for v in a.overlaps:
        eng.clear_cache()                          # one window shape at a time: two plans of a 1080p-class window
        qh, qw = spec.tile_windows(H, W, BLOCK, v)[1]
        ph, pw, _, _ = spec.padded_shape(qh, qw, 64)
        bufs = {n: torch.empty((1, 4, n, qh, qw, 3), dtype=torch.float32, device="cuda") for n in a.n}
        tiled_buf = torch.empty((1, 4, qh, qw, 3), dtype=torch.float32, device="cuda")

        def times_call(n):
            parallel.interpolate_at_tiled_device(dev, d0, d1, [k / (n + 1) for k in range(1, n + 1)], BLOCK,
                                                 out=out[:n], gather_buf=bufs[n], overlap=v)

        def tiled_calls(n):
            for i in range(n):
                parallel.interpolate_tiled_device(dev, d0, d1, BLOCK, out=out[i:i + 1], gather_buf=tiled_buf, overlap=v)

        def timed(fn, n):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(stream):
                e0.record(stream)
                for _ in range(a.calls):
                    fn(n)
                e1.record(stream)
            e1.synchronize()
            return e0.elapsed_time(e1) / a.calls

        arena = {}
        with torch.cuda.stream(stream):
            tiled_calls(1)
            torch.cuda.synchronize()
            arena["ordinary"] = eng.profile()["arena_bytes"]
            times_call(1)
            torch.cuda.synchronize()
            arena["times"] = eng.profile()["arena_bytes"]
            for n in a.n:   # warm-up: both plans built, graphs instantiated, modules loaded
                times_call(n)
                tiled_calls(n)
        torch.cuda.synchronize()

        samples = {n: {"times": [], "tiled": []} for n in a.n}
        for r in range(a.rounds):
            for n in a.n:
                order = ("times", "tiled") if r % 2 == 0 else ("tiled", "times")
                for k in order:
                    samples[n][k].append(timed(times_call if k == "times" else tiled_calls, n))
            print(f"overlap {v} round {r}: " + ", ".join(
                f"n={n} {samples[n]['times'][-1]:.1f}/{samples[n]['tiled'][-1]:.1f} ms" for n in a.n), flush=True)
        rows = []
        for n in a.n:
            t, o = samples[n]["times"], samples[n]["tiled"]
            mt, mo = statistics.median(t), statistics.median(o)
            rows.append(dict(n=n, times_ms=mt, times_spread=[min(t), max(t)], tiled_ms=mo, tiled_spread=[min(o), max(o)],
                             speedup=mo / mt))
        res["by_overlap"][str(v)] = dict(window=[qh, qw], padded_window=[ph, pw], arena_bytes=arena, rows=rows)
        del bufs, tiled_buf
    eng.close()

    print(f"\n{H}x{W} in {BLOCK[0]}x{BLOCK[1]} tiles, frames in HBM, {a.rounds} rounds x {a.calls} calls; card: {card}")
    for v, r in res["by_overlap"].items():
        ph, pw = r["padded_window"]
        ar = r["arena_bytes"]
        print(f"\ntile_overlap {v}: window {r['window'][0]}x{r['window'][1]} padded to {ph}x{pw}; arena: ordinary plan "
              f"{ar['ordinary'] / 2**30:.2f} GiB, times plan {ar['times'] / 2**30:.2f} GiB")
        print(f"{'n':>3} {'tiled times call ms':>26} {'n tiled calls ms':>26} {'ms/frame times':>15} "
              f"{'ms/frame tiled':>15} {'speed-up':>9}")
        for row in r["rows"]:
            n, mt, mo = row["n"], row["times_ms"], row["tiled_ms"]
            (t0, t1), (o0, o1) = row["times_spread"], row["tiled_spread"]
            print(f"{n:>3} {mt:10.1f} ({t0:.1f}-{t1:.1f}) {mo:12.1f} ({o0:.1f}-{o1:.1f}) {mt / n:15.1f} {mo / n:15.1f} "
                  f"{mo / mt:8.2f}x")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
