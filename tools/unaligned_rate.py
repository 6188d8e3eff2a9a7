"""Step time of an unpadded frame (align=None, option any_size = 1) against the same frame padded to 64 (align=64).

    python tools/unaligned_rate.py [--h 1080 --w 1920] [--rounds 5] [--steps 20] [--warmup 3] [--json PATH]

At 1080x1920 the unpadded call runs the network at 1080x1920 instead of 1088x1920, and its decoder resizes level 3
(67x120 -> 135x240) with a gather of its own.  Both engines live in one process on one GPU; the rounds alternate
between them so that clock and co-tenant drift hit both alike.  Each round times `steps` back-to-back calls of the
device-pointer entry (frames resident in HBM) with CUDA events.  Prints the card name and power limit with the
numbers, and the per-round step times.  Needs a GPU: there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


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
    ap.add_argument("--h", type=int, default=1080)
    ap.add_argument("--w", type=int, default=1920)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the result as JSON to this path")
    a = ap.parse_args(argv)

    import torch
    from frame_interpolation_b200 import synthetic
    from frame_interpolation_b200.interpolator import Interpolator

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs an H100")
    h, w = a.h, a.w
    engines = {"align=None": Interpolator("synthetic", align=None), "align=64": Interpolator("synthetic", align=64)}
    engines["align=None"].set_option("any_size", 1)
    x0, x1 = synthetic.frame_pair(h, w, seed=0, n_waves=8)
    d0, d1 = torch.from_numpy(x0).cuda(), torch.from_numpy(x1).cuda()
    outs = {k: torch.empty_like(d0) for k in engines}
    # a real (non-NULL) stream: the engine treats NULL as "use my own stream", and torch.cuda.Event only sees work
    # enqueued on the stream it is recorded on
    stream = torch.cuda.Stream()

    def run(name, n):
        eng = engines[name]
        for _ in range(n):
            eng.interpolate_device(d0.data_ptr(), d1.data_ptr(), 1, h, w, outs[name].data_ptr(), stream=stream.cuda_stream)

    for name in engines:                       # plan build, graph capture, first launches
        run(name, a.warmup)
    torch.cuda.synchronize()
    ms = {k: [] for k in engines}
    for r in range(a.rounds):
        order = list(engines) if r % 2 == 0 else list(reversed(engines))
        for name in order:
            run(name, 1)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            run(name, a.steps)
            e1.record(stream)
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1) / a.steps)
    resized = [r["name"] for r in engines["align=None"].op_table() if r["name"].startswith("fusion_resize@")]
    padded = engines["align=64"].profile()
    res = {
        "card": card_info(),
        "frame": f"{h}x{w}",
        "padded_align64": f"{padded['padded_h']}x{padded['padded_w']}",
        "resize_ops_align_none": resized,
        "steps_per_round": a.steps,
        "ms_per_step": {k: [round(v, 4) for v in vs] for k, vs in ms.items()},
        "median_ms": {k: round(statistics.median(vs), 4) for k, vs in ms.items()},
        "frames_per_s": {k: round(1000.0 / statistics.median(vs), 3) for k, vs in ms.items()},
    }
    res["ratio_none_over_64"] = round(res["median_ms"]["align=None"] / res["median_ms"]["align=64"], 4)
    for eng in engines.values():
        eng.close()
    print(json.dumps(res, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
