"""Cost and effect of overlapped tiles with a feathered stitch (option tile_overlap) against the reference's tiling.

    python tools/tile_overlap_rate.py [--overlaps 32 64] [--rounds 3] [--steps 4] [--stitch_launches 200] [--json PATH]

One process, one GPU, one engine.  Three measurements:

1. ms per 4K (2160x3840) frame in 2x2 tiles at tile_overlap = 0 and each of --overlaps, with the padded window size of
   each.  An overlap is timed against 0 in alternating rounds, so that clock and co-tenant drift hit both alike.  Two
   paths: the device-resident one (`parallel.interpolate_tiled_device` on one rank, frames in HBM, CUDA events), and the
   host call (`Interpolator.__call__`, pageable host frames in, pinned frame out, host clock around the blocking call).
2. The stitch kernel alone at 4K 2x2: CUDA events around --stitch_launches launches, and the bytes the stitch needs
   (every output float written once, every source float it blends read once) over that time.
3. A 1088x1920 frame, which still fits untiled: mean and max absolute distance between the 2x2-tiled result and the
   untiled one inside the +-16-pixel band around the two seams, and the mean absolute step across the seam column and
   row against the same step 8 pixels away.  With synthetic random weights this says little about real footage.

Prints the card name and power limit with the numbers.  Needs a GPU: there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card_info() -> str:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip() or r.stderr.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        return f"nvidia-smi unavailable ({e})"


def stitch_bytes(h: int, w: int, block, v: int) -> int:
    """Bytes the stitch needs: one write per output float, one read per (output float, window it blends).  Per axis the
    2v pixels around each of the b - 1 interior boundaries blend two windows, every other pixel reads one."""
    reads = (h + 2 * v * (block[0] - 1)) * (w + 2 * v * (block[1] - 1))
    return (reads + h * w) * 3 * 4


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--overlaps", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--stitch_launches", type=int, default=200)
    ap.add_argument("--json", default=None, help="also write the result as JSON to this path")
    a = ap.parse_args(argv)

    import torch
    from frame_interpolation_b200 import parallel, spec, synthetic
    from frame_interpolation_b200.interpolator import Interpolator

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement needs an H100")
    block = [2, 2]
    dt = np.full((1,), 0.5, np.float32)
    eng = Interpolator("synthetic", align=64, block_shape=block)
    eng_dev = parallel.device_engine(eng)
    res = {"card": card_info(), "block_shape": block, "steps_per_round": a.steps}

    # ---- 1. step time at 4K ------------------------------------------------------------------------------------------
    h, w = 2160, 3840
    x0, x1 = synthetic.frame_pair(h, w, seed=0, n_waves=8)
    d0, d1 = torch.from_numpy(x0).cuda(), torch.from_numpy(x1).cuda()
    d_out = torch.empty_like(d0)

    def run_device(v, n):
        for _ in range(n):
            parallel.interpolate_tiled_device(eng_dev, d0, d1, block, out=d_out, overlap=v)

    def run_host(v, n):
        eng.set_option("tile_overlap", v)
        for _ in range(n):
            eng(x0, x1, dt)

    step = {}
    for v in a.overlaps:
        eng.clear_cache()                          # two window shapes at a time: every cached 1080p-class plan holds ~20 GB
        ms = {(p, u): [] for p in ("device", "host") for u in (0, v)}
        for u in (0, v):
            run_device(u, 1)
            run_host(u, 1)
        torch.cuda.synchronize()
        for r in range(a.rounds):
            for u in ((0, v) if r % 2 == 0 else (v, 0)):
                run_device(u, 1)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run_device(u, a.steps)
                e1.record()
                torch.cuda.synchronize()
                ms[("device", u)].append(e0.elapsed_time(e1) / a.steps)
                run_host(u, 1)
                t0 = time.perf_counter()
                run_host(u, a.steps)               # every call blocks until its frame is in host memory
                ms[("host", u)].append((time.perf_counter() - t0) * 1e3 / a.steps)
        qh, qw = spec.tile_windows(h, w, block, v)[1]
        ph, pw, _, _ = spec.padded_shape(qh, qw, 64)
        p0h, p0w, _, _ = spec.padded_shape(h // 2, w // 2, 64)
        med = {k: statistics.median(t) for k, t in ms.items()}
        step[str(v)] = {
            "window": f"{qh}x{qw}", "padded_window": f"{ph}x{pw}", "padded_window_overlap_0": f"{p0h}x{p0w}",
            "network_pixels_ratio": round(ph * pw / (p0h * p0w), 4),
            "ms_per_frame": {f"{p}_overlap_{u}": [round(t, 3) for t in ts] for (p, u), ts in ms.items()},
            "median_ms": {f"{p}_overlap_{u}": round(t, 3) for (p, u), t in med.items()},
            "ratio_device": round(med[("device", v)] / med[("device", 0)], 4),
            "ratio_host": round(med[("host", v)] / med[("host", 0)], 4),
        }
    res["frame_4k"] = {"frame": f"{h}x{w}", "by_overlap": step}

    # ---- 2. the stitch kernel alone ----------------------------------------------------------------------------------
    stream = torch.cuda.Stream()                   # a real stream: the engine reads NULL as "my own stream"
    stitch = {}
    for v in a.overlaps:
        qh, qw = spec.tile_windows(h, w, block, v)[1]
        tiles = torch.rand((4, qh, qw, 3), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()

        def launch(n):
            for _ in range(n):
                eng.stitch_tiles_device(tiles.data_ptr(), qh * qw * 3, h, w, block, v, d_out.data_ptr(),
                                        stream=stream.cuda_stream)
        launch(10)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        launch(a.stitch_launches)
        e1.record(stream)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.stitch_launches
        nbytes = stitch_bytes(h, w, block, v)
        stitch[str(v)] = {"kernel": "k_stitch_feather", "launches": a.stitch_launches, "ms": round(ms, 4),
                          "algorithmic_MB": round(nbytes / 1e6, 1), "GB_per_s": round(nbytes / ms / 1e6, 1)}
        del tiles
    res["stitch_kernel_4k"] = stitch
    del d0, d1, d_out

    # ---- 3. seams at 1088x1920 ---------------------------------------------------------------------------------------
    eng.clear_cache()
    h, w = 1088, 1920
    x0, x1 = synthetic.frame_pair(h, w, seed=1, n_waves=8)
    untiled = eng.interpolate(x0, x1, dt)[0].astype(np.float64)
    sy, sx = h // 2, w // 2
    band = np.zeros((h, w), bool)
    band[sy - 16:sy + 16, :] = True
    band[:, sx - 16:sx + 16] = True

    def col_step(f, x):
        return float(np.abs(f[:, x] - f[:, x - 1]).mean())

    def row_step(f, y):
        return float(np.abs(f[y] - f[y - 1]).mean())

    seams = {}
    for v in [0] + list(a.overlaps):
        eng.set_option("tile_overlap", v)
        tiled = eng(x0, x1, dt)[0].astype(np.float64)
        d = np.abs(tiled - untiled)[band]
        seams[str(v)] = {
            "band_mean_abs_vs_untiled": float(d.mean()), "band_max_abs_vs_untiled": float(d.max()),
            "step_across_seam_column": col_step(tiled, sx), "step_8_px_away_column": col_step(tiled, sx + 8),
            "step_across_seam_row": row_step(tiled, sy), "step_8_px_away_row": row_step(tiled, sy + 8),
        }
    seams["untiled"] = {"step_across_seam_column": col_step(untiled, sx), "step_8_px_away_column": col_step(untiled, sx + 8),
                        "step_across_seam_row": row_step(untiled, sy), "step_8_px_away_row": row_step(untiled, sy + 8)}
    res["seams_1088x1920"] = seams
    eng.close()

    print(json.dumps(res, indent=1))
    print(f"\ncard: {res['card']}")
    print("| tile_overlap | padded window | device-resident ms / 4K frame (against 0, same rounds) | host call ms / 4K frame "
          "(against 0) | stitch kernel ms (GB/s) |")
    print("|---|---|---|---|---|")
    for v in a.overlaps:
        s, k = step[str(v)], stitch[str(v)]
        m = s["median_ms"]
        print(f"| {v} | {s['padded_window']} | {m[f'device_overlap_{v}']:.1f} ({m['device_overlap_0']:.1f}) | "
              f"{m[f'host_overlap_{v}']:.1f} ({m['host_overlap_0']:.1f}) | {k['ms']:.3f} ({k['GB_per_s']:.0f}) |")
    print("\n| 1088x1920, 2x2 | band mean abs vs untiled | band max abs | step across seam column (8 px away) | "
          "step across seam row (8 px away) |")
    print("|---|---|---|---|---|")
    for v in [0] + list(a.overlaps):
        s = seams[str(v)]
        print(f"| tile_overlap {v} | {s['band_mean_abs_vs_untiled']:.2e} | {s['band_max_abs_vs_untiled']:.2e} | "
              f"{s['step_across_seam_column']:.2e} ({s['step_8_px_away_column']:.2e}) | "
              f"{s['step_across_seam_row']:.2e} ({s['step_8_px_away_row']:.2e}) |")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
