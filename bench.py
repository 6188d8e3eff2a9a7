#!/usr/bin/env python
"""Benchmark of the FILM hot path: interpolated frames/sec (BASELINE.json metric).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl b200|reference] [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port P bench.py --gpus N --steps K --warmup W

A "step" is one network call on one synthetic 1080p frame pair (BASELINE.json configs[1]:
1920x1080, single mid-frame, batch 1, padded to 1088x1920 by align=64), Style-architecture
synthetic weights (no pre-trained SavedModel exists offline). With N > 1 every rank runs its
own frame pairs (frame pairs shard embarrassingly; no data-path collective) -> weak scaling.

`value`   : frames/s with the frame pair already resident in HBM (film_interpolate_device).
`e2e`     : frames/s through the reference-facing API `Interpolator.__call__(x0, x1, dt)` with
            pinned HOST numpy buffers; H2D of both frames and D2H of the result are inside
            the timed region.
`roofline`: conv implicit-GEMM kernels (wgmma), reference-graph FLOPs / summed kernel time
            measured with one CUDA-event pair per launch in a separate eager pass, against
            the bf16 peak of MEASURED_PEAKS.json or, without it, the H100 SXM data-sheet figure.
`--dump-outputs DIR`: after the timed steps, the interpolated frame of the last timed step (what a caller of
            film_interpolate_device receives) is written as DIR/interpolated_frame.npy (float32, 1x1080x1920x3 at
            the default size); a frame over 64 MB is written as a fixed seeded sample of its pixels instead
            (interpolated_frame_sample.npy + _pixels.npy). The inputs are seeded, so two builds can be compared
            output for output.
`workloads`: the other BASELINE.json configs, in the same JSON line: 4K tiled 2x2 (configs[2]),
            8K tiled 4x4 with the tiles sharded over the ranks and ONE NCCL all-gather inside the
            timed region (configs[4]), 720p recursive x6 = 63 mid-frames scheduled level-synchronously
            over the ranks (configs[3]); the sharded results are checked bit for bit against the
            same workload computed on one GPU.
`--impl reference`: the reference's algorithm on the host cores (CPU oracle port, torch-CPU;
            the TF2 reference itself cannot run here -- no TensorFlow in the image). Every step is
            ONE REAL 1080p call of the oracle; the number of steps is capped by a wall budget and
            the line reports the steps actually timed.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

H1080, W1080 = 1080, 1920
METRIC = "interpolated_frames_per_sec_1080p"
WORKLOAD_1080P = "1080p (1920x1080) single mid-frame, Style architecture, batch 1, align 64 -> 1088x1920"


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        return {"hbm_gbs": d["hbm_gbs"], "bf16_tflops": d["bf16_tflops"],
                "bf16_tflops_sustained": d.get("bf16_tflops_sustained", d["bf16_tflops"]),
                "source": "measured (MEASURED_PEAKS.json)"}
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0,
            "source": "H100 SXM data sheet (dense bf16, HBM3), not measured"}


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region: one streaming
    `nvidia-smi -lms 50` process (the recipe's clocks line), read by a thread."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.idx = gpu_index
        self.rows = []
        self._proc = None
        self._t = None

    def _run(self):
        try:
            for line in self._proc.stdout:
                self.rows.append([c.strip() for c in line.split(",")])
        except Exception:
            pass

    def __enter__(self):
        try:
            self._proc = subprocess.Popen(
                ["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-i", str(self.idx),
                 "-lms", "50"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self._t = threading.Thread(target=self._run, daemon=True)
            self._t.start()
            # nvidia-smi can take seconds to start on a fresh box: do not open the timed region before the first
            # sample has arrived, or a 0.3 s region ends with no clock record at all
            t_end = time.time() + 8.0
            while not self.rows and time.time() < t_end:
                time.sleep(0.02)
        except Exception:
            self._proc = None
        return self

    def __exit__(self, *a):
        if self._proc is not None:
            try:
                self._proc.terminate()          # the exact process we started
                self._proc.wait(timeout=5)
            except Exception:
                pass
        if self._t is not None:
            self._t.join(timeout=5)

    def summary(self):
        sm, mx, pw, reasons = [], [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            try:
                sm.append(float(r[1]))
                mx.append(float(r[2]))
                pw.append(float(r[3]))
                for n, v in zip(names, r[4:8]):
                    if v.lower().startswith("active"):
                        reasons.add(n)
            except Exception:
                continue
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        return {"sm_mhz": float(np.median(sm)), "sm_max_mhz": float(max(mx)), "reasons": sorted(reasons),
                "samples": len(sm), "power_w_max": float(max(pw)) if pw else None}


_BEST_THREADS = None
REF_WALL_BUDGET_S = 200.0      # the reference arm must end "within a few minutes"


def _pick_threads():
    """All the host threads that actually help at 1080p: torch-CPU convs stop scaling well before 128
    threads, so time one representative layer (64 -> 64, 3x3, 544x960) per candidate and keep the best."""
    global _BEST_THREADS
    if _BEST_THREADS is not None:
        return _BEST_THREADS
    import torch
    import torch.nn.functional as F
    ncpu = os.cpu_count() or 1
    try:
        ncpu = min(ncpu, len(os.sched_getaffinity(0)))
    except Exception:
        pass
    cands = sorted({c for c in (8, 16, 32, 64, ncpu) if c <= ncpu})
    x = torch.randn(2, 64, 544, 960)
    k = torch.randn(64, 64, 3, 3)
    best, best_t = cands[0], None
    for c in cands:
        torch.set_num_threads(c)
        F.conv2d(x, k, padding=1)
        t = time.perf_counter()
        for _ in range(2):
            F.conv2d(x, k, padding=1)
        el = time.perf_counter() - t
        if best_t is None or el < best_t:
            best, best_t = c, el
    _BEST_THREADS = best
    return best


class CpuOracle1080p:
    """The CPU oracle (torch-CPU port of the reference graph) on one REAL 1080p frame pair: the sample of
    both the `cpu_baseline` leg and the `--impl reference` arm, so the two report the same quantity."""

    def __init__(self):
        import torch
        from frame_interpolation_b200 import synthetic, weights
        from oracle.film_oracle import OracleInterpolator
        self.threads = _pick_threads()
        torch.set_num_threads(self.threads)
        w = weights.load(weights.ensure_synthetic_file())
        self.x0, self.x1 = synthetic.frame_pair(H1080, W1080, seed=0, n_waves=8)
        self.dt = np.full((1,), 0.5, np.float32)
        self.orc = OracleInterpolator(w, align=64)
        self.sample = (f"one call of the CPU oracle on a full {W1080}x{H1080} frame pair (padded 1088x1920), "
                       f"{self.threads} torch threads")

    def step(self) -> float:
        t = time.perf_counter()
        self.orc.interpolate(self.x0, self.x1, self.dt)
        return time.perf_counter() - t


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return 0
    t_start = time.perf_counter()
    orc = CpuOracle1080p()
    # one real call takes tens of seconds: warm-up and steps are cut to what the wall budget allows and the
    # line reports the counts actually run
    warm = 0
    secs = []
    first = orc.step()                         # doubles as the warm-up when the budget allows a second call
    if args.warmup > 0 and (time.perf_counter() - t_start) + 1.2 * first < REF_WALL_BUDGET_S:
        warm = 1
    else:
        secs.append(first)
    while len(secs) < max(args.steps, 1):
        if secs and (time.perf_counter() - t_start) + 1.1 * float(np.mean(secs)) > REF_WALL_BUDGET_S:
            break
        secs.append(orc.step())
    sec = float(np.mean(secs))
    v = 1.0 / sec
    line = {"impl": "reference", "metric": METRIC, "value": v, "unit": "frames/s", "n_gpus": args.gpus,
            "steps": len(secs), "warmup": warm, "ms_per_step": 1000.0 * sec, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": WORKLOAD_1080P,
                       "note": "CPU oracle port (torch-CPU) of the reference graph, NOT the TF2 reference (TensorFlow is "
                               "not installable offline); every step is one real 1080p call, steps/warmup are the counts "
                               f"that fit a {REF_WALL_BUDGET_S:.0f} s wall budget (requested {args.steps}/{args.warmup})"},
            "cpu_baseline": {"value": v, "unit": "frames/s", "cores": orc.threads, "kind": "port", "sample": orc.sample},
            "e2e": {"value": v, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)
    return 0


def extra_workloads(eng, world, rank, dev, dist):
    """BASELINE.json configs[2..4] through the device-resident sharded paths of frame_interpolation_b200.parallel.
    Timed with CUDA events on the current stream, barrier + synchronize on both sides, max over ranks; the
    all-gather of the sharded workloads is INSIDE the timed region. Every sharded result is compared bit for bit
    with the same workload computed by this rank alone (`group` of one) outside the timed region."""
    import torch
    from frame_interpolation_b200 import parallel, synthetic
    edev = parallel.device_engine(eng)
    solo = _SoloGroup()

    def timed(fn, reps, warm=1):
        for _ in range(warm):
            fn()
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            r = fn()
        e1.record()
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        t = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
        if dist is not None:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item()) / reps, r

    out = {}
    # ---- 4K tiled 2x2 (configs[2]; eval/interpolator.py:192-206): one 4K frame pair per GPU
    x0, x1 = synthetic.frame_pair(2160, 3840, seed=100 + rank, n_waves=8)
    d0, d1 = torch.from_numpy(x0).to(dev), torch.from_numpy(x1).to(dev)
    o4 = torch.empty_like(d0)
    gb = torch.empty((1, 4, 1080, 1920, 3), dtype=torch.float32, device=dev)
    with _solo(parallel, solo):
        ms, _ = timed(lambda: parallel.interpolate_tiled_device(edev, d0, d1, [2, 2], out=o4, gather_buf=gb), 3)
    out["4k_tiled_2x2"] = {"value": world * 1000.0 / ms, "unit": "frames/s", "ms_per_frame": ms,
                           "config": "3840x2160, block 2x2 (4 tiles of 1080x1920, each padded to 1088x1920), one frame "
                                     "pair per GPU, frames resident in HBM", "n_gpus": world}
    if world == 1:
        from frame_interpolation_b200.interpolator import Interpolator
        tiled = Interpolator("synthetic", align=64, block_shape=[2, 2], device=dev.index or 0)
        hx0, hx1 = torch.from_numpy(x0).pin_memory().numpy(), torch.from_numpy(x1).pin_memory().numpy()
        dt = np.full((1,), 0.5, np.float32)
        for _ in range(2):
            res = tiled(hx0, hx1, dt)
        secs = []
        for _ in range(5):                       # median of per-call wall times: one slow host-side call (page-locked
            t0 = time.perf_counter()             # allocation, a busy host) must not decide the number
            res = tiled(hx0, hx1, dt)
            secs.append(time.perf_counter() - t0)
        sec = float(np.median(secs))
        out["4k_tiled_2x2"]["e2e"] = {"value": 1.0 / sec, "unit": "frames/s", "api": "Interpolator(block_shape=[2, 2]).__call__",
                                      "h2d_bytes_per_step": 2 * int(x0.nbytes), "d2h_bytes_per_step": int(x0.nbytes),
                                      "bitwise_equal_to_device_path": bool(np.array_equal(res, o4.cpu().numpy()))}
        tiled.close()
    del d0, d1, o4, gb
    # ---- 8K tiled 4x4, tiles sharded over the ranks, ONE all-gather (configs[4])
    x0, x1 = synthetic.frame_pair(4320, 7680, seed=7, n_waves=8)
    d0, d1 = torch.from_numpy(x0).to(dev), torch.from_numpy(x1).to(dev)
    del x0, x1
    o8 = torch.empty_like(d0)
    m = (16 + world - 1) // world
    gb = torch.empty((world, m, 1080, 1920, 3), dtype=torch.float32, device=dev)
    ms, _ = timed(lambda: parallel.interpolate_tiled_device(edev, d0, d1, [4, 4], out=o8, gather_buf=gb), 2)
    rec8 = {"value": 1000.0 / ms, "unit": "frames/s", "ms_per_frame": ms, "n_gpus": world,
            "config": f"7680x4320, block 4x4 (16 tiles of 1080x1920), tiles round-robin over {world} GPU(s), one in-place "
                      "NCCL all-gather of the tile slots + one device stitch copy inside the timed region",
            "all_gather_bytes": int(gb.numel() * 4) if world > 1 else 0}
    if world > 1:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dist.barrier()
        torch.cuda.synchronize()
        e0.record()
        parallel._all_gather_slots(gb)
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        rec8["all_gather_ms"] = float(t.item())
        ref8 = torch.empty_like(o8)
        with _solo(parallel, solo):
            parallel.interpolate_tiled_device(edev, d0, d1, [4, 4], out=ref8)
        torch.cuda.synchronize()
        ok = torch.tensor([int(torch.equal(ref8, o8))], device=dev)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        rec8["bitwise_equal_to_1gpu"] = bool(ok.item())
        del ref8
    out["8k_tiled_4x4"] = rec8
    del d0, d1, o8, gb
    # ---- 720p recursive x6: 63 mid-frames, level-synchronous over the ranks (configs[3]; eval/util.py:62-91)
    f0, f1 = synthetic.frame_pair(720, 1280, seed=9, n_waves=8)
    t0_, t1_ = torch.from_numpy(f0[0]).to(dev), torch.from_numpy(f1[0]).to(dev)
    ms, seq = timed(lambda: parallel.interpolate_recursively_device(edev, t0_, t1_, 6), 1)
    recr = {"value": 63.0 * 1000.0 / ms, "unit": "mid-frames/s", "ms_per_sequence": ms, "n_gpus": world,
            "config": f"1280x720 (padded 768x1280), times_to_interpolate 6 = 63 network calls in 6 dependency levels, level-"
                      f"synchronous over {world} GPU(s) (critical path {sum(-(-(1 << k) // world) for k in range(6))} calls), parents "
                      "stay in HBM, one in-place NCCL all-gather of the new mid-frames per level"}
    if world > 1:
        with _solo(parallel, solo):
            ref = parallel.interpolate_recursively_device(edev, t0_, t1_, 6)
        torch.cuda.synchronize()
        ok = torch.tensor([int(torch.equal(ref, seq))], device=dev)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        recr["bitwise_equal_to_1gpu"] = bool(ok.item())
    out["720p_recursive_x6"] = recr
    torch.cuda.synchronize()
    return out


class _SoloGroup:
    """Marker: run a sharded path on this rank alone (the 1-GPU result the sharded one is checked against)."""


class _solo:
    def __init__(self, parallel, marker):
        self.p, self.marker = parallel, marker

    def __enter__(self):
        self.saved = self.p._world_rank
        self.p._world_rank = lambda group=None: (1, 0)

    def __exit__(self, *a):
        self.p._world_rank = self.saved


DUMP_BUDGET_BYTES = 64 << 20


def dump_frame(out_dir, frame):
    """The interpolated frame as float32 .npy: whole while it fits DUMP_BUDGET_BYTES, otherwise a fixed sample of pixels
    (seeded, sorted flat pixel indices, all three channels) with the indices beside it."""
    os.makedirs(out_dir, exist_ok=True)
    frame = np.ascontiguousarray(frame, dtype=np.float32)
    if frame.nbytes <= DUMP_BUDGET_BYTES:
        np.save(os.path.join(out_dir, "interpolated_frame.npy"), frame)
        return
    pix = frame.reshape(-1, frame.shape[-1])
    n = DUMP_BUDGET_BYTES // 2 // (pix.shape[1] * 4)    # half the budget for the values, the rest covers the indices
    idx = np.sort(np.random.default_rng(0).choice(pix.shape[0], size=n, replace=False))
    np.save(os.path.join(out_dir, "interpolated_frame_sample.npy"), pix[idx])
    np.save(os.path.join(out_dir, "interpolated_frame_sample_pixels.npy"), idx.astype(np.float64))   # exact below 2^53


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--height", type=int, default=H1080)
    ap.add_argument("--width", type=int, default=W1080)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-workloads", action="store_true", help="skip the 4K / 8K / 720p-recursive workloads")
    ap.add_argument("--op-table", default=None, help="write the per-kernel timing table (csv) here")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write the last timed step's interpolated frame as DIR/interpolated_frame.npy (float32)")
    args = ap.parse_args()
    if args.impl == "reference":
        return run_reference(args)

    import torch
    import torch.distributed as dist
    from frame_interpolation_b200 import spec, synthetic
    from frame_interpolation_b200.interpolator import Interpolator

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device; the engine has no CPU fallback")
    torch.cuda.set_device(local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    W = max(args.warmup, 3)
    K = max(args.steps, 1)
    h, w = args.height, args.width

    eng = Interpolator("synthetic", align=64, device=local_rank)
    x0, x1 = synthetic.frame_pair(h, w, seed=rank, n_waves=8)
    dt = np.full((1,), 0.5, np.float32)
    dev = torch.device("cuda", local_rank)
    d0 = torch.from_numpy(x0).to(dev)
    d1 = torch.from_numpy(x1).to(dev)
    dout = torch.empty_like(d0)
    # a real (non-NULL) stream: the engine treats NULL as "use my own stream", and
    # torch.cuda.Event only sees work enqueued on the stream it is recorded on.
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def step_device():
        eng.interpolate_device(d0.data_ptr(), d1.data_ptr(), 1, h, w, dout.data_ptr(), stream=stream.cuda_stream)

    # ---- device-resident throughput ------------------------------------------------
    for _ in range(W):
        step_device()
    barrier()
    sampler = ClockSampler(local_rank)
    with sampler:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        barrier()
        e0.record(stream)
        for _ in range(K):
            step_device()
        e1.record(stream)
        barrier()
        ms = e0.elapsed_time(e1)
    if args.dump_outputs and rank == 0:
        dump_frame(args.dump_outputs, dout.cpu().numpy())
    t_ms = torch.tensor([ms], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t_ms, op=dist.ReduceOp.MAX)
    ms_total = float(t_ms.item())
    value = world * K / (ms_total / 1e3)
    prof = eng.profile()

    # ---- end to end through the reference-facing API (host buffers) -----------------
    hx0 = torch.from_numpy(x0).pin_memory().numpy()
    hx1 = torch.from_numpy(x1).pin_memory().numpy()
    for _ in range(2):
        eng(hx0, hx1, dt)
    barrier()
    t0 = time.perf_counter()
    for _ in range(K):
        res = eng(hx0, hx1, dt)
    torch.cuda.synchronize()
    t_e2e = torch.tensor([time.perf_counter() - t0], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t_e2e, op=dist.ReduceOp.MAX)
    e2e_value = world * K / float(t_e2e.item())
    frame_bytes = int(x0.nbytes)

    # parity guard: device path and host path must agree bit for bit
    same = bool(np.array_equal(res, dout.cpu().numpy()))

    # ---- the same call with 8-bit frames at the boundary (eval/util.py read_image / write_image semantics on the
    #      device): a quarter of the PCIe bytes; reported next to `e2e`, never instead of it
    e2e_u8 = None
    try:
        from frame_interpolation_b200 import eval_util
        u0 = torch.from_numpy(eval_util.to_uint8(x0)).pin_memory().numpy()
        u1 = torch.from_numpy(eval_util.to_uint8(x1)).pin_memory().numpy()
        for _ in range(2):
            eng.interpolate_u8(u0, u1)
        barrier()
        t0 = time.perf_counter()
        for _ in range(K):
            eng.interpolate_u8(u0, u1)
        torch.cuda.synchronize()
        t_u8 = torch.tensor([time.perf_counter() - t0], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t_u8, op=dist.ReduceOp.MAX)
        e2e_u8 = {"value": world * K / float(t_u8.item()), "unit": "frames/s", "api": "Interpolator.interpolate_u8(x0, x1)",
                  "h2d_bytes_per_step": 2 * int(u0.nbytes), "d2h_bytes_per_step": int(u0.nbytes)}
    except Exception as exc:           # secondary number: never fatal
        e2e_u8 = {"error": f"{type(exc).__name__}: {exc}"}

    # ---- per-kernel pass (eager, one event pair per launch) -------------------------
    eng.set_option("time_ops", 1)
    acc = None
    reps = 3
    for _ in range(reps):
        eng.interpolate_device(d0.data_ptr(), d1.data_ptr(), 1, h, w, dout.data_ptr())
        eng.synchronize()
        tab = eng.op_table()
        if acc is None:
            acc = tab
        else:
            for a, b in zip(acc, tab):
                a["ms"] += b["ms"]
    for a in acc:
        a["ms"] /= reps
    eng.set_option("time_ops", 0)
    conv = [a for a in acc if a["category"] == 0]
    gath = [a for a in acc if a["category"] == 1]
    conv_ms = sum(a["ms"] for a in conv)
    gath_ms = sum(a["ms"] for a in gath)
    all_ms = sum(a["ms"] for a in acc)
    conv_flops = sum(a["ref_flops"] for a in conv)
    gath_bytes = sum(a["alg_bytes"] for a in gath)
    peaks = load_peaks()
    mask = eng.get_option("onepass_mask")
    names = eng.stage_names()
    one_pass = [n for i, n in enumerate(names) if (mask >> i) & 1]
    three_pass = [n for i, n in enumerate(names) if not (mask >> i) & 1]
    ach_tf = conv_flops / (conv_ms * 1e-3) / 1e12
    roofline = {
        "bound": "tensor", "kernel": "k_conv_tc / k_conv3x3_tc (wgmma implicit-GEMM conv, all call sites)",
        "achieved": ach_tf, "peak": peaks["bf16_tflops_sustained"], "unit": "TFLOP/s",
        "frac": ach_tf / peaks["bf16_tflops_sustained"],
        "traffic_note": "`algorithmic_bytes_per_step` is the engine's own count (every source plane a call site consumes "
                        "read once, every destination plane written once)",
        "algorithmic_bytes_per_step": sum(a["alg_bytes"] for a in conv),
        "peak_source": peaks["source"],
        "mma_kind": "wgmma.mma_async f32.f16.f16 (fp16 operands, fp32 accumulate); per-stage precision plan: 1 pass (hi*hi) on "
                    + ",".join(one_pass) + "; 3 passes (hi*hi + hi*lo + lo*hi) on " + ",".join(three_pass) + " and the heads",
        "onepass_mask": hex(mask),
        "issued_tflops": prof["mma_flops"] / (conv_ms * 1e-3) / 1e12,
        "issued_frac": prof["mma_flops"] / (conv_ms * 1e-3) / 1e12 / peaks["bf16_tflops_sustained"],
        "algorithmic_flops_per_step": conv_flops, "conv_kernel_ms_per_step": conv_ms,
        "conv_launches_per_step": len(conv), "share_of_step": conv_ms / all_ms,
    }
    gather = {"bound": "hbm", "kernel": "k_flow_warp / k_fusion_warp (bilinear gather)",
              "achieved": gath_bytes / (gath_ms * 1e-3) / 1e9, "peak": peaks["hbm_gbs"], "unit": "GB/s",
              "frac": gath_bytes / (gath_ms * 1e-3) / 1e9 / peaks["hbm_gbs"], "ms_per_step": gath_ms,
              "algorithmic_bytes_per_step": gath_bytes, "share_of_step": gath_ms / all_ms}
    extra = None
    if not args.no_workloads:
        try:
            extra = extra_workloads(eng, world, rank, dev, dist if world > 1 else None)
        except Exception as exc:      # the headline line must survive a failure of the secondary workloads
            import traceback
            traceback.print_exc()
            extra = {"error": f"{type(exc).__name__}: {exc}"}
            torch.cuda.synchronize()
    if args.op_table and rank == 0:
        with open(args.op_table, "w") as f:
            f.write("idx,category,name,ms,ref_flops,alg_bytes\n")
            for a in acc:
                f.write(f'{a["idx"]},{a["category"]},{a["name"]},{a["ms"]:.5f},{a["ref_flops"]:.0f},{a["alg_bytes"]:.0f}\n')

    line = {
        "metric": METRIC, "value": value, "unit": "frames/s", "n_gpus": world, "steps": K, "warmup": W,
        "ms_per_step": ms_total / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f16x2-split (activations/weights as fp16 hi+lo planes; fp32 accumulate)", "data": "synthetic",
        "config": {"workload": WORKLOAD_1080P if (h, w) == (H1080, W1080) else
                               f"{w}x{h} single mid-frame, Style architecture, batch 1, align 64 -> {prof['padded_h']}x{prof['padded_w']}",
                   "per_gpu": "one frame pair per GPU per step",
                   "weights": "synthetic seed 1234 (random-init Style architecture)",
                   "l2": f"per-step working set {prof['arena_bytes'] / 1e9:.1f} GB >> 50 MB L2 (no flush needed)",
                   "parallelism": f"frame-pair sharding x{world} (one process per GPU, no data-path collective)",
                   "cuda_graph": bool(prof["used_graph"])},
        "e2e": {"value": e2e_value, "unit": "frames/s", "h2d_bytes_per_step": 2 * frame_bytes,
                "d2h_bytes_per_step": frame_bytes, "host_memory": "pinned", "api": "Interpolator.__call__(x0, x1, dt)",
                "device_vs_host_path_bitwise_equal": same},
        "e2e_u8": e2e_u8,
        "gpu_launches": int(prof["kernel_launches"]) * K,
        "clocks": sampler.summary(),
        "roofline": roofline,
        "gather": gather,
        "conv_tflops_per_step_algorithmic": conv_flops / 1e12,
    }
    if extra is not None:
        line["workloads"] = extra
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        orc = CpuOracle1080p()
        sec = orc.step()
        line["cpu_baseline"] = {"value": 1.0 / sec, "unit": "frames/s", "cores": orc.threads, "kind": "port",
                                "sample": orc.sample + " (same sample as the --impl reference arm)"}
    if rank == 0:
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
