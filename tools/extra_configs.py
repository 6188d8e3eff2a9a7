"""BASELINE.json configs[2..4] on one H100 through the public API (host buffers): 4K tiled 2x2,
720p recursive times_to_interpolate=6 (63 mid-frames, device-resident recursion), 8K tiled 4x4."""
import json, os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from frame_interpolation_b200 import synthetic
from frame_interpolation_b200.interpolator import Interpolator

dt = np.full((1,), 0.5, np.float32)
out = {}

def tile_frame(h, w, seed):
    # synthetic texture generation is O(pixels * waves): build 1080p once and tile it
    a, b = synthetic.frame_pair(1080, 1920, seed=seed, n_waves=6)
    ry, rx = h // 1080, w // 1920
    return np.tile(a, (1, ry, rx, 1)), np.tile(b, (1, ry, rx, 1))

# 4K tiled 2x2
x0, x1 = tile_frame(2160, 3840, 0)
eng = Interpolator("synthetic", align=64, block_shape=[2, 2])
eng(x0, x1, dt)
t = time.perf_counter(); n = 3
for _ in range(n): y = eng(x0, x1, dt)
el = (time.perf_counter() - t) / n
single = Interpolator("synthetic", align=64)
tile = single(x0[:, :1080, :1920], x1[:, :1080, :1920], dt)
out["4k_tiled_2x2"] = {"ms_per_frame": el * 1e3, "frames_per_s": 1 / el, "tile_equals_single_call": bool(np.array_equal(y[:, :1080, :1920], tile)),
                       "profile": {k: eng.profile()[k] for k in ("last_call_ms", "last_h2d_ms", "last_d2h_ms")}}
eng.close()

# 720p recursive x6
a, b = synthetic.frame_pair(720, 1280, seed=1, n_waves=6)
single.interpolate_recursively(a[0], b[0], 1)
t = time.perf_counter()
seq = single.interpolate_recursively(a[0], b[0], 6)
el = time.perf_counter() - t
p = single.profile()
out["720p_recursive_x6"] = {"mid_frames": 63, "seconds": el, "mid_frames_per_s": 63 / el, "device_ms": p["last_call_ms"],
                            "h2d_ms": p["last_h2d_ms"], "d2h_ms": p["last_d2h_ms"], "finite": bool(np.isfinite(seq).all())}
# host-path recursion for comparison (the reference's calling pattern: H2D + D2H + sync per mid-frame)
t = time.perf_counter()
def rec(f1, f2, n):
    if n == 0: return [f1]
    m = single(f1[None], f2[None], dt)[0]
    return rec(f1, m, n - 1) + rec(m, f2, n - 1)
ref = rec(a[0], b[0], 4)
el = time.perf_counter() - t
out["720p_recursive_x4_host_path"] = {"mid_frames": 15, "mid_frames_per_s": 15 / el,
                                      "equal_to_device_path": bool(all(np.array_equal(u, v) for u, v in zip(ref, seq[::4])))}
single.close()

# 8K tiled 4x4
x0, x1 = tile_frame(4320, 7680, 2)
eng = Interpolator("synthetic", align=64, block_shape=[4, 4])
eng(x0, x1, dt)
t = time.perf_counter()
y = eng(x0, x1, dt)
el = time.perf_counter() - t
out["8k_tiled_4x4"] = {"ms_per_frame": el * 1e3, "frames_per_s": 1 / el, "finite": bool(np.isfinite(y).all())}
print(json.dumps(out, indent=1))
