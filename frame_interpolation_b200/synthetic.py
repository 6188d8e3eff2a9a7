"""Seeded synthetic frame pairs.

Not white noise (flow would be undefined and warps degenerate): a band-limited
texture (sum of random-phase sinusoids per channel) rescaled to [0.05, 0.95];
`x1` is `x0` translated by a sub-pixel global shift plus an independently moving
rectangle and a 2 % gain change, so flows of several pixels exist at level 0.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np


def _texture(rng: np.random.Generator, h: int, w: int, dy: float, dx: float,
             params) -> np.ndarray:
    yy, xx = np.meshgrid(np.arange(h, dtype=np.float64) + dy,
                         np.arange(w, dtype=np.float64) + dx, indexing="ij")
    img = np.zeros((h, w, 3), np.float64)
    for c in range(3):
        for (fy, fx, ph, amp) in params[c]:
            img[..., c] += amp * np.sin(2 * np.pi * (fy * yy + fx * xx) + ph)
    return img


def frame_pair(h: int, w: int, seed: int = 0, n_waves: int = 24) -> Tuple[np.ndarray, np.ndarray]:
    """Returns (x0, x1), each float32 (1, h, w, 3) in [0, 1]."""
    rng = np.random.default_rng(seed)
    params = []
    for _ in range(3):
        p = []
        for _ in range(n_waves):
            period = rng.uniform(6.0, 160.0)
            ang = rng.uniform(0, 2 * np.pi)
            f = 1.0 / period
            p.append((f * np.sin(ang), f * np.cos(ang), rng.uniform(0, 2 * np.pi),
                      rng.uniform(0.3, 1.0) * (period / 160.0) ** 0.5))
        params.append(p)
    t0 = _texture(rng, h, w, 0.0, 0.0, params)
    t1 = _texture(rng, h, w, -3.25, 7.5, params)   # x1(y,x) = x0(y-3.25, x+7.5)
    lo, hi = t0.min(), t0.max()
    x0 = 0.05 + 0.9 * (t0 - lo) / (hi - lo)
    x1 = 0.05 + 0.9 * (t1 - lo) / (hi - lo)
    # moving rectangle (24 px to the right between the frames)
    rh, rw = max(h // 6, 4), max(w // 8, 4)
    ry, rx = h // 3, w // 4
    col = np.array([0.85, 0.2, 0.3])
    x0[ry:ry + rh, rx:rx + rw] = col
    sx = min(rx + 24, w - rw)
    x1[ry:ry + rh, sx:sx + rw] = col
    x1 = np.clip(x1 * 1.02, 0.0, 1.0)
    x0 = np.clip(x0, 0.0, 1.0)
    return x0[None].astype(np.float32), x1[None].astype(np.float32)
