"""Image-quality metrics of the reference's benchmark evaluator, TensorFlow-free:
`psnr` / `ssim` as used by losses/losses.py:103-113
(`tf.image.psnr(max_val=1.0)`, `tf.image.ssim(max_val=1.0)` with TF's defaults: 11x11 Gaussian
window, sigma 1.5, k1 = 0.01, k2 = 0.03, VALID windows, mean over channels and positions).
Used for the PSNR-delta parity figure; inputs are (..., H, W, C) float arrays."""
from __future__ import annotations

import numpy as np


def l1(a: np.ndarray, b: np.ndarray) -> float:
    """losses.py:72-74 (l1_loss): mean absolute difference."""
    return float(np.mean(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64))))


def l2(a: np.ndarray, b: np.ndarray) -> float:
    """losses.py:98-100 (l2_loss): mean squared difference."""
    return float(np.mean((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2))


def psnr(a: np.ndarray, b: np.ndarray, max_val: float = 1.0) -> float:
    """10 * log10(max_val^2 / mse), mse over the last three axes (per image), averaged over the batch."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    mse = np.mean((a - b) ** 2, axis=(-3, -2, -1))
    with np.errstate(divide="ignore"):
        return float(np.mean(10.0 * np.log10(max_val * max_val / mse)))


def _gauss_window(size: int = 11, sigma: float = 1.5) -> np.ndarray:
    x = np.arange(size, dtype=np.float64) - (size - 1) / 2.0
    g = np.exp(-(x * x) / (2.0 * sigma * sigma))
    return g / g.sum()


def _filter_valid(x: np.ndarray, g: np.ndarray) -> np.ndarray:
    """Separable VALID correlation over the H and W axes of (..., H, W, C)."""
    n = len(g)
    h, w = x.shape[-3], x.shape[-2]
    out = sum(g[i] * x[..., i:h - n + 1 + i, :, :] for i in range(n))
    return sum(g[i] * out[..., :, i:w - n + 1 + i, :] for i in range(n))


def ssim(a: np.ndarray, b: np.ndarray, max_val: float = 1.0, filter_size: int = 11, filter_sigma: float = 1.5,
         k1: float = 0.01, k2: float = 0.03) -> float:
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    if a.shape[-3] < filter_size or a.shape[-2] < filter_size:
        raise ValueError("images must be at least filter_size x filter_size")
    g = _gauss_window(filter_size, filter_sigma)
    c1, c2 = (k1 * max_val) ** 2, (k2 * max_val) ** 2
    mu_a, mu_b = _filter_valid(a, g), _filter_valid(b, g)
    s_aa = _filter_valid(a * a, g) - mu_a * mu_a
    s_bb = _filter_valid(b * b, g) - mu_b * mu_b
    s_ab = _filter_valid(a * b, g) - mu_a * mu_b
    lum = (2 * mu_a * mu_b + c1) / (mu_a * mu_a + mu_b * mu_b + c1)
    cs = (2 * s_ab + c2) / (s_aa + s_bb + c2)
    return float(np.mean(lum * cs))
