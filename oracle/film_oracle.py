"""CPU ORACLE for the FILM inference hot path -- TEST INFRASTRUCTURE, NOT PRODUCT.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module. The engine (frame_interpolation_b200/) never does and has
no CPU fallback.

PARITY UNPINNED: the reference ships no unit tests and no golden vectors, and its arithmetic
lives in un-vendored third-party packages that are absent
from this image -- tensorflow==2.6.2 and tensorflow-addons==0.15.0 (reference
requirements.txt:2,4) -- and no pre-trained SavedModel exists on disk. This file is an
op-for-op restatement of the reference graph in PyTorch-CPU with the TF / TFA op semantics
written out explicitly (each one has a closed-form unit test in tests/test_oracle_ops.py).
It has NOT been executed against TensorFlow. An independently written pure-numpy restatement of the whole graph
(tests/test_oracle_independent.py) agrees with this file to 1e-9 in fp64.

Restated functions (reference file:line):
  build_image_pyramid      models/film_net/util.py:23-45
  SubTreeExtractor.call    models/film_net/feature_extractor.py:125-147
  FeatureExtractor.call    models/film_net/feature_extractor.py:163-193
  FlowEstimator.call       models/film_net/pyramid_flow_estimator.py:85-98
  PyramidFlowEstimator.call models/film_net/pyramid_flow_estimator.py:125-163
  warp                     models/film_net/util.py:48-82 (+ tfa.image.dense_image_warp 0.15)
  multiply_pyramid         models/film_net/util.py:85-103
  flow_pyramid_synthesis   models/film_net/util.py:106-117
  pyramid_warp / concatenate_pyramids  models/film_net/util.py:120-143
  Fusion.call              models/film_net/fusion.py:103-140
  create_model             models/film_net/interpolator.py:120-207
  _pad_to_align            eval/interpolator.py:30-63
  image_to_patches / patches_to_image  eval/interpolator.py:66-126
  Interpolator.interpolate / __call__  eval/interpolator.py:152-209

Everything is NHWC at the interface (like the reference) and NCHW internally.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Mapping, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

# --- architecture constants: training/config/film_net-Style.gin:17-23 -------------------
PYRAMID_LEVELS = 7
FUSION_PYRAMID_LEVELS = 5
SPECIALIZED_LEVELS = 3
SUB_LEVELS = 4
FLOW_CONVS = [3, 3, 3, 3]
FLOW_FILTERS = [32, 64, 128, 256]
FILTERS = 64
FLOW_PREDICTOR_NAMES = ["flow_predictor_0", "flow_predictor_1", "flow_predictor_2",
                        "flow_predictor_shared"]

Tensor = torch.Tensor


# =========================================================================================
# Third-party op semantics (TF 2.6 / TFA 0.15), written out
# =========================================================================================
def leaky_relu(x: Tensor) -> Tensor:
    """tf.nn.leaky_relu(x, alpha=0.2) (feature_extractor.py:89-90)."""
    return torch.where(x >= 0, x, x * 0.2)


def conv2d_same(x: Tensor, kernel_hwio: Tensor, bias: Tensor, activation: bool) -> Tensor:
    """tf.keras.layers.Conv2D(padding='same', strides=1): cross-correlation, HWIO kernel.

    SAME padding puts the odd pixel AFTER: k=3 -> 1 on every side; k=2 -> 0 top/left and
    1 bottom/right; k=1 -> none. x is NCHW.
    """
    kh, kw = int(kernel_hwio.shape[0]), int(kernel_hwio.shape[1])
    pt, pl = (kh - 1) // 2, (kw - 1) // 2
    pb, pr = (kh - 1) - pt, (kw - 1) - pl
    if pt or pl or pb or pr:
        x = F.pad(x, (pl, pr, pt, pb))
    w = kernel_hwio.permute(3, 2, 0, 1).contiguous()
    y = F.conv2d(x, w, bias)
    return leaky_relu(y) if activation else y


def avg_pool_2x2(x: Tensor) -> Tensor:
    """AveragePooling2D(pool_size=2, strides=2, padding='valid'): trailing odd row/col dropped."""
    h, w = x.shape[-2] // 2 * 2, x.shape[-1] // 2 * 2
    x = x[..., :h, :w]
    return (x[..., 0::2, 0::2] + x[..., 0::2, 1::2] + x[..., 1::2, 0::2] + x[..., 1::2, 1::2]) * 0.25


def _resize_weights(in_size: int, out_size: int, dtype, device):
    """TF2 resize, half_pixel_centers=True, antialias=False:
    src = (dst + 0.5) * (in/out) - 0.5 ; lo = max(floor(src), 0) ; hi = min(ceil(src), in-1) ;
    lerp = src - floor(src)."""
    scale = in_size / out_size
    dst = torch.arange(out_size, dtype=dtype, device=device)
    src = (dst + 0.5) * scale - 0.5
    fl = torch.floor(src)
    lo = torch.clamp(fl, min=0).long()
    hi = torch.clamp(torch.ceil(src), max=in_size - 1).long()
    return lo, hi, src - fl


def resize_bilinear(x: Tensor, size: Tuple[int, int]) -> Tensor:
    """tf.image.resize(x, size) with the TF2 default method (bilinear). NCHW."""
    ih, iw = x.shape[-2:]
    oh, ow = size
    ylo, yhi, yl = _resize_weights(ih, oh, x.dtype, x.device)
    xlo, xhi, xl = _resize_weights(iw, ow, x.dtype, x.device)
    top_rows, bot_rows = x[..., ylo, :], x[..., yhi, :]
    tl, tr = top_rows[..., xlo], top_rows[..., xhi]
    bl, br = bot_rows[..., xlo], bot_rows[..., xhi]
    top = tl + (tr - tl) * xl
    bot = bl + (br - bl) * xl
    return top + (bot - top) * yl[:, None]


def resize_nearest(x: Tensor, size: Tuple[int, int]) -> Tensor:
    """tf.image.resize(..., NEAREST_NEIGHBOR) in TF2: src = floor((dst + 0.5) * in/out)."""
    ih, iw = x.shape[-2:]
    oh, ow = size
    ys = torch.clamp(torch.floor((torch.arange(oh, dtype=torch.float64) + 0.5) * (ih / oh)).long(), max=ih - 1)
    xs = torch.clamp(torch.floor((torch.arange(ow, dtype=torch.float64) + 0.5) * (iw / ow)).long(), max=iw - 1)
    return x[..., ys, :][..., xs]


def dense_image_warp(image: Tensor, flow_yx: Tensor) -> Tensor:
    """tfa.image.dense_image_warp(image, flow) (TFA 0.15). image NCHW, flow_yx (N,2,H,W) in
    (dy, dx) order. query = grid - flow; interpolate_bilinear(indexing='ij'):
    per axis floor = min(max(0, floor(q)), size-2), alpha = clip(q - floor, 0, 1)."""
    n, c, h, w = image.shape
    assert h >= 2 and w >= 2, "dense_image_warp needs H, W >= 2"
    gy = torch.arange(h, dtype=image.dtype).view(1, h, 1)
    gx = torch.arange(w, dtype=image.dtype).view(1, 1, w)
    qy = gy - flow_yx[:, 0]
    qx = gx - flow_yx[:, 1]
    fy = torch.clamp(torch.floor(qy), 0, h - 2)
    fx = torch.clamp(torch.floor(qx), 0, w - 2)
    ay = torch.clamp(qy - fy, 0, 1).unsqueeze(1)
    ax = torch.clamp(qx - fx, 0, 1).unsqueeze(1)
    fy, fx = fy.long(), fx.long()
    flat = image.reshape(n, c, h * w)

    def gather(yy, xx):
        idx = (yy * w + xx).view(n, 1, h * w).expand(n, c, h * w)
        return torch.gather(flat, 2, idx).view(n, c, h, w)

    tl, tr = gather(fy, fx), gather(fy, fx + 1)
    bl, br = gather(fy + 1, fx), gather(fy + 1, fx + 1)
    top = ax * (tr - tl) + tl
    bot = ax * (br - bl) + bl
    return ay * (bot - top) + top


# =========================================================================================
# models/film_net restated
# =========================================================================================
def warp(image: Tensor, flow_xy: Tensor) -> Tensor:
    """util.py:48-82: out[y,x] = bilinear(image, y + flow[...,1], x + flow[...,0]);
    implemented as dense_image_warp(image, -flow[..., ::-1])."""
    return dense_image_warp(image, -flow_xy.flip(1))


def build_image_pyramid(image: Tensor) -> List[Tensor]:
    pyr = []
    for i in range(PYRAMID_LEVELS):
        pyr.append(image)
        if i < PYRAMID_LEVELS - 1:
            image = avg_pool_2x2(image)
    return pyr


class Oracle:
    """Holds the weights as torch tensors and evaluates the reference graph."""

    def __init__(self, weights: Mapping[str, np.ndarray], dtype=torch.float32,
                 conv_hook: Optional[Callable] = None, num_threads: Optional[int] = None):
        self.dtype = dtype
        self.w = {k: torch.from_numpy(np.asarray(v)).to(dtype) for k, v in weights.items()}
        # conv_hook(x, kernel, layer_name) -> (x', kernel') lets error-budget studies emulate reduced
        # precision operand formats; None for the oracle proper.
        self.conv_hook = conv_hook
        if num_threads:
            torch.set_num_threads(num_threads)

    def _conv(self, x: Tensor, name: str, activation: bool) -> Tensor:
        k, b = self.w[name + "/kernel"], self.w[name + "/bias"]
        if self.conv_hook is not None:
            x, k = self.conv_hook(x, k, name)
        return conv2d_same(x, k, b, activation)

    # feature_extractor.py:125-147
    def sub_tree(self, image: Tensor, n: int) -> List[Tensor]:
        head, pyr = image, []
        for i in range(n):
            head = self._conv(head, f"feat_net/sub_extractor/cfeat_conv_{2 * i}", True)
            head = self._conv(head, f"feat_net/sub_extractor/cfeat_conv_{2 * i + 1}", True)
            pyr.append(head)
            if i < n - 1:
                head = avg_pool_2x2(head)
        return pyr

    # feature_extractor.py:163-193
    def feature_pyramid(self, image_pyramid: Sequence[Tensor]) -> List[Tensor]:
        subs = [self.sub_tree(image_pyramid[i], min(len(image_pyramid) - i, SUB_LEVELS))
                for i in range(len(image_pyramid))]
        out = []
        for i in range(len(image_pyramid)):
            feats = subs[i][0]
            for j in range(1, SUB_LEVELS):
                if j <= i:
                    feats = torch.cat([feats, subs[i - j][j]], dim=1)
            out.append(feats)
        return out

    # pyramid_flow_estimator.py:85-98
    def flow_estimator(self, p: int, a: Tensor, b: Tensor) -> Tensor:
        name = FLOW_PREDICTOR_NAMES[p]
        net = torch.cat([a, b], dim=1)
        n3 = FLOW_CONVS[p]
        for k in range(n3):
            net = self._conv(net, f"predict_flow/{name}/conv_{k}", True)
        net = self._conv(net, f"predict_flow/{name}/conv_{n3}", True)
        return self._conv(net, f"predict_flow/{name}/conv_{n3 + 1}", False)

    # pyramid_flow_estimator.py:125-163
    def pyramid_flow(self, fa: Sequence[Tensor], fb: Sequence[Tensor]) -> List[Tensor]:
        levels = len(fa)
        pred = lambda l: min(l, SPECIALIZED_LEVELS)
        v = self.flow_estimator(pred(levels - 1), fa[-1], fb[-1])
        residuals = [v]
        for i in reversed(range(levels - 1)):
            v = resize_bilinear(2 * v, tuple(fa[i].shape[-2:]))
            warped = warp(fb[i], v)
            r = self.flow_estimator(pred(i), fa[i], warped)
            residuals.append(r)
            v = r + v
        return list(reversed(residuals))

    # fusion.py:103-140
    def fusion(self, pyramid: Sequence[Tensor]) -> Tensor:
        net = pyramid[-1]
        for i in reversed(range(FUSION_PYRAMID_LEVELS - 1)):
            net = resize_nearest(net, tuple(pyramid[i].shape[-2:]))
            net = self._conv(net, f"fusion/level_{i}/conv_0", False)
            net = torch.cat([pyramid[i], net], dim=1)
            net = self._conv(net, f"fusion/level_{i}/conv_1", True)
            net = self._conv(net, f"fusion/level_{i}/conv_2", True)
        return self._conv(net, "fusion/output_conv", False)

    # interpolator.py:120-207
    def model(self, x0: Tensor, x1: Tensor, aux: Optional[Dict] = None) -> Tensor:
        """x0, x1: NCHW. Returns NCHW image (B,3,H,W). `time` is ignored by the
        reference (interpolator.py:102,163), so it is not an argument here."""
        img_pyr = [build_image_pyramid(x0), build_image_pyramid(x1)]
        feat_pyr = [self.feature_pyramid(img_pyr[0]), self.feature_pyramid(img_pyr[1])]
        fwd_res = self.pyramid_flow(feat_pyr[0], feat_pyr[1])
        bwd_res = self.pyramid_flow(feat_pyr[1], feat_pyr[0])
        n = FUSION_PYRAMID_LEVELS
        fwd_flow = flow_pyramid_synthesis(fwd_res)[:n]
        bwd_flow = flow_pyramid_synthesis(bwd_res)[:n]
        # multiply_pyramid with mid_time = 0.5 and 1 - 0.5
        backward_flow = [f * 0.5 for f in bwd_flow]
        forward_flow = [f * 0.5 for f in fwd_flow]
        to_warp = [[torch.cat([img_pyr[k][l], feat_pyr[k][l]], dim=1) for l in range(n)]
                   for k in range(2)]
        fwd_warped = [warp(t, f) for t, f in zip(to_warp[0], backward_flow)]
        bwd_warped = [warp(t, f) for t, f in zip(to_warp[1], forward_flow)]
        aligned = [torch.cat([a, b, c, d], dim=1)
                   for a, b, c, d in zip(fwd_warped, bwd_warped, backward_flow, forward_flow)]
        pred = self.fusion(aligned)
        if aux is not None:
            aux.update(image_pyramids=img_pyr, feature_pyramids=feat_pyr,
                       forward_residual_flow_pyramid=fwd_res, backward_residual_flow_pyramid=bwd_res,
                       forward_flow_pyramid=fwd_flow, backward_flow_pyramid=bwd_flow,
                       aligned_pyramid=aligned)
        return pred[:, :3]


def flow_pyramid_synthesis(residuals: Sequence[Tensor]) -> List[Tensor]:
    """util.py:106-117."""
    flow = residuals[-1]
    out = [flow]
    for r in reversed(residuals[:-1]):
        flow = resize_bilinear(2 * flow, tuple(r.shape[-2:]))
        flow = r + flow
        out.append(flow)
    return list(reversed(out))


# =========================================================================================
# eval/interpolator.py restated (numpy NHWC at the boundary)
# =========================================================================================
def pad_to_align(x: np.ndarray, align: int):
    """eval/interpolator.py:30-63. Returns (padded, (off_h, off_w, h, w))."""
    assert np.ndim(x) == 4
    assert align > 0, "align must be a positive number."
    h, w = x.shape[-3:-1]
    ph = (align - h % align) if h % align != 0 else 0
    pw = (align - w % align) if w % align != 0 else 0
    oh, ow = ph // 2, pw // 2
    out = np.zeros((x.shape[0], h + ph, w + pw, x.shape[3]), x.dtype)
    out[:, oh:oh + h, ow:ow + w] = x
    return out, (oh, ow, h, w)


def image_to_patches(image: np.ndarray, block_shape: Sequence[int]) -> np.ndarray:
    """eval/interpolator.py:66-99: row-major non-overlapping tiles, tile index r*bw + c."""
    bh, bw = block_shape
    h, w, c = image.shape[-3:]
    ph, pw = h // bh, w // bw
    assert h == ph * bh, "block_height=%d should evenly divide height=%d." % (bh, h)
    assert w == pw * bw, "block_width=%d should evenly divide width=%d." % (bw, w)
    x = image.reshape(bh, ph, bw, pw, c).transpose(0, 2, 1, 3, 4)
    return np.ascontiguousarray(x.reshape(bh * bw, ph, pw, c))


def patches_to_image(patches: np.ndarray, block_shape: Sequence[int]) -> np.ndarray:
    """eval/interpolator.py:102-126."""
    bh, bw = block_shape
    ph, pw, c = patches.shape[-3:]
    x = patches.reshape(bh, bw, ph, pw, c).transpose(0, 2, 1, 3, 4)
    return np.ascontiguousarray(x.reshape(1, bh * ph, bw * pw, c))


class OracleInterpolator:
    """eval/interpolator.py:129-209 with the SavedModel call replaced by `Oracle.model`."""

    def __init__(self, weights: Mapping[str, np.ndarray], align: Optional[int] = None,
                 block_shape: Optional[Sequence[int]] = None, dtype=torch.float32,
                 conv_hook=None, num_threads: Optional[int] = None):
        self._oracle = Oracle(weights, dtype, conv_hook, num_threads)
        self._align = align or None
        self._block_shape = block_shape or None

    def interpolate(self, x0: np.ndarray, x1: np.ndarray, dt: np.ndarray,
                    aux: Optional[Dict] = None) -> np.ndarray:
        if self._align is not None:
            x0, (oh, ow, h, w) = pad_to_align(x0, self._align)
            x1, _ = pad_to_align(x1, self._align)
        dt = np.asarray(dt)
        assert dt.shape[0] == x0.shape[0]
        t0 = torch.from_numpy(np.ascontiguousarray(x0)).to(self._oracle.dtype).permute(0, 3, 1, 2)
        t1 = torch.from_numpy(np.ascontiguousarray(x1)).to(self._oracle.dtype).permute(0, 3, 1, 2)
        with torch.no_grad():
            img = self._oracle.model(t0, t1, aux).permute(0, 2, 3, 1)
        out = img.to(torch.float32).numpy() if self._oracle.dtype == torch.float32 else img.numpy()
        if self._align is not None:
            out = out[:, oh:oh + h, ow:ow + w]
        return np.ascontiguousarray(out)

    def __call__(self, x0: np.ndarray, x1: np.ndarray, dt: np.ndarray) -> np.ndarray:
        if self._block_shape is not None and np.prod(self._block_shape) > 1:
            p0 = image_to_patches(x0, self._block_shape)
            p1 = image_to_patches(x1, self._block_shape)
            outs = [self.interpolate(a[np.newaxis], b[np.newaxis], dt) for a, b in zip(p0, p1)]
            return patches_to_image(np.concatenate(outs, axis=0), self._block_shape)
        return self.interpolate(x0, x1, dt)
