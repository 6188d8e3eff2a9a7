"""Architecture constants of the FILM network (Style / L1 / VGG share them).

Source of every number: reference `training/config/film_net-Style.gin:17-23`
(pyramid_levels=7, fusion_pyramid_levels=5, specialized_levels=3, sub_levels=4,
flow_convs=[3,3,3,3], flow_filters=[32,64,128,256], filters=64) combined with the
layer constructors in `models/film_net/feature_extractor.py:114-123`,
`models/film_net/pyramid_flow_estimator.py:64-83,112-123` and
`models/film_net/fusion.py:70-101`.

The same tables are compiled into the CUDA engine (csrc/film_spec.h); the weight
file is validated against them at load time.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np

PYRAMID_LEVELS = 7
FUSION_PYRAMID_LEVELS = 5
SPECIALIZED_LEVELS = 3
SUB_LEVELS = 4
FLOW_CONVS = [3, 3, 3, 3]
FLOW_FILTERS = [32, 64, 128, 256]
FILTERS = 64
LEAKY_SLOPE = 0.2
ALIGN = 1 << (PYRAMID_LEVELS - 1)  # 64, reference options.py:36-37

FLOW_PREDICTOR_NAMES = ["flow_predictor_0", "flow_predictor_1", "flow_predictor_2",
                        "flow_predictor_shared"]


def feature_channels(level: int) -> int:
    """Channels of the cascaded feature pyramid at `level` (feature_extractor.py:186-192)."""
    return sum(FILTERS << j for j in range(min(level, SUB_LEVELS - 1) + 1))


def fusion_filters(level: int) -> int:
    """fusion.py:77-79."""
    return (FILTERS << level) if level < SPECIALIZED_LEVELS else (FILTERS << SPECIALIZED_LEVELS)


def aligned_channels(level: int) -> int:
    """interpolator.py:167-183: 2*(3 + C_l) + 4."""
    return 2 * (3 + feature_channels(level)) + 4


def weight_table() -> List[Tuple[str, Tuple[int, ...]]]:
    """Ordered list of (name, shape) of every variable. Kernels are HWIO like Keras."""
    t: List[Tuple[str, Tuple[int, ...]]] = []
    # feature extractor: feature_extractor.py:118-123
    cin = 3
    for i in range(SUB_LEVELS):
        c = FILTERS << i
        for k in (2 * i, 2 * i + 1):
            t.append((f"feat_net/sub_extractor/cfeat_conv_{k}/kernel", (3, 3, cin, c)))
            t.append((f"feat_net/sub_extractor/cfeat_conv_{k}/bias", (c,)))
            cin = c
    # flow predictors: pyramid_flow_estimator.py:64-83
    for p, name in enumerate(FLOW_PREDICTOR_NAMES):
        nf = FLOW_FILTERS[p]
        cin = 2 * feature_channels(p)
        for k in range(FLOW_CONVS[p]):
            t.append((f"predict_flow/{name}/conv_{k}/kernel", (3, 3, cin, nf)))
            t.append((f"predict_flow/{name}/conv_{k}/bias", (nf,)))
            cin = nf
        k = FLOW_CONVS[p]
        t.append((f"predict_flow/{name}/conv_{k}/kernel", (1, 1, nf, nf // 2)))
        t.append((f"predict_flow/{name}/conv_{k}/bias", (nf // 2,)))
        t.append((f"predict_flow/{name}/conv_{k + 1}/kernel", (1, 1, nf // 2, 2)))
        t.append((f"predict_flow/{name}/conv_{k + 1}/bias", (2,)))
    # fusion: fusion.py:70-101 (created fine-to-coarse; conv_0 = 2x2, conv_1/2 = 3x3)
    for i in range(FUSION_PYRAMID_LEVELS - 1):
        nf = fusion_filters(i)
        coarse_c = aligned_channels(i + 1) if i == FUSION_PYRAMID_LEVELS - 2 else fusion_filters(i + 1)
        t.append((f"fusion/level_{i}/conv_0/kernel", (2, 2, coarse_c, nf)))
        t.append((f"fusion/level_{i}/conv_0/bias", (nf,)))
        t.append((f"fusion/level_{i}/conv_1/kernel", (3, 3, aligned_channels(i) + nf, nf)))
        t.append((f"fusion/level_{i}/conv_1/bias", (nf,)))
        t.append((f"fusion/level_{i}/conv_2/kernel", (3, 3, nf, nf)))
        t.append((f"fusion/level_{i}/conv_2/bias", (nf,)))
    t.append(("fusion/output_conv/kernel", (1, 1, FILTERS, 3)))
    t.append(("fusion/output_conv/bias", (3,)))
    return t


def level_sizes(h: int, w: int) -> List[Tuple[int, int]]:
    """Sizes of the 7 image-pyramid levels (util.py:38-44, VALID pool floors)."""
    out = []
    for _ in range(PYRAMID_LEVELS):
        out.append((h, w))
        h, w = h // 2, w // 2
    return out


def conv_macs(h: int, w: int) -> Dict[str, int]:
    """Multiply-accumulates of every Conv2D call site for ONE network call on a
    (padded) h x w frame pair, counted as kh*kw*Cin*Cout per output pixel on the
    reference graph (no credit for algebraic shortcuts)."""
    sizes = level_sizes(h, w)
    fe = 0
    for i in range(PYRAMID_LEVELS):
        depth = min(PYRAMID_LEVELS - i, SUB_LEVELS)
        cin = 3
        for j in range(depth):
            hh, ww = sizes[i + j]
            c = FILTERS << j
            fe += hh * ww * 9 * (cin * c + c * c)
            cin = c
    fe *= 2  # two images
    flow = 0
    for l in range(PYRAMID_LEVELS):
        p = min(l, SPECIALIZED_LEVELS)
        nf = FLOW_FILTERS[p]
        hh, ww = sizes[l]
        cin = 2 * feature_channels(l)
        per_px = 9 * cin * nf + 9 * nf * nf * (FLOW_CONVS[p] - 1) + nf * (nf // 2) + (nf // 2) * 2
        flow += hh * ww * per_px
    flow *= 2  # two directions
    fus = 0
    for i in range(FUSION_PYRAMID_LEVELS - 1):
        nf = fusion_filters(i)
        hh, ww = sizes[i]
        coarse_c = aligned_channels(i + 1) if i == FUSION_PYRAMID_LEVELS - 2 else fusion_filters(i + 1)
        fus += hh * ww * (4 * coarse_c * nf + 9 * (aligned_channels(i) + nf) * nf + 9 * nf * nf)
    fus += sizes[0][0] * sizes[0][1] * FILTERS * 3
    return {"feature_extractor": fe, "flow": flow, "fusion": fus, "total": fe + flow + fus}


def padded_shape(h: int, w: int, align: int | None) -> Tuple[int, int, int, int]:
    """eval/interpolator.py:30-63 -> (padded_h, padded_w, offset_h, offset_w)."""
    if not align:
        return h, w, 0, 0
    ph = (align - h % align) if h % align else 0
    pw = (align - w % align) if w % align else 0
    return h + ph, w + pw, ph // 2, pw // 2


# ---------------------------------------------------------------------------------------------------------------------
# Overlapped tiling (engine option tile_overlap; no reference counterpart: eval/interpolator.py:66-126 cuts and pastes
# non-overlapping tiles).  One rule per axis, the same along H and W; csrc/film_engine.cu (stitch_axis) and
# csrc/film_kernels.cu (k_stitch_feather) restate it.
# ---------------------------------------------------------------------------------------------------------------------
def _axis_windows(length: int, blocks: int, overlap: int, name: str) -> Tuple[List[int], int, int]:
    """-> (window origins, window length q, effective overlap v) of one frame axis of `length` in `blocks` blocks."""
    p = length // blocks
    assert length == p * blocks, 'block_%s=%d should evenly divide %s=%d.' % (name, blocks, name, length)
    v = int(overlap) if blocks > 1 else 0          # a single block has no boundary to blend across
    assert v >= 0, 'tile overlap must not be negative'
    # keeps the ramps of consecutive boundaries apart: no pixel sees more than two windows per axis
    assert 2 * v <= p, 'tile_overlap=%d is more than half the tile %s=%d.' % (v, name, p)
    q = p + 2 * v
    # every window has the length q: border windows are shifted inward, not shortened, so a frame needs one plan
    return [min(max(k * p - v, 0), length - q) for k in range(blocks)], q, v


def tile_windows(h: int, w: int, block_shape: Sequence[int], overlap: int) -> Tuple[List[Tuple[int, int]], Tuple[int, int]]:
    """Windows of an h x w frame cut into block_shape = [bh, bw] tiles that reach `overlap` pixels past every interior
    tile boundary: (origins, (q_h, q_w)) with origins[t] = (y, x) of tile t (row-major) and one shape for all windows.
    overlap = 0 gives the reference's tiles (eval/interpolator.py:66-99)."""
    bh, bw = int(block_shape[0]), int(block_shape[1])
    oy, qh, _ = _axis_windows(h, bh, overlap, "height")
    ox, qw, _ = _axis_windows(w, bw, overlap, "width")
    return [(y, x) for y in oy for x in ox], (qh, qw)


def _axis_blend(length: int, blocks: int, overlap: int, name: str):
    """Per coordinate x of the axis: the two windows (ka, kb) it blends, the weight t of kb, and its coordinate inside
    each of them.  At the boundary c = k*p, for x in [c - v, c + v): t = (x + 0.5 - (c - v)) / 2v between windows k-1
    and k; elsewhere ka == kb == the window whose core contains x."""
    origins, _, v = _axis_windows(length, blocks, overlap, name)
    p = length // blocks
    x = np.arange(length)
    k = x // p
    ka, kb, t = k.copy(), k.copy(), np.zeros(length, np.float64)
    for c in range(p, length, p) if v else ():
        ramp = (x >= c - v) & (x < c + v)
        ka[ramp], kb[ramp] = c // p - 1, c // p
        t[ramp] = (x[ramp] + 0.5 - (c - v)) / (2 * v)
    o = np.asarray(origins)
    return ka, kb, t, x - o[ka], x - o[kb]


def stitch_overlapped(tiles: np.ndarray, h: int, w: int, block_shape: Sequence[int], overlap: int) -> np.ndarray:
    """Feathered stitch of the (bh*bw, q_h, q_w, C) window results of `tile_windows` into a (1, h, w, C) float64 frame:
    out = a + t * (b - a) across every interior boundary, along W first, then along H.  The numpy statement of what
    the engine's k_stitch_feather computes in float32."""
    bh, bw = int(block_shape[0]), int(block_shape[1])
    _, (qh, qw) = tile_windows(h, w, block_shape, overlap)
    t = np.asarray(tiles, np.float64)
    assert t.shape[:3] == (bh * bw, qh, qw), "expected %d windows of %dx%d" % (bh * bw, qh, qw)
    t = t.reshape(bh, bw, qh, qw, -1)
    xa, xb, tx, ia, ib = _axis_blend(w, bw, overlap, "width")
    ya, yb, ty, ja, jb = _axis_blend(h, bh, overlap, "height")
    a, b = t[:, xa, :, ia], t[:, xb, :, ib]                  # (w, bh, q_h, C): every tile row blended along W
    rows = a + tx[:, None, None, None] * (b - a)
    a, b = rows[:, ya, ja], rows[:, yb, jb]                  # (w, h, C)
    out = a + ty[None, :, None] * (b - a)
    return np.ascontiguousarray(out.transpose(1, 0, 2))[np.newaxis]
