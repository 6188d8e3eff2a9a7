"""A second, independently written restatement of the reference graph -- pure numpy, explicit tap sums and index arithmetic,
no torch ops -- checked against `oracle/film_oracle.py` on a 64x64 frame pair. The two share nothing but the weight table:
if either mis-states a TF / TFA rule of the reference graph (SAME padding asymmetry of the 2x2 conv, VALID pooling, half-pixel
bilinear resize of `2 * v`, NEAREST resize, TFA's clamp-then-lerp warp with the (dy, dx) flip, concat orders, predictor
indexing, flow scaling by 0.5), the outputs diverge. This does not pin the oracle to TensorFlow (nothing offline can); it
removes "one author's reading of torch semantics" as a single point of failure."""
import numpy as np

from frame_interpolation_b200 import spec, synthetic, weights


def conv_same(x, k, b, act):
    """x (H, W, Cin), k (kh, kw, Cin, Cout) HWIO, cross-correlation, TF SAME padding: extra pixel AFTER for even kernels."""
    kh, kw = k.shape[:2]
    pt, pl = (kh - 1) // 2, (kw - 1) // 2
    pb, pr = kh - 1 - pt, kw - 1 - pl
    xp = np.pad(x, ((pt, pb), (pl, pr), (0, 0)))
    h, w = x.shape[:2]
    y = np.zeros((h, w, k.shape[3]), np.float64) + b
    for i in range(kh):
        for j in range(kw):
            y += xp[i:i + h, j:j + w, :] @ k[i, j]
    return np.where(y >= 0, y, 0.2 * y) if act else y


def pool(x):
    h, w = x.shape[0] // 2 * 2, x.shape[1] // 2 * 2
    return 0.25 * (x[0:h:2, 0:w:2] + x[0:h:2, 1:w:2] + x[1:h:2, 0:w:2] + x[1:h:2, 1:w:2])


def resize_bilinear(x, oh, ow):
    ih, iw = x.shape[:2]
    out = np.zeros((oh, ow, x.shape[2]))
    for y in range(oh):
        sy = (y + 0.5) * ih / oh - 0.5
        y0 = int(np.floor(sy)); wy = sy - y0
        ya, yb = max(y0, 0), min(int(np.ceil(sy)), ih - 1)
        for xx in range(ow):
            sx = (xx + 0.5) * iw / ow - 0.5
            x0 = int(np.floor(sx)); wx = sx - x0
            xa, xb = max(x0, 0), min(int(np.ceil(sx)), iw - 1)
            top = x[ya, xa] + (x[ya, xb] - x[ya, xa]) * wx
            bot = x[yb, xa] + (x[yb, xb] - x[yb, xa]) * wx
            out[y, xx] = top + (bot - top) * wy
    return out


def resize_nearest(x, oh, ow):
    ih, iw = x.shape[:2]
    ys = np.minimum(np.floor((np.arange(oh) + 0.5) * ih / oh).astype(int), ih - 1)
    xs = np.minimum(np.floor((np.arange(ow) + 0.5) * iw / ow).astype(int), iw - 1)
    return x[ys][:, xs]


def warp(img, flow):
    """util.warp: sample img at (y + flow[..., 1], x + flow[..., 0]) with TFA's rule per axis:
    floor = min(max(0, floor(q)), size - 2); alpha = clip(q - floor, 0, 1)."""
    h, w = img.shape[:2]
    out = np.zeros_like(img)
    for y in range(h):
        for x in range(w):
            qy, qx = y + flow[y, x, 1], x + flow[y, x, 0]
            fy = min(max(0, int(np.floor(qy))), h - 2)
            fx = min(max(0, int(np.floor(qx))), w - 2)
            ay, ax = min(max(qy - fy, 0.0), 1.0), min(max(qx - fx, 0.0), 1.0)
            top = ax * (img[fy, fx + 1] - img[fy, fx]) + img[fy, fx]
            bot = ax * (img[fy + 1, fx + 1] - img[fy + 1, fx]) + img[fy + 1, fx]
            out[y, x] = ay * (bot - top) + top
    return out


def film(w, x0, x1):
    g = lambda n: (w[n + "/kernel"].astype(np.float64), w[n + "/bias"].astype(np.float64))
    L, F = spec.PYRAMID_LEVELS, spec.FUSION_PYRAMID_LEVELS

    def pyramid(im):
        p = [im]
        for _ in range(L - 1):
            p.append(pool(p[-1]))
        return p

    def subtree(im, n):
        out, head = [], im
        for i in range(n):
            head = conv_same(head, *g(f"feat_net/sub_extractor/cfeat_conv_{2 * i}"), True)
            head = conv_same(head, *g(f"feat_net/sub_extractor/cfeat_conv_{2 * i + 1}"), True)
            out.append(head)
            if i < n - 1:
                head = pool(head)
        return out

    def features(pyr):
        subs = [subtree(pyr[i], min(L - i, spec.SUB_LEVELS)) for i in range(L)]
        return [np.concatenate([subs[i - j][j] for j in range(min(i, spec.SUB_LEVELS - 1) + 1)], axis=-1) for i in range(L)]

    def predict(level, a, b):
        name = spec.FLOW_PREDICTOR_NAMES[min(level, spec.SPECIALIZED_LEVELS)]
        net = np.concatenate([a, b], axis=-1)
        for k in range(3):
            net = conv_same(net, *g(f"predict_flow/{name}/conv_{k}"), True)
        net = conv_same(net, *g(f"predict_flow/{name}/conv_3"), True)
        return conv_same(net, *g(f"predict_flow/{name}/conv_4"), False)

    def flows(fa, fb):
        v = predict(L - 1, fa[-1], fb[-1])
        out = [v]
        for i in range(L - 2, -1, -1):
            v = resize_bilinear(2.0 * v, *fa[i].shape[:2])
            v = predict(i, fa[i], warp(fb[i], v)) + v
            out.append(v)
        return out[::-1]                                   # absolute flows, fine -> coarse (== flow_pyramid_synthesis)

    p0, p1 = pyramid(x0), pyramid(x1)
    f0, f1 = features(p0), features(p1)
    fwd, bwd = flows(f0, f1), flows(f1, f0)
    aligned = []
    for l in range(F):
        t0 = np.concatenate([p0[l], f0[l]], axis=-1)
        t1 = np.concatenate([p1[l], f1[l]], axis=-1)
        aligned.append(np.concatenate([warp(t0, 0.5 * bwd[l]), warp(t1, 0.5 * fwd[l]), 0.5 * bwd[l], 0.5 * fwd[l]], axis=-1))
    net = aligned[-1]
    for i in range(F - 2, -1, -1):
        net = resize_nearest(net, *aligned[i].shape[:2])
        net = conv_same(net, *g(f"fusion/level_{i}/conv_0"), False)
        net = np.concatenate([aligned[i], net], axis=-1)
        net = conv_same(net, *g(f"fusion/level_{i}/conv_1"), True)
        net = conv_same(net, *g(f"fusion/level_{i}/conv_2"), True)
    return conv_same(net, *g("fusion/output_conv"), False)


def test_independent_numpy_restatement_agrees_with_the_oracle():
    import torch
    from oracle.film_oracle import OracleInterpolator
    w = weights.synthetic_weights()
    x0, x1 = synthetic.frame_pair(64, 64, seed=4, n_waves=6)
    ref = OracleInterpolator(w, align=64, dtype=torch.float64).interpolate(x0, x1, np.full((1,), 0.5, np.float32))[0]
    got = film(w, x0[0].astype(np.float64), x1[0].astype(np.float64))
    assert got.shape == ref.shape == (64, 64, 3)
    assert np.abs(got - ref).max() < 1e-9, np.abs(got - ref).max()
