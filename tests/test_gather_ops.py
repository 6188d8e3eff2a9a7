"""Every gather of a plan against a float64 restatement of its own inputs.

The gathers sit between the convs and decide where every pixel of the network reads from:
  flow_warp@L<l>    v_up[d] = resize_bilinear(2 * v[l+1][d]) (fp32), warped[d] = warp(feat[1-d], v_up[d])  (split)
  fusion_warp@L<l>  warped[k] = warp(feat[k], 0.5 * v[1-k])                                                 (split)
  fusion_side@L<l>  side tensor, 64 channels: 0-2 warp(img0, 0.5 * bwd), 3-5 warp(img1, 0.5 * fwd), 6-7 0.5 * bwd,
                    8-9 0.5 * fwd, 10-63 zero                                                               (split)
  pad_image         img/0, the input zero-padded at (off_y, off_x)                                          (fp32)
The engine runs with keep_debug = 1; the test walks the op table and reads each gather's inputs and outputs through
film_debug_read.  The restatement follows the reference's rules, not the engine's code:
  warp    util.py:48-82 with TFA 0.15 interpolate_bilinear: per axis q = y + f, floor = min(max(0, floor(q)), size - 2),
          alpha = clip(q - floor, 0, 1); top = tl + ax (tr - tl), bot likewise, out = top + ay (bot - top)
  resize  TF2 bilinear, half-pixel centres: src = (dst + 0.5) in/out - 0.5, lo = max(floor, 0), hi = min(ceil, in - 1),
          w = src - floor
The taps (corner indices and weights) are reproduced bit for bit in numpy float32 from the values the kernel read: the
kernel forms q = (float)y + f in fp32 (0.5 * f is exact), and at level 0 of a wide frame that rounding alone moves q by
up to 2^-13.  For the resize, src = (dst + 0.5f) * scale - 0.5f may be one FFMA or a multiply and an add; both
candidates are computed (the FFMA one as the exact float64 product-sum rounded once) and each element is compared with
the closer one.  Only the lerps run in float64.  A hi+lo gather reads hi + lo (exact in fp32), a hi-only one hi alone.

With M the largest |corner| of the four values an element interpolates, each element must satisfy
  |got - ref| <= 8 * 2^-24 * M + eps_out * |ref| + 2^-25
eps_out = 2^-(2p-1) when the destination's lo plane is written, 2^-p when only its hi plane is (p = 11 fp16, 8 bf16);
for the fp32 v_up eps_out = 2^-24 and there is no 2^-25 term.  The 8 is analysis: two fp32 lerps, each a subtraction
and a multiply-add, are worth about 6 * 2^-24 * M.  Bit for bit: side channels 6-9 are split(0.5 * flow), 10-63 are
zero in both planes, img/0 is the padded input.  Which gathers are hi-only comes from the plan (gather_hi_only), and a
warp destination's lo plane must be all zero exactly when hi-only is expected.  The side tensor always writes both
planes; a lo plane it failed to write shows in its bound, which is 2^-21 relative (its warped images can all be exactly
representable, as when every sample lands on the zero border of a padded frame).

Measured over every case of this file on an H100 80GB HBM3 (700 W), per kind: the largest err / bound, and the largest
err / (2^-24 M) left after the output-rounding allowance (the part the 8 has to cover):
  flow_warp, hi-only destination     0.999   0.77        fusion_warp, hi-only destination   0.999   0.40
  flow_warp, hi+lo destination       0.965   1.09        fusion_warp, hi+lo destination     0.980   1.22
  flow_warp v_up (fp32)              0.223   1.38        fusion_side channels 0-5           0.430   0.00
err / bound near 1 is the output rounding itself (round to nearest is within 2^-p of the value, the bound's eps_out
term); the arithmetic stays 5.8x under the 8.  Side channels 6-63 and img/0 are equal bit for bit.  At the odd sizes
the two fp32 forms of the resize position give different taps at up to 1984 pixels of a case, and every element
matches one of them.  The file takes about 2.5 minutes with -m gpu.

Memory: film_debug_read returns whole tensors, so at 704x1536 each level-0 plane arrives as one float32 array (about
277 MB at 64 channels); hi, lo and their exact fp32 sum are held together, about 1.7 GB of host memory at the peak.  The
float64 work is done only at the sampled pixels, in chunks of pixels, so no float64 array of a whole level-0 tensor is
ever formed; the reads themselves are not row-blocked.

The mutant self-check recomputes the reference under wrong rules (hi plane only, the other flow direction, unclamped
alpha, the same image's features, the resize without half-pixel centres, v_up without the factor 2) and requires the
bound to reject each of them on at least one element, in the 256x320 and the out-of-frame cases.
"""
import re

import numpy as np
import pytest

from frame_interpolation_b200 import spec
from test_conv_layers import (CAT2_CONVS, FUSION, LEVELS, ST_FLOW_L0, Plan, Report, op_stage, rule_of, run_plan,
                              sampled_pixels, split_w, all_pixels, _network_op_names)

K_GATHER = 8.0
ULP = 2.0 ** -24
FLOW_PREDICTORS = ("flow_predictor_0", "flow_predictor_1", "flow_predictor_2", "flow_predictor_shared")


# ---------------------------------------------------------------------------------------------------------------------
# taps and lerps
# ---------------------------------------------------------------------------------------------------------------------
def warp_axis(q, n, clamp=True):
    """TFA interpolate_bilinear along one axis of length n at positions q (float32: the kernel's single fp32 ops, or
    float64): floor = min(max(0, floor(q)), n - 2), alpha = clip(q - floor, 0, 1).  -> (floor index, alpha float64).
    clamp = False leaves alpha unclamped (a mutant: edge pixels extrapolate)."""
    t = q.dtype.type
    fl = np.minimum(np.maximum(np.floor(q), t(0)), t(n - 2))
    a = q - fl
    if clamp:
        a = np.clip(a, t(0), t(1))
    return fl.astype(np.int64), a.astype(np.float64)


def positions(y, x, f, dtype=np.float32):
    """q = y + f per axis; f[..., 0] is the x component.  In float32 q is one correctly rounded fp32 add, like the
    kernel's (float)y + f."""
    f = np.asarray(f, dtype)
    return np.asarray(y, dtype) + f[..., 1], np.asarray(x, dtype) + f[..., 0]


def bilerp(src, y0, x0, ay, ax):
    """float64 bilinear of src [H, W, C] at corners (y0, x0) .. (y0 + 1, x0 + 1) -> (ref [n, C], M [n, C])."""
    tl, tr = src[y0, x0].astype(np.float64), src[y0, x0 + 1].astype(np.float64)
    bl, br = src[y0 + 1, x0].astype(np.float64), src[y0 + 1, x0 + 1].astype(np.float64)
    ax, ay = ax[:, None], ay[:, None]
    top = tl + ax * (tr - tl)
    bot = bl + ax * (br - bl)
    M = np.maximum(np.maximum(np.abs(tl), np.abs(tr)), np.maximum(np.abs(bl), np.abs(br)))
    return top + ay * (bot - top), M


def warp_at(src, y, x, f, dtype=np.float32, clamp=True):
    """warp(src, f) at pixels (y, x): out = bilinear(src, y + f_y, x + f_x) with the TFA border rule.  src [H, W, C],
    f [n, 2] the flow the kernel read at those pixels.  Chunked over pixels.  -> (ref [n, C], M [n, C])."""
    H, W, C = src.shape
    n = len(y)
    ref, M = np.empty((n, C)), np.empty((n, C))
    step = max(1024, (1 << 22) // C)
    for s in range(0, n, step):
        qy, qx = positions(y[s:s + step], x[s:s + step], f[s:s + step], dtype)
        y0, ay = warp_axis(qy, H, clamp)
        x0, ax = warp_axis(qx, W, clamp)
        ref[s:s + step], M[s:s + step] = bilerp(src, y0, x0, ay, ax)
    return ref, M


def resize_axis(n_out, n_in, form):
    """TF2 bilinear resize taps along one axis -> (lo, hi, w float64).  form "f64": float64 arithmetic; "mul" / "fma":
    the kernel's fp32 src = (dst + 0.5f) * scale - 0.5f rounded after each op, or once (FFMA: the float64 product-sum
    is exact, (dst + 0.5) * scale >= 1/6 has at most 37 significant bits); "no_half": the mutant src = dst * in/out."""
    dst = np.arange(n_out)
    if form == "f64":
        src = (dst + 0.5) * (n_in / n_out) - 0.5
    elif form == "no_half":
        src = dst * (n_in / n_out)
    else:
        scale = np.float32(n_in) / np.float32(n_out)
        d5 = (dst + 0.5).astype(np.float32)
        if form == "mul":
            src = d5 * scale - np.float32(0.5)
        else:
            src = (d5.astype(np.float64) * np.float64(scale) - 0.5).astype(np.float32)
    fl = np.floor(src)
    lo = np.maximum(fl, 0).astype(np.int64)
    hi = np.minimum(np.ceil(src), n_in - 1).astype(np.int64)
    return lo, hi, (src - fl).astype(np.float64)


def resize_flow(v, H, W, form_y, form_x, factor=2.0):
    """resize_bilinear(factor * v, (H, W)) of a [Hc, Wc, 2] flow -> (ref [H, W, 2], M [H, W, 2])."""
    Hc, Wc = v.shape[:2]
    ylo, yhi, wy = resize_axis(H, Hc, form_y)
    xlo, xhi, wx = resize_axis(W, Wc, form_x)
    a = factor * np.asarray(v, np.float64)
    tl, tr = a[ylo][:, xlo], a[ylo][:, xhi]
    bl, br = a[yhi][:, xlo], a[yhi][:, xhi]
    wx, wy = wx[None, :, None], wy[:, None, None]
    top = tl + (tr - tl) * wx
    bot = bl + (br - bl) * wx
    M = np.maximum(np.maximum(np.abs(tl), np.abs(tr)), np.maximum(np.abs(bl), np.abs(br)))
    return top + (bot - top) * wy, M


# ---------------------------------------------------------------------------------------------------------------------
# rules: which op this file checks, and which gathers write hi planes only
# ---------------------------------------------------------------------------------------------------------------------
GATHER_RULES = [("flow_warp", re.compile(r"^flow_warp@L(\d)$")), ("fusion_warp", re.compile(r"^fusion_warp@L(\d)$")),
                ("fusion_side", re.compile(r"^fusion_side@L(\d)$")), ("pad_image", re.compile(r"^pad_image$"))]
# the producers that feed a conv, checked by test_conv_layers.py
CONV_TEST_PRODUCERS = re.compile(r"^(image_pool|fe_split32|fe_im2col|fe_pool|fusion_resize)@L\d$")


def is_conv(name, category):
    return category == 0 or (category == 2 and CAT2_CONVS.match(name) is not None)


def gather_rule(name):
    for kind, rx in GATHER_RULES:
        m = rx.match(name)
        if m:
            return kind, (int(m.group(1)) if m.groups() else None)
    return None


def claim(name, category):
    """Which test checks op `name`: "conv" (test_conv_layers.py), "producer" (the same file) or "gather" (this one)."""
    if is_conv(name, category):
        rule_of(name)
        return "conv"
    if CONV_TEST_PRODUCERS.match(name):
        return "producer"
    if gather_rule(name):
        return "gather"
    raise AssertionError(f"op {name!r} is neither a conv nor a known gather or producer: a new op needs a rule")


def gather_hi_only(P, kind, l):
    """flow_warp@L<l> feeds flow_conv0@L<l> only; fusion_warp@L<l> feeds fusion_conv1@L<l>, or fusion_up@L3 for the
    coarsest fusion level.  Hi-only iff that consumer runs single-pass and plane_skip is on."""
    if kind == "flow_warp":
        return P.hi_only(ST_FLOW_L0 + l)
    if kind == "fusion_warp":
        return P.hi_only(op_stage(f"fusion_up@L{FUSION - 2}" if l == FUSION - 1 else f"fusion_conv1@L{l}"))
    return False


# ---------------------------------------------------------------------------------------------------------------------
# the walk
# ---------------------------------------------------------------------------------------------------------------------
MUTANTS = ("hi_only_source", "other_direction", "unclamped_alpha", "same_image", "no_half_pixel", "no_factor_2")


class GatherReport(Report):
    def __init__(self):
        super().__init__()
        self.mutant = {}      # mutant -> largest err / bound it reached
        self.coverage = []    # record_coverage of every warp direction
        self.resize_forms = []  # (op, pixels where the two fp32 forms of the resize position give different taps)
        self.hi_only = {}       # gather -> whether the plan makes it hi-only

    def check_gather(self, op, what, got, ref, bound, M, pix):
        """The report row: max err/bound and the error left after the output-rounding allowance in units of 2^-24 M."""
        r = ratios(got, ref, bound)
        k = int(np.argmax(r))   # a NaN ratio (a NaN result) is the one argmax picks, and fails below
        worst = float(r.flat[k])
        acc = float(((np.abs(got - ref) - (bound - K_GATHER * ULP * M)) / (ULP * np.maximum(M, 1e-300))).max())
        where = (int(pix[0][k // r.shape[1]]), int(pix[1][k // r.shape[1]]), k % r.shape[1])
        self.rows.append((op, what, "", 0, worst, acc, where))
        if not np.isfinite(got).all() or not worst <= 1.0:
            self.fail.append(f"{op} [{what}]: max err/bound {worst:.3g} at (y, x, c) = {where}: got {got.flat[k]:.9g}, "
                             f"want {ref.flat[k]:.9g}, bound {bound.flat[k]:.3g}")

    def reject(self, name, got, ref, bound):
        r = np.nan_to_num(ratios(got, ref, bound), nan=np.inf)   # a NaN result differs from any mutant
        self.mutant[name] = max(self.mutant.get(name, 0.0), float(r.max()))


def ratios(got, ref, bound):
    """err / bound per element; an element equal to its reference is 0 even where the bound is 0 (an exact zero of the
    fp32 v_up, whose bound has no absolute term), so 0 / 0 never yields a NaN that would hide the other elements."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(got == ref, 0.0, np.abs(got - ref) / bound)


def rd(P, name, shape):
    """A debug tensor as float32 (16-bit planes widen exactly)."""
    return P.eng.debug_read(name).reshape(shape)


def split_bound(P, ref, M, hi_only):
    eps = 2.0 ** -P.p if hi_only else 2.0 ** -(2 * P.p - 1)
    return K_GATHER * ULP * M + eps * np.abs(ref) + 2.0 ** -25


def check_dest(P, rep, op, name, shape, hi_only):
    """The destination's planes; its lo plane must be all zero iff hi-only is expected.  -> fp32 value hi + lo."""
    hi, lo = rd(P, name + ".hi", shape), rd(P, name + ".lo", shape)
    if hi_only:
        rep.require(not lo.any(), f"{op}: lo plane of {name} written although its reader is single-pass")
    else:
        rep.require(lo.any(), f"{op}: lo plane of {name} never written although a three-pass conv reads it")
    return hi + lo


def record_coverage(rep, op, what, y, x, f, H, W):
    """Where the warp's sample positions land: fractions below 0 and above size - 1 per axis (y, x), strictly inside
    on both axes, exactly on size - 1; whether every alpha is 0 or 1; the largest |flow|."""
    qy, qx = positions(y, x, f)
    alphas = np.concatenate([warp_axis(qy, H)[1], warp_axis(qx, W)[1]])
    rep.coverage.append(dict(
        op=op, what=what, below=(float((qy < 0).mean()), float((qx < 0).mean())),
        above=(float((qy > H - 1).mean()), float((qx > W - 1).mean())),
        inside=float(((qy > 0) & (qy < H - 1) & (qx > 0) & (qx < W - 1)).mean()),
        on_last=int((qy == H - 1).sum() + (qx == W - 1).sum()), integer_alpha=bool(np.isin(alphas, (0.0, 1.0)).all()),
        vmax=float(np.abs(f).max())))


def check_warp(P, rep, op, what, src_name, H, W, C, f_at, pix, dest, hi_only, mutants):
    """One warp direction: src_name the feature planes it gathers, f_at(y, x) the flow it read, dest the fp32 result.
    mutants: {name: (source planes, flow, clamp alpha, hi plane only)}: wrong references the bound must reject."""
    y, x = pix
    def source(name, hi_plane_only):
        s = rd(P, name + ".hi", (H, W, C))
        return s if hi_plane_only else s + rd(P, name + ".lo", (H, W, C))
    src = source(src_name, hi_only)
    got = dest[y, x].astype(np.float64)
    f = f_at(y, x)
    ref, M = warp_at(src, y, x, f)
    rep.check_gather(op, what, got, ref, split_bound(P, ref, M, hi_only), M, pix)
    record_coverage(rep, op, what, y, x, f, H, W)
    for name, (m_src, m_f, clamp, m_hi_only) in mutants.items():
        s = src if (m_src, m_hi_only) == (src_name, hi_only) else source(m_src, m_hi_only)
        r, Mm = warp_at(s, y, x, m_f(y, x), clamp=clamp)
        rep.reject(name, got, r, split_bound(P, r, Mm, hi_only))


def check_plan_gathers(P, rep, x0, x1, pixels, mutants=False):
    names = [r["name"] for r in P.table]
    for r in P.table:   # coverage guard: every op of the plan is checked by this file or by test_conv_layers.py
        claim(r["name"], r["category"])
    H0, W0 = P.sizes[0]
    for op in names:
        kind, l = gather_rule(op) or (None, None)
        if kind is None:
            continue
        if kind == "pad_image":
            img = rd(P, "img/0", (2, H0, W0, 3))
            want = np.zeros_like(img)
            want[:, P.off_y:P.off_y + P.h, P.off_x:P.off_x + P.w] = np.stack([x0, x1]).reshape(2, P.h, P.w, 3)
            rep.require(np.array_equal(img, want), "pad_image: img/0 is not the input zero-padded at "
                                                   f"({P.off_y}, {P.off_x})")
            continue
        H, W = P.sizes[l]
        pix = pixels(H, W)
        hi_only = gather_hi_only(P, kind, l)
        rep.hi_only[op] = hi_only
        if kind == "flow_warp":
            Hc, Wc = P.sizes[l + 1]
            C = spec.feature_channels(l)
            vprev = [rd(P, f"flow_{dn}/{l + 1}", (Hc, Wc, 2)) for dn in ("fwd", "bwd")]
            vup = [rd(P, f"flow_vup{d}/{l}", (H, W, 2)) for d in range(2)]
            for d in range(2):
                got = vup[d].astype(np.float64)
                cands = [resize_flow(vprev[d], H, W, fy, fx) for fy in ("mul", "fma") for fx in ("mul", "fma")]
                errs = np.stack([np.abs(got - c[0]) for c in cands])
                pick = np.argmin(errs, axis=0)
                ref = np.choose(pick, [c[0] for c in cands])
                M = np.choose(pick, [c[1] for c in cands])
                rep.resize_forms.append((op, int((np.abs(cands[0][0] - cands[3][0]) > 0).any(-1).sum())))
                bound = K_GATHER * ULP * M + ULP * np.abs(ref)
                rep.check_gather(op, f"v_up{d}", got.reshape(-1, 2), ref.reshape(-1, 2), bound.reshape(-1, 2),
                                 M.reshape(-1, 2), all_pixels(1, H, W)[1:])
                if mutants:
                    for name, kw in (("no_half_pixel", dict(form_y="no_half", form_x="no_half")),
                                     ("no_factor_2", dict(form_y="fma", form_x="fma", factor=1.0))):
                        r, Mm = resize_flow(vprev[d], H, W, **kw)
                        rep.reject(name, got, r, K_GATHER * ULP * Mm + ULP * np.abs(r))
            for d in range(2):
                dest = check_dest(P, rep, op, f"flow_warped{d}/{l}", (H, W, C), hi_only)
                fd = lambda y, x, d=d: vup[d][y, x]
                fo = lambda y, x, d=d: vup[1 - d][y, x]
                src = f"feat{1 - d}/{l}"
                m = {}
                if mutants:
                    m = {"other_direction": (src, fo, True, hi_only), "unclamped_alpha": (src, fd, False, hi_only),
                         "same_image": (f"feat{d}/{l}", fd, True, hi_only)}
                    if not hi_only:
                        m["hi_only_source"] = (src, fd, True, True)
                check_warp(P, rep, op, f"warped{d}", src, H, W, C, fd, pix, dest, hi_only, m)
                del dest
        elif kind == "fusion_warp":
            C = spec.feature_channels(l)
            half = [0.5 * rd(P, f"flow_{dn}/{l}", (H, W, 2)) for dn in ("fwd", "bwd")]   # exact halving
            for k in range(2):
                dest = check_dest(P, rep, op, f"warped{k}/{l}", (H, W, C), hi_only)
                fk = lambda y, x, k=k: half[1 - k][y, x]
                fo = lambda y, x, k=k: half[k][y, x]
                src = f"feat{k}/{l}"
                m = {}
                if mutants:
                    m = {"other_direction": (src, fo, True, hi_only), "unclamped_alpha": (src, fk, False, hi_only)}
                    if not hi_only:
                        m["hi_only_source"] = (src, fk, True, True)
                check_warp(P, rep, op, f"warped{k}", src, H, W, C, fk, pix, dest, hi_only, m)
                del dest
        elif kind == "fusion_side":
            name = f"out:fusion_side@L{l}"
            hi, lo = rd(P, name + ".hi", (H, W, 64)), rd(P, name + ".lo", (H, W, 64))
            img = rd(P, f"img/{l}", (2, H, W, 3))
            half = [(0.5 * rd(P, f"flow_{dn}/{l}", (H, W, 2))).astype(np.float32) for dn in ("fwd", "bwd")]
            for c, f in ((6, half[1]), (8, half[0])):   # 6-7: 0.5 * bwd, 8-9: 0.5 * fwd
                wh, wl = split_w(f, P.fmt)
                rep.require(np.array_equal(hi[..., c:c + 2], wh) and np.array_equal(lo[..., c:c + 2], wl),
                            f"{op}: channels {c}-{c + 1} are not split(0.5 * {'bwd' if c == 6 else 'fwd'})")
            rep.require(not hi[..., 10:].any() and not lo[..., 10:].any(), f"{op}: channels 10-63 are not zero")
            val = hi + lo
            y, x = pix
            for k in range(2):   # channels 3k..3k+2: image k warped by 0.5 * v[1 - k]
                got = val[y, x, 3 * k:3 * k + 3].astype(np.float64)
                ref, M = warp_at(img[k], y, x, half[1 - k][y, x])
                rep.check_gather(op, f"img{k}", got, ref, split_bound(P, ref, M, False), M, pix)
                if mutants:
                    r, Mm = warp_at(img[k], y, x, half[k][y, x])
                    rep.reject("other_direction", got, r, split_bound(P, r, Mm, False))
                    r, Mm = warp_at(img[k], y, x, half[1 - k][y, x], clamp=False)
                    rep.reject("unclamped_alpha", got, r, split_bound(P, r, Mm, False))
    checked = {op for op in names if gather_rule(op)}
    rep.require({f"flow_warp@L{l}" for l in range(LEVELS - 1)} | {f"fusion_warp@L{l}" for l in range(FUSION)}
                | {f"fusion_side@L{l}" for l in range(FUSION)} | {"pad_image"} <= checked,
                f"gathers missing from the op table: {sorted(checked)}")
    return rep


def run_case(weights_path, h, w, align, opts, sampled=False, mutants=False, seed=7):
    eng, _, x0, x1 = run_plan(weights_path, h, w, align, opts, seed=seed)
    try:
        P = Plan(eng, h, w, align, opts)
        rng = np.random.default_rng(11)
        pixels = (lambda H, W: sampled_pixels(1, H, W, rng)[1:]) if sampled else (lambda H, W: all_pixels(1, H, W)[1:])
        rep = GatherReport()
        check_plan_gathers(P, rep, x0, x1, pixels, mutants)
        return rep, P
    finally:
        eng.close()


def assert_gathers(rep, label, mutants=False):
    by = {}
    for op, what, _, _, worst, acc, _ in rep.rows:
        kind = re.sub(r"@L\d$", "", op) + ("/v_up" if what.startswith("v_up") else "") + \
            ("" if what.startswith("v_up") or op.startswith("fusion_side") else
             "/hi" if rep.hi_only.get(op) else "/hi+lo")
        b = by.setdefault(kind, [0.0, 0.0])
        b[0], b[1] = float(np.maximum(b[0], worst)), float(np.maximum(b[1], acc))   # NaN propagates
    print(f"\n[{label}] gather: max err/bound, max err/(2^-24 M) after the output rounding")
    for k in sorted(by):
        print(f"  {k:28s} {by[k][0]:8.4f} {by[k][1]:8.3f}")
    print("  hi-only:", sorted(op for op, v in rep.hi_only.items() if v))
    print("  pixels where the two resize tap forms differ:", sum(n for _, n in rep.resize_forms))
    if mutants:
        print("  mutants, max err/bound:", ", ".join(f"{k} {v:.3g}" for k, v in sorted(rep.mutant.items())))
        for name in MUTANTS:
            rep.require(rep.mutant.get(name, 0.0) > 1.0, f"mutant {name} is not rejected by the bound "
                                                         f"({rep.mutant.get(name, 0.0):.3g})")
    assert not rep.fail, f"{label}: {len(rep.fail)} failures\n" + "\n".join(rep.fail[:30])


DEFAULT_HI_ONLY = {f"flow_warp@L{l}" for l in range(5)} | {"fusion_warp@L2", "fusion_warp@L3", "fusion_warp@L4"}
HI_LO = {"flow_warp@L5", "fusion_warp@L0", "fusion_warp@L1"}


# ---------------------------------------------------------------------------------------------------------------------
# GPU cases
# ---------------------------------------------------------------------------------------------------------------------
CASES = [  # (h, w, align, options, mutants); the mask cases say which gathers are hi-only
    (256, 320, 64, {}, True),                     # default mask: flow_warp@L0-4, fusion_warp@L2-4 hi-only
    (256, 320, 64, {"onepass_mask": 0}, False),   # every gather hi+lo
    (65, 129, None, {}, False),                   # odd levels: upsample scales like 16/33, a 2-pixel-high level 5
    (67, 95, None, {}, False),                    # 2x2 level 5, 1x1 level 6
    (67, 95, None, {"onepass_mask": 0}, False),
    (64, 64, 64, {}, False),                      # the flow upsampled from a 1x1 level, the warp clamp on 2x2
    (128, 192, 64, {"plane_skip": 0}, False),     # lo planes written behind single-pass consumers
    (128, 192, 64, {"conv_impl": 1}, False),      # validation path: every gather hi+lo
]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("h,w,align,opts,mutants", CASES,
                         ids=[f"{h}x{w}-" + (",".join(f"{k}={v}" for k, v in o.items()) or "default")
                              for h, w, _, o, _ in CASES])
def test_every_gather_matches_float64(synthetic_weights, h, w, align, opts, mutants):
    rep, P = run_case(synthetic_weights[0], h, w, align, opts, mutants=mutants)
    if not opts:
        assert {op for op, v in rep.hi_only.items() if v} == DEFAULT_HI_ONLY
        assert {op for op, v in rep.hi_only.items() if not v} >= HI_LO
    elif opts.get("onepass_mask") == 0 or "conv_impl" in opts or "plane_skip" in opts:
        assert not any(rep.hi_only.values())
    assert_gathers(rep, f"{h}x{w} {opts or 'default'}", mutants)


@pytest.mark.gpu
@pytest.mark.timeout(1200)
def test_gathers_at_704x1536_sampled(synthetic_weights):
    rep, _ = run_case(synthetic_weights[0], 704, 1536, 64, {}, sampled=True)
    assert_gathers(rep, "704x1536 sampled")


def _scaled_flow_weights(tmp_path, base, scales=None, biases=None, bias_xy=None, tag=""):
    """Synthetic weights for the flow predictors' conv_4 (flow_predictor_0, _1, _2, _shared): kernels scaled by
    scales[i] and biases set to biases[i] (flows that vary across pixels and leave the frame on every side), or
    conv_4 = 0 and bias = bias_xy (a constant residual: v_l = 2 v_{l+1} + b in closed form)."""
    from frame_interpolation_b200 import weights as W
    w = {k: np.array(v, copy=True) for k, v in base.items()}
    for i, p in enumerate(FLOW_PREDICTORS):
        k = f"predict_flow/{p}/conv_4/"
        if scales is not None:
            w[k + "kernel"] = (w[k + "kernel"] * np.float32(scales[i])).astype(np.float32)
            w[k + "bias"] = np.asarray(biases[i], np.float32)
        else:
            w[k + "kernel"][...] = 0.0
            w[k + "bias"][...] = np.asarray(bias_xy, np.float32)
    path = str(tmp_path / f"gather_{tag}.filmw")
    W.save(path, w)
    return path


SIDES = ("q_y < 0", "q_x < 0", "q_y > H - 1", "q_x > W - 1")
# conv_4 scale and bias per flow predictor (flow_predictor_0, _1, _2, _shared), searched on the CPU oracle for these
# frames (run_plan, seed 7): the bias cancels most of the mean residual, which otherwise pushes the pixels of a level
# off the same sides, and the scale sets the spread.  Every direction of every warped level must have at least 1 % of
# its pixels past each of the four sides and at least 10 % strictly inside, except where `exceptions` gives a smaller
# minimum for one side of one op (see test_gathers_with_flows_that_leave_the_frame).
OUT_OF_FRAME = [
    (128, 192, 64, (20.208, 17.561, 23.93, 29.396), ((0.229, 1.69), (3.339, 6.451), (0.868, 1.946), (-0.235, -0.891)),
     {"flow_warp@L5": {"q_y > H - 1": 0.0}}),
    (100, 150, None, (12.462, 13.928, 11.966, 87.834), ((2.191, 2.19), (2.157, 2.936), (-0.007, 3.326), (0.312, -0.663)),
     {"flow_warp@L5": {"q_x < 0": 0.0, "q_y > H - 1": 0.0}, "fusion_warp@L0": {"q_x < 0": 0.002},
      "fusion_warp@L1": {"q_x < 0": 0.002}, "fusion_warp@L2": {"q_x < 0": 0.002}}),
]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("h,w,align,scales,biases,exceptions", OUT_OF_FRAME, ids=[f"{h}x{w}" for h, w, *_ in OUT_OF_FRAME])
def test_gathers_with_flows_that_leave_the_frame(tmp_path, synthetic_weights, h, w, align, scales, biases, exceptions):
    """Where the sample positions land, per warp direction and level (measured on the H100, fractions of pixels):
    128x192 meets every figure, every side at least 2.6 %, except the bottom side of flow_warp@L5.  That level is 4x6
    pixels, and its v_up is the bilinear upsample of the 2x3 level 6, whose y flow does not grow toward the bottom row
    for any predictor scale and bias the search tried.  100x150 (any_size) also misses two sides of its 3x4 flow_warp@L5
    (left, bottom).  The left side of fusion_warp@L0-2 is reached by only 0.4 % to 1.4 % of the pixels there, so 0.2 %
    is required: the search found no setting of the four predictors that brings the left side of the half flows over
    1 % without losing another side.  The out-of-frame behaviour of every side is still exercised at full strength:
    the 128x192 case reaches each side with at least 2.6 % of the pixels at every level below 5."""
    path = _scaled_flow_weights(tmp_path, synthetic_weights[1], scales=scales, biases=biases, tag=f"oof{h}")
    rep, P = run_case(path, h, w, align, {}, mutants=True)
    lines = []
    for c in rep.coverage:   # the flow_warp and fusion_warp directions of every warped level
        fracs = c["below"] + c["above"]
        lines.append(f"  {c['op']:15s} {c['what']:8s} " + " ".join(f"{s} {f:.3f}" for s, f in zip(SIDES, fracs)) +
                     f"  inside {c['inside']:.3f}  max |v| {c['vmax']:.1f}")
        for side, frac in zip(SIDES, fracs):
            want = exceptions.get(c["op"], {}).get(side, 0.01)
            rep.require(frac >= want, f"{c['op']}/{c['what']}: only {frac:.4f} of the pixels have {side}")
        rep.require(c["inside"] >= 0.10, f"{c['op']}/{c['what']}: only {c['inside']:.4f} of the pixels land inside")
        rep.require(c["vmax"] <= 4096, f"{c['op']}/{c['what']}: |v| up to {c['vmax']:.0f}")
    print("\n" + "\n".join(lines))
    warped = {(c["op"], c["what"]) for c in rep.coverage}
    rep.require(len(warped) == 2 * (LEVELS - 1 + FUSION), f"coverage of {len(warped)} warp directions")
    assert_gathers(rep, f"{h}x{w} flows leaving the frame", mutants=True)


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("bias_xy", [(3.0, -2.0), (2.0, 1.0)], ids=["3,-2", "2,1"])
def test_gathers_with_integer_landings(tmp_path, synthetic_weights, bias_xy):
    """conv_4 = 0, bias = b: every flow is an integer vector, so every flow_warp alpha is exactly 0, or 1 where the
    floor clamps to size - 2.  b = (2, 1) lands pixels exactly on q = size - 1 (level 5: q_x = x + 4 = 5 at x = 1).
    120x180 pads to 128x192 at offsets (4, 6), which pad_image has to honour."""
    path = _scaled_flow_weights(tmp_path, synthetic_weights[1], bias_xy=bias_xy, tag="b%g_%g" % bias_xy)
    rep, P = run_case(path, 120, 180, 64, {})
    assert (P.off_y, P.off_x) == (4, 6)
    flow = [c for c in rep.coverage if c["op"].startswith("flow_warp")]
    assert len(flow) == 2 * (LEVELS - 1) and all(c["integer_alpha"] for c in flow)
    assert any(max(c["above"]) > 0 for c in flow)            # clamped floors: alpha = 1
    if bias_xy == (2.0, 1.0):
        assert sum(c["on_last"] for c in flow) > 0            # q exactly size - 1
    assert_gathers(rep, f"integer landings {bias_xy}")


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the restatements against the oracle, the fp32 tap emulation, the rule table
# ---------------------------------------------------------------------------------------------------------------------
def test_restatements_match_the_oracle_in_float64():
    """warp_at and resize_flow in float64 against oracle.film_oracle.warp / resize_bilinear in float64 torch: flows
    several frames wide, integer landings (on 0, on size - 1, past it) and odd sizes."""
    import torch
    from oracle import film_oracle as O
    rng = np.random.default_rng(5)
    for H, W in ((2, 2), (3, 5), (9, 11), (16, 33)):
        src = rng.standard_normal((H, W, 4))
        y, x = all_pixels(1, H, W)[1:]
        flows = [rng.standard_normal((H, W, 2)) * 3 * max(H, W),                     # several frames wide
                 rng.integers(-2 * max(H, W), 2 * max(H, W), (H, W, 2)).astype(np.float64),
                 np.stack([W - 1 - x, H - 1 - y], -1).reshape(H, W, 2).astype(np.float64),   # exactly on size - 1
                 rng.uniform(-1.5, 1.5, (H, W, 2))]
        for f in flows:
            ref, M = warp_at(src, y, x, f.reshape(-1, 2), dtype=np.float64)
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).permute(2, 0, 1)[None]
            want = O.warp(t(src), t(f))[0].permute(1, 2, 0).reshape(-1, 4).numpy()
            assert np.abs(ref - want).max() <= 1e-12
            assert (M >= np.abs(ref) - 1e-12).all()
        for Hc, Wc in ((1, 1), (1, 2), (H // 2 or 1, W // 2 or 1), ((H + 1) // 2, (W + 1) // 2)):
            v = rng.standard_normal((Hc, Wc, 2)) * 50
            ref, _ = resize_flow(v, H, W, "f64", "f64")
            want = O.resize_bilinear(torch.from_numpy(2 * v).permute(2, 0, 1)[None], (H, W))[0].permute(1, 2, 0).numpy()
            assert np.abs(ref - want).max() <= 1e-12


def test_float32_taps_reproduce_the_kernel_rounding():
    """q = float32(y + f): hand-picked positions where the fp32 sum rounds onto an integer (float64 would take the
    floor below with alpha ~ 1), onto size - 1 (floor clamps to size - 2, alpha = 1), and a level-0 position whose
    fractional part moves by the fp32 rounding."""
    f32 = np.float32
    cases = [  # y, f, n -> floor, alpha
        (1000, f32(-1e-5), 1920, 1000, 0.0),              # 999.99999 rounds to 1000
        (5, f32(-2.0 ** -25), 64, 5, 0.0),                # 5 - 2^-25 rounds to 5
        (62, f32(1 - 2.0 ** -24), 64, 62, 1.0),           # 62.99999994 rounds to 63 = size - 1: floor 62, alpha 1
        (0, f32(-2.0 ** -30), 64, 0, 0.0),                # q < 0 by a hair: floor clamps to 0, alpha clips to 0
        (3, f32(-3.5), 64, 0, 0.0),                       # q = -0.5
        (1, f32(1e6), 8, 6, 1.0),                         # far past the end
    ]
    for y, f, n, fl, a in cases:
        i, al = warp_axis(f32(y) + f, n)
        assert (int(i), float(al)) == (fl, a), (y, f, n, int(i), float(al))
    assert warp_axis(np.float64(1000) + np.float64(f32(-1e-5)), 1920)[0] == 999   # float64 takes the other floor
    q = f32(1919) + f32(0.3)
    i, al = warp_axis(q, 1920)
    assert i == 1918 and al == 1.0                        # on the last column's clamp
    q = f32(1500) + f32(0.3)
    i, al = warp_axis(q, 1920)
    assert i == 1500 and al == float(f32(q - f32(1500))) and abs(al - 0.3) > 1e-6
    # fp32 resize positions: at 2x upsampling both the FFMA form and the rounded pair are exact
    for n_in in (1, 2, 5, 24, 960):
        ref = resize_axis(2 * n_in, n_in, "f64")
        for form in ("mul", "fma"):
            got = resize_axis(2 * n_in, n_in, form)
            assert all(np.array_equal(a, b) for a, b in zip(ref, got))
    # odd sizes: the fp32 scale 32/65 carries its own rounding, so w follows the float64 rule to dst * 2^-25
    lo_m, hi_m, w_m = resize_axis(65, 32, "mul")
    lo_f, hi_f, w_f = resize_axis(65, 32, "fma")
    lo_d, hi_d, w_d = resize_axis(65, 32, "f64")
    assert np.abs(w_m - w_d).max() < 65 * 2.0 ** -24 and np.abs(w_f - w_d).max() < 65 * 2.0 ** -24
    assert np.array_equal(lo_m, lo_d) and np.array_equal(hi_f, hi_d)
    assert (w_m != w_f).any()   # and the two fp32 forms are not the same rule


def _network_gather_names():
    return ({"pad_image"} | {f"flow_warp@L{l}" for l in range(LEVELS - 1)} | {f"fusion_warp@L{l}" for l in range(FUSION)}
            | {f"fusion_side@L{l}" for l in range(FUSION)})


def _network_producer_names():
    return ({f"image_pool@L{l}" for l in range(LEVELS - 1)} | {f"fe_split32@L{l}" for l in range(LEVELS)}
            | {f"fe_im2col@L{l}" for l in range(LEVELS)} | {f"fe_pool@L{l}" for l in range(LEVELS - 1)}
            | {f"fusion_resize@L{l}" for l in range(FUSION - 1)})


def test_rule_table_claims_every_op_and_refuses_unknown_names():
    for name in _network_op_names():
        assert claim(name, 0) == "conv"
    for name in ("fe_conv0@L0", "flow_head@L3", "rgb_head"):   # the fp32 convs of the validation path
        assert claim(name, 2) == "conv"
    for name in _network_producer_names():
        assert claim(name, 2) == "producer"
    for name in _network_gather_names():
        assert claim(name, 1 if "warp@" in name else 2) == "gather"
    for bad in ("pad_images", "flow_warp@L", "fusion_warp2@L0", "new_gather@L0", "stitch_feather", "flow_vup@L1"):
        with pytest.raises(AssertionError, match="needs a rule"):
            claim(bad, 2)


def test_hi_only_rule_of_the_default_and_other_plans():
    """The plan's wiring, on a stand-in for an engine plan: the default mask makes flow_warp@L0-4 and fusion_warp@L2-4
    hi-only; no mask, plane_skip = 0 or the validation path make every gather hi+lo."""
    from test_conv_layers import ST_FUS

    def plan(mask, plane_skip=1, impl=0):
        P = Plan.__new__(Plan)
        P.mask, P.plane_skip, P.impl = mask, plane_skip, impl
        return P

    default = (0b1110 << 0) | (0x1F << ST_FLOW_L0) | (0x3F << (ST_FUS + 6))
    gathers = [(k, l) for k in ("flow_warp", "fusion_warp") for l in range(LEVELS - 1 if k == "flow_warp" else FUSION)]
    got = {f"{k}@L{l}" for k, l in gathers if gather_hi_only(plan(default), k, l)}
    assert got == DEFAULT_HI_ONLY
    assert not ({f"{k}@L{l}" for k, l in gathers} - got) ^ HI_LO
    for P in (plan(0), plan(default, plane_skip=0), plan(default, impl=1)):
        assert not any(gather_hi_only(P, k, l) for k, l in gathers)
    assert not gather_hi_only(plan(-1), "fusion_side", 0)


def test_report_fails_on_errors_next_to_zero_bounds_and_on_nan():
    """An exact element with a zero bound (v_up where all four corners are 0) must not hide a wrong neighbour, and a
    NaN result must fail."""
    pix = (np.zeros(3, np.int64), np.arange(3))
    ref = np.array([[0.0], [1.0], [2.0]])
    bound = np.array([[0.0], [1e-6], [1e-6]])
    for got, bad in (([0.0, 1.0, 2.0], False), ([0.0, 1.0, 2.1], True), ([0.0, np.nan, 2.0], True),
                     ([1e-30, 1.0, 2.0], True)):
        rep = GatherReport()
        rep.check_gather("flow_warp@L0", "v_up0", np.array(got)[:, None], ref, bound, np.abs(ref), pix)
        assert bool(rep.fail) == bad, (got, rep.fail)
    rep = GatherReport()
    rep.reject("no_factor_2", ref, ref, bound)
    assert rep.mutant["no_factor_2"] == 0.0
