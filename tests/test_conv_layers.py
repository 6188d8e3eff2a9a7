"""Every conv call site of a plan against a float64 conv of its own inputs.

The engine runs with keep_debug = 1, which keeps every intermediate readable and changes nothing else.  The test walks
the op table; for each conv it reads the 16-bit planes the kernel consumed ("<tensor>.hi" / ".lo"), recomputes the
layer in float64 from exactly the operands the kernel multiplies, and compares with the layer's own output:

  weights       w_hi = rn(w), w_lo = rn(w - w_hi) from the HWIO kernels (rn: the split format of film_version()); the
                taps of a decoder parity class carry the fp32 sum of the 2x2 weights that land on one coarse pixel
  three-pass    a_hi.w_hi + a_hi.w_lo + a_lo.w_hi         single-pass   a_hi.w_hi
  fp32 kernels  cfeat_conv_0 on the FMA pipes and the conv_impl = 1 validation kernels: the fp32 values they read
  then bias, LeakyReLU, and the 2x2 mean of the activated values for a fused pool.

What is left is fp32 accumulation order and the rounding of the result into its planes.  With S = |b| + sum |a||w|
(one more float64 conv, of absolute values), each output element must satisfy

  |got - ref| <= TAU * 2^-24 * S + eps_out * |ref| + 2^-25

eps_out = 2^-(2p-1) when the destination's lo plane is written, 2^-p when only its hi plane is (every reader is a
single-pass conv and plane_skip is on), 2^-24 for fp32 destinations; p = 11 for fp16 planes, 8 for bf16.  The test
derives which case applies from the wiring and the one-pass mask, and checks that a lo plane is all zeros exactly when
it expects hi-only.  The fused heads (flow conv_3 / conv_4, the RGB 1x1) propagate the 3x3 conv's bound through the
fp32 1x1 layers with their absolute weights.

The error term scales with sqrt(K), K = products per output element (taps x input channels): S is sqrt(K) * sum |a||w|.
A bound linear in sum |a||w| alone did not fit.  Calibrated on an H100 80GB HBM3 (700 W) with TAU = 32 and no sqrt(K),
err / (2^-24 sum |a||w|) grew from about 8 at K = 576 (fe_conv1) and 25 at K = 2304 (fe_conv5) to 41 at K = 17280
(flow_conv0@L3..6) and 47 at K = 19674 (fusion_conv1@L3): wgmma's fp32 accumulation, not a single rounding per add.
Over every case of this file, the largest err / (2^-24 S) with the sqrt(K) scale, after the output-rounding allowance:
  tensor-core convs   0.90 (fe_conv0 on the 3x3 kernel, K = 27), otherwise <= 0.71 (fe_conv4 0.71, fe_conv1 on
                      pixels on N 0.56, fe_conv5 0.56, fusion_conv1 on pixels on N 0.54, fusion_up 0.41, flow_conv0 0.32)
  validation kernels  <= 0.30 (conv_impl = 1);  cfeat_conv_0 on the FMA pipes <= 0.31
TAU = 4 is 4.4x above the largest.

The per-element bound cannot tell a three-pass layer from one that silently ran single-pass once K is large: there
wgmma's own accumulation error comes within 4x of the single-pass product error (measured 0.5x to 3.9x of the bound on
the K >= 1152 layers and the fused heads).  So every tensor-core layer that runs three-pass also has to pass a per-layer
statistic, the share of the single-pass deviation in its output, c = <got - ref3, ref1 - ref3> / |ref1 - ref3|^2 with
ref1 the single-pass reference (Report.single_pass_fraction): |c| <= FRAC_MAX = 0.2.  A layer that ran single-pass has
c ~ 1, one that lost the low-order terms of some taps or channels has about their share.  Measured on the H100: at most
0.006 on three-pass layers; 0.998 to 1.003 on every layer of the single-pass self-check, which requires 4 x FRAC_MAX
on each of them.

Cases and cost: three small sizes with full tensors, 14 option cases at 64x128, the CTA-pair layers at 256x320, 704x1536
on sampled pixels, the self-check and the bitwise invariants.  1088x1920 runs only when its keep_debug arena stays
under a third of free device memory; on an H100 80GB it does not, and the case skips.  The file takes about 25 minutes
with -m gpu on an H100 host with 8 CPU cores, nearly all of it float64 reference work: about 95 s per 256x320 plan and
about 5 minutes per sampled 704x1536 plan.
"""
import re

import numpy as np
import pytest

from frame_interpolation_b200 import spec, synthetic

TAU = 4.0
FRAC_MAX = 0.2   # largest share of the single-pass deviation a three-pass layer may carry (Report.single_pass_fraction)
DT = np.full((1,), 0.5, np.float32)
LEVELS = spec.PYRAMID_LEVELS
FUSION = spec.FUSION_PYRAMID_LEVELS
SLICE_OFF = (0, 64, 192, 448)
FE = "feat_net/sub_extractor/cfeat_conv_"

# stages of the precision plan (film_engine.cu `enum Stage`; checked against film_stage_name below)
ST_FLOW_L0 = 7
ST_FUS = ST_FLOW_L0 + LEVELS
ST_COUNT = ST_FUS + 3 * (FUSION - 1)


def fe_stage(image_level, k):
    if image_level == 0:
        return k // 2
    return 4 if image_level == 1 else 5 if image_level == 2 else 6


def stage_names():
    fe = ["fe_i0_k01", "fe_i0_k23", "fe_i0_k45", "fe_i0_k67", "fe_i1", "fe_i2", "fe_i3p"]
    return fe + [f"flow_L{l}" for l in range(LEVELS)] + [f"fus{i}_c{c}" for i in range(FUSION - 1) for c in range(3)]


# ---------------------------------------------------------------------------------------------------------------------
# split format
# ---------------------------------------------------------------------------------------------------------------------
def rn(x, fmt):
    """Round float32 values to the 16-bit split format (round to nearest even), returned as float64."""
    x = np.asarray(x, np.float32)
    if fmt == "fp16":
        return x.astype(np.float16).astype(np.float64)
    u = x.view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32).astype(np.float64)


def split_w(w, fmt):
    """pack_conv: hi = rn(w), lo = rn(w - hi) with the difference taken in fp32."""
    w = np.asarray(w, np.float32)
    hi = rn(w, fmt)
    lo = rn((w - hi.astype(np.float32)).astype(np.float32), fmt)
    return hi, lo


def fmt_bits(fmt):
    return 11 if fmt == "fp16" else 8


# ---------------------------------------------------------------------------------------------------------------------
# float64 reference of one conv at a set of output pixels
# ---------------------------------------------------------------------------------------------------------------------
class Src:
    """Activation operands [B, H, W, C] in the reference channel order: the two planes, or fp32 values (lo = 0)."""

    def __init__(self, hi, lo=None):
        self.hi = np.asarray(hi, np.float64)
        self.lo = np.zeros_like(self.hi) if lo is None else np.asarray(lo, np.float64)


def taps_3x3(kernel):
    return [(ky - 1, kx - 1, kernel[ky, kx]) for kx in range(3) for ky in range(3)]


def taps_parity(kernel, py, px):
    """fusion conv_0 (2x2 SAME after a 2x NN upsample) per output parity class on the coarse grid: the fp32 sum of the
    fine taps that hit one coarse pixel, in the engine's order (taps_up2x2 in film_engine.cu)."""
    taps = []
    for dy in range(py + 1):
        for dx in range(px + 1):
            acc = np.zeros(kernel.shape[2:], np.float32)
            for fy in range(2):
                for fx in range(2):
                    if (py + fy) // 2 == dy and (px + fx) // 2 == dx:
                        acc = (acc + kernel[fy, fx]).astype(np.float32)
            taps.append((dy, dx, acc))
    return taps


def conv_at(src, taps, b, y, x, mode, fmt):
    """sum over taps of A[b, y + dy, x + dx] . W_tap (zero outside the grid) at the given input-grid pixels.
    mode "three": a_hi.(w_hi + w_lo) + a_lo.w_hi;  "one": a_hi.w_hi  (split products of the planes);
    "simt": the validation kernel, (a_hi + a_lo).(w_hi + w_lo);
    "fp32": the fp32 kernels that read fp32 values and the unsplit fp32 weights.
    Returns (ref, S, ref1) without bias; S = sqrt(K) * sum |a||w| over the K products of an output element; ref1 is
    the single-pass product a_hi.w_hi when mode is "three" (None otherwise)."""
    n = len(b)
    cin, cout = taps[0][2].shape[-2:]
    ref, S = np.zeros((n, cout)), np.zeros((n, cout))
    ref1 = np.zeros((n, cout)) if mode == "three" else None
    H, W = src.hi.shape[1:3]
    wh, wl = split_w(np.concatenate([w for _, _, w in taps]), fmt)   # im2col order: tap-major, then channel
    if mode == "fp32":
        wh, wl = np.concatenate([w for _, _, w in taps]).astype(np.float64), 0 * wh
    elif mode == "simt":
        wh, wl = wh + wl, 0 * wh
    w_abs = np.abs(wh + wl)
    chunk = max(256, (1 << 23) // (len(taps) * cin))
    for s in range(0, n, chunk):
        bb, yy0, xx0 = b[s:s + chunk], y[s:s + chunk], x[s:s + chunk]
        ah, al = np.empty((len(bb), len(taps) * cin)), np.empty((len(bb), len(taps) * cin))
        for t, (dy, dx, _) in enumerate(taps):
            yy, xx = yy0 + dy, xx0 + dx
            ok = ((yy >= 0) & (yy < H) & (xx >= 0) & (xx < W))[:, None]
            yc, xc = np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)
            ah[:, t * cin:(t + 1) * cin] = src.hi[bb, yc, xc] * ok
            al[:, t * cin:(t + 1) * cin] = src.lo[bb, yc, xc] * ok
        if mode == "three":
            ref1[s:s + chunk] = ah @ wh
            ref[s:s + chunk] = ref1[s:s + chunk] + ah @ wl + al @ wh
        elif mode == "one":
            ref[s:s + chunk] = ah @ wh
        else:
            ref[s:s + chunk] = (ah + al) @ wh
        S[s:s + chunk] = np.abs(ah + al) @ w_abs
    return ref, np.sqrt(len(taps) * cin) * S, ref1


def leaky(x):
    return np.where(x >= 0, x, 0.2 * x)


def ratio(got, ref, bound):
    return np.abs(got - ref) / bound


# ---------------------------------------------------------------------------------------------------------------------
# pixel samples
# ---------------------------------------------------------------------------------------------------------------------
def all_pixels(B, H, W):
    b, y, x = np.meshgrid(np.arange(B), np.arange(H), np.arange(W), indexing="ij")
    return b.ravel(), y.ravel(), x.ravel()


def sampled_pixels(B, H, W, rng, n_random=2000):
    """First / last two rows and columns, whole rows and columns on both sides of a random subset of the 8/16/32-pixel
    tile boundaries, and n_random random pixels; every batch."""
    rows, cols = {0, 1, H - 2, H - 1}, {0, 1, W - 2, W - 1}
    for t in (8, 16, 32):
        for lines, n in ((rows, H), (cols, W)):
            cand = np.arange(t, n, t)
            for c in rng.choice(cand, size=min(2, len(cand)), replace=False) if len(cand) else []:
                lines.update({int(c) - 1, int(c)})
    pts = set()
    for bb in range(B):
        for r in rows:
            if 0 <= r < H:
                pts.update((bb, r, xx) for xx in range(W))
        for c in cols:
            if 0 <= c < W:
                pts.update((bb, yy, c) for yy in range(H))
    pts.update(zip(rng.integers(0, B, n_random).tolist(), rng.integers(0, H, n_random).tolist(),
                   rng.integers(0, W, n_random).tolist()))
    a = np.array(sorted(pts), np.int64)
    return a[:, 0], a[:, 1], a[:, 2]


# ---------------------------------------------------------------------------------------------------------------------
# wiring: which op reads what (one rule per op-name pattern)
# ---------------------------------------------------------------------------------------------------------------------
RULES = [
    ("fe_conv0", re.compile(r"^fe_conv0(\+pool)?@L(\d)$")),
    ("fe_conv_even", re.compile(r"^fe_conv([246])@L(\d)$")),
    ("fe_conv_odd", re.compile(r"^fe_conv([1357])@L(\d)$")),
    ("flow_conv", re.compile(r"^flow_conv([012])@L(\d)$")),
    ("flow_head", re.compile(r"^flow_(conv2\+head|head)@L(\d)$")),
    ("fusion_up", re.compile(r"^fusion_up[0-3]?@L(\d)$")),
    ("fusion_conv1", re.compile(r"^fusion_conv1@L(\d)$")),
    ("fusion_conv2", re.compile(r"^fusion_conv2@L(\d)$")),
    ("rgb", re.compile(r"^(fusion_conv2\+rgb@L0|rgb_head)$")),
]
CAT2_CONVS = re.compile(r"^(fe_conv0|flow_head|rgb_head)")


def rule_of(name):
    for kind, rx in RULES:
        m = rx.match(name)
        if m:
            return kind, m
    raise AssertionError(f"op {name!r} matches no wiring rule: a new layer or form needs a rule in this file")


def op_stage(name):
    """Precision-plan stage of a conv op (None: always three-pass / fp32)."""
    kind, m = rule_of(name)
    if kind == "fe_conv0":
        return fe_stage(int(m.group(2)), 0)
    if kind in ("fe_conv_even", "fe_conv_odd"):
        k, r = int(m.group(1)), int(m.group(2))
        return fe_stage(r - k // 2, k)
    if kind == "flow_conv":
        return ST_FLOW_L0 + int(m.group(2))
    if kind == "flow_head":
        return ST_FLOW_L0 + int(m.group(2)) if m.group(1) == "conv2+head" else None
    if kind == "rgb":
        return ST_FUS + 2 if name.startswith("fusion") else None
    i = int(m.group(1))
    return ST_FUS + 3 * i + {"fusion_up": 0, "fusion_conv1": 1, "fusion_conv2": 2}[kind]


def consumer_stage(name):
    """Stage of the only reader of the op's split destination when that reader is a conv (None otherwise)."""
    kind, m = rule_of(name)
    if kind == "fe_conv0":
        return fe_stage(int(m.group(2)), 1)
    if kind == "fe_conv_even":
        k, r = int(m.group(1)), int(m.group(2))
        return fe_stage(r - k // 2, k + 1)
    if kind == "flow_conv":
        return ST_FLOW_L0 + int(m.group(2)) if m.group(1) != "2" else None
    if kind in ("fusion_up", "fusion_conv1"):
        return op_stage(name) + 1
    if kind == "fusion_conv2":
        i = int(m.group(1))
        return ST_FUS + 3 * (i - 1) if i > 0 else None
    return None


class Plan:
    """What the test needs to know of one engine plan."""

    def __init__(self, eng, h, w, align, opts):
        self.eng, self.opts = eng, opts
        self.fmt = "fp16" if "split=fp16" in eng.version else "bf16"
        self.p = fmt_bits(self.fmt)
        ph, pw, self.off_y, self.off_x = spec.padded_shape(h, w, align)
        self.h, self.w = h, w
        self.sizes = [(ph >> l, pw >> l) for l in range(LEVELS)]
        self.mask = eng.get_option("onepass_mask")
        self.impl = eng.get_option("conv_impl")
        self.plane_skip = eng.get_option("plane_skip")
        self.table = eng.op_table()
        self.names = {r["name"] for r in self.table}

    def onepass(self, stage):
        return stage is not None and self.impl == 0 and (self.mask >> stage) & 1 == 1

    def hi_only(self, consumer):
        return bool(self.plane_skip) and self.onepass(consumer)

    def read(self, name, shape):
        return self.eng.debug_read(name).astype(np.float64).reshape(shape)

    def planes(self, name, shape):
        return Src(self.read(name + ".hi", shape), self.read(name + ".lo", shape))


def aligned_level(P, l):
    """concat of the aligned pyramid level l in the reference channel order:
    [img0w(3), feat0w(C), img1w(3), feat1w(C), bwd(2), fwd(2)] = [side 0:3, warped0, side 3:6, warped1, side 6:10]."""
    H, W = P.sizes[l]
    C = spec.feature_channels(l)
    side = P.planes(f"aligned_side/{l}", (1, H, W, 10))
    w0 = P.planes(f"warped0/{l}", (1, H, W, C))
    w1 = P.planes(f"warped1/{l}", (1, H, W, C))
    cat = lambda k: np.concatenate([getattr(side, k)[..., 0:3], getattr(w0, k), getattr(side, k)[..., 3:6],
                                    getattr(w1, k), getattr(side, k)[..., 6:10]], axis=-1)
    return Src(cat("hi"), cat("lo"))


def concat(*srcs):
    return Src(np.concatenate([s.hi for s in srcs], -1), np.concatenate([s.lo for s in srcs], -1))


# ---------------------------------------------------------------------------------------------------------------------
# the walk over the op table
# ---------------------------------------------------------------------------------------------------------------------
class Report:
    def __init__(self):
        self.rows = []        # (op, what, form, passes, max err/bound, max err/(2^-24 S), worst pixel)
        self.frac = {}        # op -> single-pass fractions of its outputs
        self.fail = []

    def single_pass_fraction(self, op, what, passes, got, want3, want1):
        """Projection of the layer's error on the single-pass deviation d = want1 - want3: c = <got - want3, d> / <d, d>.
        A correct three-pass layer has c ~ 0 (its accumulation error does not follow the low-order product terms),
        one that ran single-pass has c ~ 1, one that dropped a share of the low-order terms has about that share."""
        if want1 is None:
            return
        d = want1 - want3
        dd = float((d * d).sum())
        c = float(((got - want3) * d).sum()) / dd if dd > 0 else 0.0
        self.frac.setdefault(op, []).append(c)
        if passes == 3 and not abs(c) <= FRAC_MAX:
            self.fail.append(f"{op} [{what}]: runs three-pass, but {c:.3f} of the single-pass deviation is in its output")

    def check(self, op, what, form, passes, got, ref, bound, S, pix):
        r = ratio(got, ref, bound)
        k = int(np.argmax(r)) if r.size else 0
        worst = float(r.flat[k]) if r.size else 0.0
        # the part of the error the TAU term has to cover: what is left after the output rounding allowance
        acc = float(((np.abs(got - ref) - (bound - TAU * 2.0 ** -24 * S)) / (2.0 ** -24 * np.maximum(S, 1e-300))).max()
                    ) if r.size else 0.0
        where = tuple(int(a[k // r.shape[1]]) for a in pix) + (k % r.shape[1],) if r.ndim == 2 and r.size else ()
        self.rows.append((op, what, form, passes, worst, acc, where))
        if not np.isfinite(got).all() or worst > 1.0:
            self.fail.append(f"{op} [{what}, form {form}, {passes}-pass]: max err/bound {worst:.3g} at (b, y, x, c) = "
                             f"{where}: got {got.flat[k]:.9g}, want {ref.flat[k]:.9g}, bound {bound.flat[k]:.3g}")

    def require(self, cond, msg):
        if not cond:
            self.fail.append(msg)


def pick(arr, pix):
    b, y, x = pix
    return arr[b, y, x]


def check_plan(P, wts, rng, sampled, mode_override=None):
    """Walks the op table of the last call of P.eng; returns a Report.  mode_override = "three" checks every
    tensor-core layer against the three-pass reference whatever it ran (the self-check)."""
    rep = Report()
    eps_hi, eps_lo = 2.0 ** -P.p, 2.0 ** -(2 * P.p - 1)
    conv_ops = [r for r in P.table if r["category"] == 0 or (r["category"] == 2 and CAT2_CONVS.match(r["name"]))]
    for r in P.table:   # coverage guard: every conv matches a rule, and its passes follow the plan
        if r in conv_ops:
            rule_of(r["name"])
            if r["category"] == 0:
                st = op_stage(r["name"])
                want = 1 if P.onepass(st) else 3
                rep.require(r["passes"] == want, f"{r['name']}: passes {r['passes']}, the plan says {want}")
    tau = TAU * 2.0 ** -24

    def pix_for(B, H, W):
        return sampled_pixels(B, H, W, rng) if sampled else all_pixels(B, H, W)

    def finish_split(op, name, B, H, W, cout, act, ref, S, bias, pix, passes, form, consumer, ref1=None, what="out"):
        """Compares the split destination `name` with the reference at pix; returns the activated fp64 reference."""
        f = leaky if act else (lambda v: v)
        want = f(ref + bias)
        S = S + np.abs(bias)
        hi_only = consumer is not None and P.hi_only(consumer)
        got_hi = pick(P.read(name + ".hi", (B, H, W, cout)), pix)
        lo = P.read(name + ".lo", (B, H, W, cout))
        if hi_only:
            rep.require(not lo.any(), f"{op}: lo plane of {name} written although every reader is single-pass")
        else:
            rep.require(lo.any(), f"{op}: lo plane of {name} never written although a three-pass conv reads it")
        got = got_hi + pick(lo, pix)
        eps = eps_hi if hi_only else eps_lo
        rep.check(op, what, form, passes, got, want, tau * S + eps * np.abs(want) + 2.0 ** -25, S, pix)
        rep.single_pass_fraction(op, what, passes, got, want, None if ref1 is None else f(ref1 + bias))
        return want, S

    for r in conv_ops:
        op, form, passes = r["name"], r["form"], r["passes"]
        kind, m = rule_of(op)
        if kind == "fusion_up" and op[9] != "@":
            if op[9] != "0":
                continue   # the validation path's four parity-class launches share one destination: checked once
        mode = {"simt": "simt", "": "fp32"}.get(form) or mode_override or ("one" if passes == 1 else "three")
        if kind == "fe_conv0":
            l = int(m.group(2))
            H, W = P.sizes[l]
            img = P.read(f"img/{l}", (2, H, W, 3))
            if l + 1 < LEVELS:   # the image pyramid, fused into this conv or not: avg_pool to 2 ulp
                nxt = P.read(f"img/{l + 1}", (2,) + P.sizes[l + 1] + (3,))
                h2, w2 = P.sizes[l + 1]
                want = 0.25 * (img[:, 0:2 * h2:2, 0:2 * w2:2] + img[:, 0:2 * h2:2, 1:2 * w2:2]
                               + img[:, 1:2 * h2:2, 0:2 * w2:2] + img[:, 1:2 * h2:2, 1:2 * w2:2])
                rep.require(np.all(np.abs(nxt - want) <= 2 * np.spacing(np.abs(want).astype(np.float32))),
                            f"img/{l + 1} is not the 2x2 mean of img/{l}")
            k = wts[FE + "0/kernel"]
            if form == "3x3":   # tensor-core form over the 32-channel split image
                sp = P.planes(f"out:fe_split32@L{l}", (2, H, W, 32))
                hi, lo = split_w(img.astype(np.float32), P.fmt)
                rep.require(np.array_equal(sp.hi[..., :3], hi) and np.array_equal(sp.lo[..., :3], lo)
                            and not sp.hi[..., 3:].any(), f"fe_split32@L{l} is not the split image")
                src, taps = Src(sp.hi[..., :3], sp.lo[..., :3]), taps_3x3(k)
            elif form == "tc":   # generic kernel: a 1x1 conv over the 27 im2col channels
                col = P.planes(f"out:fe_im2col@L{l}", (2, H, W, 32))
                pad = np.pad(img, ((0, 0), (1, 1), (1, 1), (0, 0)))
                want = np.concatenate([pad[:, ky:ky + H, kx:kx + W] for ky in range(3) for kx in range(3)], -1)
                hi, lo = split_w(want.astype(np.float32), P.fmt)
                rep.require(np.array_equal(col.hi[..., :27], hi) and np.array_equal(col.lo[..., :27], lo),
                            f"fe_im2col@L{l} is not the split im2col of img/{l}")
                src, taps = Src(col.hi[..., :27], col.lo[..., :27]), [(0, 0, k.reshape(27, 64))]
            else:                # fp32 FMA kernel or validation kernel, straight from the fp32 image
                src, taps = Src(img), taps_3x3(k)
            pix = pix_for(2, H, W)
            ref, S, ref1 = conv_at(src, taps, *pix, mode, P.fmt)
            finish_split(op, "out:" + op, 2, H, W, 64, True, ref, S, wts[FE + "0/bias"], pix,
                         passes or 3, form, None if P.impl else consumer_stage(op), ref1)
        elif kind in ("fe_conv_even", "fe_conv_odd"):
            kk, l = int(m.group(1)), int(m.group(2))
            j, H, W = kk // 2, *P.sizes[l]
            cin, cout = (64 << (j - 1) if kk % 2 == 0 else 64 << j), 64 << j
            if kind == "fe_conv_even":   # the pooled previous pair: fused into its second conv, or fe_pool@L{l - 1}
                name = f"pool:fe_conv{kk - 1}@L{l - 1}"
                if f"fe_pool@L{l - 1}" in P.names:
                    _check_fe_pool(P, rep, f"fe_conv{kk - 1}@L{l - 1}", l - 1, cin, eps_lo)
            elif kk == 1:
                name = "out:" + next(n for n in (f"fe_conv0+pool@L{l}", f"fe_conv0@L{l}") if n in P.names)
            else:
                name = f"out:fe_conv{kk - 1}@L{l}"
            src = P.planes(name, (2, H, W, cin))
            pix = pix_for(2, H, W)
            ref, S, ref1 = conv_at(src, taps_3x3(wts[f"{FE}{kk}/kernel"]), *pix, mode, P.fmt)
            want, Sb = finish_split(op, "out:" + op, 2, H, W, cout, True, ref, S, wts[f"{FE}{kk}/bias"], pix,
                                    passes, form, consumer_stage(op), ref1)
            if kind == "fe_conv_odd":
                for k in range(2):   # the destination is channel slice j of the cascaded feature tensor
                    C = spec.feature_channels(l)
                    feat = P.read(f"feat{k}/{l}", (H, W, C))[..., SLICE_OFF[j]:SLICE_OFF[j] + cout]
                    out = P.read("out:" + op, (2, H, W, cout))[k]
                    rep.require(np.array_equal(feat.astype(np.float32), out.astype(np.float32)),
                                f"{op} did not write channel slice {SLICE_OFF[j]} of feat{k}/{l}")
                if f"fe_conv{kk + 1}@L{l + 1}" in P.names and f"fe_pool@L{l}" not in P.names:
                    _check_pool(P, rep, op, l, cout, src, wts, kk, mode, passes, form, eps_lo, tau, sampled, rng)
        elif kind == "flow_conv":
            k, l = int(m.group(1)), int(m.group(2))
            p = min(l, 3)
            nf, C, (H, W) = spec.FLOW_FILTERS[p], spec.feature_channels(l), P.sizes[l]
            pre = f"predict_flow/{spec.FLOW_PREDICTOR_NAMES[p]}/conv_{k}/"
            if k == 0:
                feats = [P.planes(f"feat{d}/{l}", (1, H, W, C)) for d in range(2)]
                if l == LEVELS - 1:
                    other = [feats[1], feats[0]]   # bswap: the features of the other image, unwarped
                else:
                    other = [P.planes(f"flow_warped{d}/{l}", (1, H, W, C)) for d in range(2)]
                src = Src(np.concatenate([concat(feats[d], other[d]).hi for d in range(2)]),
                          np.concatenate([concat(feats[d], other[d]).lo for d in range(2)]))
            else:
                src = P.planes(f"out:flow_conv{k - 1}@L{l}", (2, H, W, nf))
            pix = pix_for(2, H, W)
            ref, S, ref1 = conv_at(src, taps_3x3(wts[pre + "kernel"]), *pix, mode, P.fmt)
            finish_split(op, "out:" + op, 2, H, W, nf, True, ref, S, wts[pre + "bias"], pix, passes, form,
                         None if P.impl else consumer_stage(op), ref1)
        elif kind == "flow_head":
            l = int(m.group(2))
            p = min(l, 3)
            nf, (H, W) = spec.FLOW_FILTERS[p], P.sizes[l]
            pre = f"predict_flow/{spec.FLOW_PREDICTOR_NAMES[p]}/conv_"
            pix = pix_for(2, H, W)
            if m.group(1) == "conv2+head":   # conv_2 on the tensor cores, its activation stays in fp32 registers
                src = P.planes(f"out:flow_conv1@L{l}", (2, H, W, nf))
                ref, S, ref1 = conv_at(src, taps_3x3(wts[pre + "2/kernel"]), *pix, mode, P.fmt)
                h2 = leaky(ref + wts[pre + "2/bias"])
                e2 = tau * (S + np.abs(wts[pre + "2/bias"])) + 2.0 ** -24 * np.abs(h2)
                w3 = wts[pre + "3/kernel"][0, 0].astype(np.float64)
                h3 = leaky(h2 @ w3 + wts[pre + "3/bias"])
                h3_1 = None if ref1 is None else leaky(leaky(ref1 + wts[pre + "2/bias"]) @ w3 + wts[pre + "3/bias"])
                e3 = e2 @ np.abs(w3) + tau * np.sqrt(nf) * (np.abs(wts[pre + "3/bias"]) + np.abs(h2) @ np.abs(w3))
                S3 = None
            else:   # conv_3 (1x1) on the tensor cores (three-pass) or on the validation kernel, from conv_2's planes
                src = P.planes(f"out:flow_conv2@L{l}", (2, H, W, nf))
                ref3, S3, ref31 = conv_at(src, [(0, 0, wts[pre + "3/kernel"][0, 0])], *pix, mode, P.fmt)
                h3 = leaky(ref3 + wts[pre + "3/bias"])
                h3_1 = None if ref31 is None else leaky(ref31 + wts[pre + "3/bias"])
                e3 = tau * (S3 + np.abs(wts[pre + "3/bias"])) + 2.0 ** -24 * np.abs(h3)
            w4 = wts[pre + "4/kernel"][0, 0].astype(np.float64)
            res = h3 @ w4 + wts[pre + "4/bias"]
            res1 = None if h3_1 is None else h3_1 @ w4 + wts[pre + "4/bias"]
            e_res = e3 @ np.abs(w4) + tau * np.sqrt(nf // 2) * (np.abs(wts[pre + "4/bias"]) + np.abs(h3) @ np.abs(w4)) + 2.0 ** -25
            S_res = (S3 if S3 is not None else S).max(axis=1, keepdims=True) * np.ones_like(res)
            for d, dn in enumerate(("fwd", "bwd")):
                sel = pix[0] == d
                sub = tuple(a[sel] for a in pix)
                got = P.read(f"res_{dn}/{l}", (H, W, 2))[sub[1], sub[2]]
                rep.check(op, f"res_{dn}", form, passes, got, res[sel], e_res[sel], S_res[sel], sub)
                rep.single_pass_fraction(op, f"res_{dn}", passes, got, res[sel], None if res1 is None else res1[sel])
                v = res[sel] + (P.read(f"flow_vup{d}/{l}", (H, W, 2))[sub[1], sub[2]] if l < LEVELS - 1 else 0.0)
                got = P.read(f"flow_{dn}/{l}", (H, W, 2))[sub[1], sub[2]]
                rep.check(op, f"flow_{dn}", form, passes, got, v, e_res[sel] + 2.0 ** -24 * np.abs(v), S_res[sel], sub)
        elif kind == "fusion_up":
            i = int(m.group(1))
            nf, (H, W), (Hc, Wc) = spec.fusion_filters(i), P.sizes[i], P.sizes[i + 1]
            k0 = wts[f"fusion/level_{i}/conv_0/kernel"]
            if i == FUSION - 2:
                x = aligned_level(P, i + 1)
            else:
                x = P.planes(f"out:fusion_conv2@L{i + 1}", (1, Hc, Wc, spec.fusion_filters(i + 1)))
            pix = pix_for(1, H, W)
            ref, S = np.zeros((len(pix[0]), nf)), np.zeros((len(pix[0]), nf))
            ref1 = np.zeros((len(pix[0]), nf)) if mode == "three" else None
            if f"fusion_resize@L{i}" in P.names:   # a gather of its own, then a plain 2x2 SAME conv on the fine grid
                xr = _check_resize(P, rep, i, x, H, W)
                ref, S, ref1 = conv_at(xr, [(ty, tx, k0[ty, tx]) for ty in range(2) for tx in range(2)], *pix, mode, P.fmt)
            else:   # one launch over the coarse grid per parity class
                for py in range(2):
                    for px in range(2):
                        sel = (pix[1] % 2 == py) & (pix[2] % 2 == px)
                        ref[sel], S[sel], r1 = conv_at(x, taps_parity(k0, py, px), pix[0][sel], pix[1][sel] // 2,
                                                   pix[2][sel] // 2, mode, P.fmt)
                        if r1 is not None:
                            ref1[sel] = r1
            finish_split(op, f"out:fusion_up@L{i}", 1, H, W, nf, False, ref, S,
                         wts[f"fusion/level_{i}/conv_0/bias"], pix, passes or 3, form,
                         None if P.impl else consumer_stage(f"fusion_up@L{i}"), ref1)
        elif kind in ("fusion_conv1", "fusion_conv2") or kind == "rgb":
            i = int(m.group(1)) if kind != "rgb" else 0
            nf, (H, W) = spec.fusion_filters(i), P.sizes[i]
            c = 1 if kind == "fusion_conv1" else 2
            pre = f"fusion/level_{i}/conv_{c}/"
            pix = pix_for(1, H, W)
            if op == "rgb_head":   # fp32 1x1 on the values of conv_2's destination
                src = P.planes("out:fusion_conv2@L0", (1, H, W, nf))
                h2, e2, ref, ref1 = pick(src.hi + src.lo, pix), 0.0, None, None
            else:
                if c == 1:
                    src = concat(aligned_level(P, i), P.planes(f"out:fusion_up@L{i}", (1, H, W, nf)))
                else:
                    src = P.planes(f"out:fusion_conv1@L{i}", (1, H, W, nf))
                ref, S, ref1 = conv_at(src, taps_3x3(wts[pre + "kernel"]), *pix, mode, P.fmt)
            if kind != "rgb":
                finish_split(op, "out:" + op, 1, H, W, nf, True, ref, S, wts[pre + "bias"], pix, passes, form,
                             None if P.impl else consumer_stage(op), ref1)
                continue
            if ref is not None:   # fused: conv_2 in fp32 registers, then output_conv and the crop in the epilogue
                h2 = leaky(ref + wts[pre + "bias"])
                e2 = tau * (S + np.abs(wts[pre + "bias"])) + 2.0 ** -24 * np.abs(h2)
            wr = wts["fusion/output_conv/kernel"][0, 0].astype(np.float64)
            rgb = h2 @ wr + wts["fusion/output_conv/bias"]
            rgb1 = None if ref1 is None else leaky(ref1 + wts[pre + "bias"]) @ wr + wts["fusion/output_conv/bias"]
            e_rgb = (np.asarray(e2) @ np.abs(wr) if np.ndim(e2) else 0.0) + \
                tau * 8.0 * (np.abs(wts["fusion/output_conv/bias"]) + np.abs(h2) @ np.abs(wr)) + 2.0 ** -25
            oy, ox = pix[1] - P.off_y, pix[2] - P.off_x
            inside = (oy >= 0) & (oy < P.h) & (ox >= 0) & (ox < P.w)
            img = P.read("image", (P.h, P.w, 3))
            got = img[oy[inside], ox[inside]]
            S_rgb = np.abs(h2) @ np.abs(wr) + np.abs(wts["fusion/output_conv/bias"])   # the 1x1 layer's own sum
            rep.check(op, "image", form, passes, got, rgb[inside], e_rgb[inside], S_rgb[inside],
                      tuple(a[inside] for a in pix))
            rep.single_pass_fraction(op, "image", passes, got, rgb[inside], None if rgb1 is None else rgb1[inside])
    return rep


def _check_fe_pool(P, rep, prev, l, c, eps):
    """The stand-alone pool: 2x2 mean of the activated feature slice, re-split."""
    H, W = P.sizes[l]
    h2, w2 = P.sizes[l + 1]
    src = P.read("out:" + prev, (2, H, W, c))
    want = 0.25 * (src[:, 0:2 * h2:2, 0:2 * w2:2] + src[:, 0:2 * h2:2, 1:2 * w2:2]
                   + src[:, 1:2 * h2:2, 0:2 * w2:2] + src[:, 1:2 * h2:2, 1:2 * w2:2])
    got = P.read(f"pool:{prev}", (2, h2, w2, c))
    bound = 2.0 ** -23 * np.abs(want) + eps * np.abs(want) + 2.0 ** -25
    rep.check(f"fe_pool@L{l}", "out", "", 0, got.reshape(-1, c), want.reshape(-1, c), bound.reshape(-1, c),
              np.abs(want).reshape(-1, c), all_pixels(2, h2, w2))


def _check_pool(P, rep, op, l, cout, src, wts, kk, mode, passes, form, eps, tau, sampled, rng):
    """Fused pool of a conv: the 2x2 mean of the activated fp32 values, the last odd row / column clipped."""
    h2, w2 = P.sizes[l + 1]
    pp = sampled_pixels(2, h2, w2, rng, 500) if sampled else all_pixels(2, h2, w2)
    acc = np.zeros((len(pp[0]), cout))
    Ssum = np.zeros_like(acc)
    for dy in range(2):
        for dx in range(2):
            ref, S, ref1 = conv_at(src, taps_3x3(wts[f"{FE}{kk}/kernel"]), pp[0], 2 * pp[1] + dy, 2 * pp[2] + dx,
                                    mode, P.fmt)
            acc += leaky(ref + wts[f"{FE}{kk}/bias"])
            Ssum += S + np.abs(wts[f"{FE}{kk}/bias"])
    want, S = 0.25 * acc, 0.25 * Ssum
    got = pick(P.read(f"pool:{op}.hi", (2, h2, w2, cout)) + P.read(f"pool:{op}.lo", (2, h2, w2, cout)), pp)
    rep.check(op, "pool", form, passes, got, want, tau * S + 2.0 ** -23 * np.abs(want) + eps * np.abs(want)
              + 2.0 ** -25, S, pp)


def _check_resize(P, rep, i, x, H, W):
    """fusion_resize: an exact nearest gather of the coarse planes (TF2 NEAREST, half-pixel centres)."""
    Hc, Wc = x.hi.shape[1:3]
    ys = np.minimum((2 * np.arange(H) + 1) * Hc // (2 * H), Hc - 1)
    xs = np.minimum((2 * np.arange(W) + 1) * Wc // (2 * W), Wc - 1)
    want = Src(x.hi[:, ys][:, :, xs], x.lo[:, ys][:, :, xs])
    if i == FUSION - 2:   # the warped B = 2 tensor and the side tensor, read back in the reference channel order
        C = spec.feature_channels(i + 1)
        w = P.planes(f"out:fusion_resize@L{i}", (2, H, W, C))
        sd = P.planes(f"out:fusion_resize@L{i}:side", (1, H, W, 64))
        got = Src(*(np.concatenate([getattr(sd, k)[..., 0:3], getattr(w, k)[0:1], getattr(sd, k)[..., 3:6],
                                    getattr(w, k)[1:2], getattr(sd, k)[..., 6:10]], -1) for k in ("hi", "lo")))
    else:
        got = P.planes(f"out:fusion_resize@L{i}", (1, H, W, x.hi.shape[-1]))
    hi_only = P.hi_only(ST_FUS + 3 * i)
    rep.require(np.array_equal(got.hi, want.hi) and np.array_equal(got.lo, 0 * want.lo if hi_only else want.lo),
                f"fusion_resize@L{i} is not the nearest resize of its source planes")
    return got


# ---------------------------------------------------------------------------------------------------------------------
# engines and cases
# ---------------------------------------------------------------------------------------------------------------------
def run_plan(weights_path, h, w, align, opts, seed=7):
    from frame_interpolation_b200.interpolator import Interpolator
    eng = Interpolator(weights_path, align=align)
    if align is None:
        eng.set_option("any_size", 1)
    eng.set_option("keep_debug", 1)
    for k, v in opts.items():
        eng.set_option(k, v)
    x0, x1 = synthetic.frame_pair(h, w, seed=seed, n_waves=8)
    out = eng(x0, x1, DT).copy()
    return eng, out, x0, x1


def summarize(rep):
    by = {}
    for op, what, form, passes, worst, acc, _ in rep.rows:
        kind = re.sub(r"@L\d$", "", op) + f"/{form or 'fp32'}/{passes or '-'}"
        b = by.setdefault(kind, [0.0, 0.0])
        b[0], b[1] = max(b[0], worst), max(b[1], acc)
    return by


def assert_report(rep, label):
    by = summarize(rep)
    print(f"\n[{label}] layer type: max err/bound, max err/(2^-24 S)")
    for k in sorted(by):
        print(f"  {k:40s} {by[k][0]:8.4f} {by[k][1]:10.3f}")
    three = {op: max(abs(c) for c in cs) for op, cs in rep.frac.items()
             if any(r[0] == op and r[3] == 3 for r in rep.rows)}
    if three:
        top = max(three, key=three.get)
        print(f"  largest single-pass fraction of a three-pass layer: {three[top]:.4f} ({top})")
    print("  largest err/(2^-24 S):", ", ".join(f"{op} {what} {acc:.2f}" for op, what, _, _, _, acc, _ in
                                                 sorted(rep.rows, key=lambda r: -r[5])[:8]))
    assert not rep.fail, f"{label}: {len(rep.fail)} failures\n" + "\n".join(rep.fail[:30])


SMALL = [(256, 320, 64), (100, 150, None), (65, 129, None)]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("mask", ["default", 0])
@pytest.mark.parametrize("h,w,align", SMALL, ids=[f"{h}x{w}" for h, w, _ in SMALL])
def test_every_conv_layer_matches_float64(synthetic_weights, h, w, align, mask):
    opts = {} if mask == "default" else {"onepass_mask": mask}
    eng, _, _, _ = run_plan(synthetic_weights[0], h, w, align, opts)
    try:
        assert eng.stage_names() == stage_names()
        P = Plan(eng, h, w, align, opts)
        assert_report(check_plan(P, synthetic_weights[1], np.random.default_rng(1), sampled=False), f"{h}x{w} {mask}")
    finally:
        eng.close()


OPTION_CASES = [({"conv3x3_pxn": 0}, lambda f: "3x3_pxn" not in f.values()),
                ({"conv3x3_pxn": 2}, lambda f: "3x3_pxn" in f.values()),
                ({"conv3x3_halo": 0}, None), ({"conv3x3_halo": 2}, None),
                ({"conv3x3_2cta": 2}, lambda f: "3x3_pair" in f.values()), ({"mma_straight": 0}, None),
                ({"conv3x3_v2": 0}, lambda f: set(f.values()) == {"tc"}),
                ({"fe_conv0_tc": 1}, lambda f: f["fe_conv0@L0"] == "3x3"),
                ({"fe_conv0_tc": 1, "conv3x3_v2": 0}, lambda f: f["fe_conv0@L0"] == "tc"),
                ({"fuse_flow_head": 0}, lambda f: "flow_head@L0" in f and not any("+head" in n for n in f)),
                ({"fuse_flow_head": 2}, lambda f: "flow_conv2+head@L1" in f),
                ({"fuse_rgb_head": 0}, lambda f: "fusion_conv2@L0" in f and "fusion_conv2+rgb@L0" not in f),
                ({"plane_skip": 0}, None),
                ({"conv_impl": 1}, lambda f: set(f.values()) == {"simt"})]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("opts,form_ok", OPTION_CASES, ids=[",".join(f"{k}={v}" for k, v in o.items()) for o, _ in OPTION_CASES])
def test_every_conv_layer_matches_float64_per_option(synthetic_weights, opts, form_ok):
    h, w = 64, 128
    eng, _, _, _ = run_plan(synthetic_weights[0], h, w, 64, opts)
    try:
        P = Plan(eng, h, w, 64, opts)
        forms = {r["name"]: r["form"] for r in P.table if r["category"] == 0}
        assert form_ok is None or form_ok(forms), forms
        assert_report(check_plan(P, synthetic_weights[1], np.random.default_rng(2), sampled=False), str(opts))
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_cta_pair_layers_match_float64(synthetic_weights):
    """conv3x3_2cta = 1 pairs only layers with at least 4 tiles per SM; at 256x320 fusion_conv1@L0 (640 16x8 tiles,
    streamed weights) is one.  conv3x3_halo = 1 gives the wide halo to the paired layers only."""
    opts = {"conv3x3_2cta": 1, "conv3x3_halo": 1}
    eng, _, _, _ = run_plan(synthetic_weights[0], 256, 320, 64, opts)
    try:
        P = Plan(eng, 256, 320, 64, opts)
        paired = [r["name"] for r in P.table if r["form"] == "3x3_pair"]
        assert "fusion_conv1@L0" in paired, paired
        assert_report(check_plan(P, synthetic_weights[1], np.random.default_rng(5), sampled=False), str(opts))
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.timeout(1200)
@pytest.mark.parametrize("h,w", [(704, 1536), (1088, 1920)])
@pytest.mark.parametrize("mask", ["default", 0])
def test_conv_layers_at_large_sizes_sampled(synthetic_weights, h, w, mask):
    import torch
    opts = {} if mask == "default" else {"onepass_mask": mask}
    eng, _, _, _ = run_plan(synthetic_weights[0], h, w, 64, opts)
    try:
        free, _ = torch.cuda.mem_get_info()
        if h == 1088 and eng.profile()["arena_bytes"] * 3 > free + eng.profile()["arena_bytes"]:
            pytest.skip(f"keep_debug arena {eng.profile()['arena_bytes'] / 2**30:.1f} GiB is over a third of free memory")
        P = Plan(eng, h, w, 64, opts)
        if h == 1088 and mask == "default":
            assert {r["name"]: r["form"] for r in P.table}["fusion_conv1@L0"] == "3x3_pxn"
        assert_report(check_plan(P, synthetic_weights[1], np.random.default_rng(3), sampled=True), f"{h}x{w} {mask}")
    finally:
        eng.close()


@pytest.mark.gpu
def test_single_pass_plan_is_caught_on_every_tensor_core_layer(synthetic_weights):
    """Self-check: every stage single-pass, every lo plane written (plane_skip = 0, as behind a three-pass layer).  The
    layers pass against the single-pass reference, and checked as if they had run three-pass, every tensor-core layer
    carries at least 4 x FRAC_MAX of the single-pass deviation: a three-pass layer that ran single-pass is caught.  The
    per-element bound is printed for comparison: it alone misses the larger-K layers (module docstring)."""
    h, w = 100, 150
    opts = {"onepass_mask": (1 << ST_COUNT) - 1, "plane_skip": 0}
    eng, _, _, _ = run_plan(synthetic_weights[0], h, w, None, opts)
    try:
        P = Plan(eng, h, w, None, opts)
        assert_report(check_plan(P, synthetic_weights[1], np.random.default_rng(4), sampled=False), "all single-pass")
        rep3 = check_plan(P, synthetic_weights[1], np.random.default_rng(4), sampled=False, mode_override="three")
        worst = {}
        for op, what, form, passes, r, _, _ in rep3.rows:
            worst[op] = max(worst.get(op, 0.0), r)
        tc = [r["name"] for r in P.table if r["category"] == 0 and r["passes"] == 1]   # all but the unfused flow heads
        assert len(tc) > 60 and set(tc) <= set(rep3.frac)
        frac = {op: min(rep3.frac[op]) for op in tc}
        print("\n[self-check] single-pass fraction (max err/bound against three-pass):",
              ", ".join(f"{op} {frac[op]:.3f} ({worst[op]:.1f})" for op in sorted(tc, key=frac.get)))
        weak = {op: round(c, 3) for op, c in frac.items() if c < 4 * FRAC_MAX}
        assert not weak, weak
    finally:
        eng.close()


BITWISE_SIZES = [(256, 320, 64), (100, 150, None), (704, 1536, 64)]


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("h,w,align", BITWISE_SIZES, ids=[f"{h}x{w}" for h, w, _ in BITWISE_SIZES])
def test_scheduling_options_do_not_change_a_bit(synthetic_weights, h, w, align):
    """arena_reuse, use_graph, time_ops and keep_debug change scheduling and memory, not arithmetic: any difference in
    the output is a liveness or race bug."""
    from frame_interpolation_b200.interpolator import Interpolator
    x0, x1 = synthetic.frame_pair(h, w, seed=5, n_waves=8)
    outs = {}
    for opt, val in ((None, None), ("arena_reuse", 0), ("use_graph", 0), ("time_ops", 1), ("keep_debug", 1)):
        eng = Interpolator(synthetic_weights[0], align=align)
        if align is None:
            eng.set_option("any_size", 1)
        if opt:
            eng.set_option(opt, val)
        outs[opt] = eng(x0, x1, DT).copy()
        eng.close()
    for opt, out in outs.items():
        np.testing.assert_array_equal(out, outs[None], err_msg=str(opt))


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the reference machinery against the oracle, in float64 on synthetic tensors
# ---------------------------------------------------------------------------------------------------------------------
def _oracle_conv(x_nhwc, kernel, bias):
    import torch
    from oracle.film_oracle import conv2d_same
    x = torch.from_numpy(np.asarray(x_nhwc, np.float64)).permute(0, 3, 1, 2)
    y = conv2d_same(x, torch.from_numpy(np.asarray(kernel, np.float64)), torch.from_numpy(np.asarray(bias, np.float64)),
                    False)
    return y.permute(0, 2, 3, 1).numpy()


def test_reference_conv_and_parity_classes_match_the_oracle():
    import torch
    from oracle.film_oracle import resize_nearest
    rng = np.random.default_rng(0)
    x = rng.standard_normal((2, 9, 11, 5)).astype(np.float32)
    k3 = rng.standard_normal((3, 3, 5, 4)).astype(np.float32)
    b = rng.standard_normal(4).astype(np.float32)
    pix = all_pixels(2, 9, 11)
    ref, S, ref1 = conv_at(Src(x), taps_3x3(k3), *pix, "fp32", "fp16")
    want = _oracle_conv(x, k3, b)
    assert np.abs(ref + b - want.reshape(-1, 4)).max() < 1e-12
    assert (S >= np.abs(ref) - 1e-12).all()
    # decoder conv_0 per parity class on the coarse grid == 2x2 SAME conv of the nearest 2x upsample (weights on a
    # 1/64 grid, so their fp32 tap sums are exact)
    xc = rng.standard_normal((1, 5, 6, 5)).astype(np.float32)
    k2 = (np.round(rng.standard_normal((2, 2, 5, 4)) * 64) / 64).astype(np.float32)
    fine = resize_nearest(torch.from_numpy(xc.astype(np.float64)).permute(0, 3, 1, 2), (10, 12))
    want = _oracle_conv(fine.permute(0, 2, 3, 1).numpy(), k2, np.zeros(4))
    fp = all_pixels(1, 10, 12)
    got = np.zeros((len(fp[0]), 4))
    for py in range(2):
        for px in range(2):
            sel = (fp[1] % 2 == py) & (fp[2] % 2 == px)
            got[sel] = conv_at(Src(xc), taps_parity(k2, py, px), fp[0][sel], fp[1][sel] // 2, fp[2][sel] // 2, "fp32",
                               "fp16")[0]
    assert np.abs(got - want.reshape(-1, 4)).max() < 1e-12


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
def test_split_emulation(fmt):
    rng = np.random.default_rng(1)
    w = (rng.standard_normal(20000) * np.exp(rng.uniform(-6, 3, 20000))).astype(np.float32)
    hi, lo = split_w(w, fmt)
    p = fmt_bits(fmt)
    if fmt == "fp16":
        np.testing.assert_array_equal(hi, w.astype(np.float16).astype(np.float64))
    else:   # round to nearest even on the top 16 bits; ties: 1 + 2^-8 -> 1, 1 + 3 * 2^-8 -> 1 + 2^-6
        assert rn(np.float32(1 + 2.0 ** -8), fmt) == 1.0 and rn(np.float32(1 + 3 * 2.0 ** -8), fmt) == 1 + 2.0 ** -6
    w64 = w.astype(np.float64)
    assert (np.abs(hi - w64) <= 2.0 ** -p * np.abs(w64) + 2.0 ** -25).all()
    assert (np.abs(hi + lo - w64) <= 2.0 ** -(2 * p - 1) * np.abs(w64) + 2.0 ** -25).all()
    # the three-pass product of split operands is fp32-grade, the single-pass one is not
    a = rng.standard_normal((1, 4, 4, 64)).astype(np.float32)
    k = rng.standard_normal((3, 3, 64, 8)).astype(np.float32) * 0.05
    ah, al = split_w(a, fmt)
    pix = all_pixels(1, 4, 4)
    exact, S, _ = conv_at(Src(a), taps_3x3(k), *pix, "fp32", fmt)
    ref3 = conv_at(Src(ah, al), taps_3x3(k), *pix, "three", fmt)[0]
    ref1 = conv_at(Src(ah, al), taps_3x3(k), *pix, "one", fmt)[0]
    assert np.abs(ref3 - exact).max() <= 4 * 2.0 ** -(2 * p - 1) * S.max()
    assert np.abs(ref1 - exact).max() > 16 * np.abs(ref3 - exact).max()


def test_sampled_pixels_cover_edges_and_tile_boundaries():
    rng = np.random.default_rng(2)
    b, y, x = sampled_pixels(2, 88, 192, rng)
    pts = set(zip(b.tolist(), y.tolist(), x.tolist()))
    assert len(pts) == len(b) >= 2000
    for bb in range(2):
        for r in (0, 1, 86, 87):
            assert all((bb, r, c) in pts for c in range(192))
        for c in (0, 1, 190, 191):
            assert all((bb, r, c) in pts for r in range(88))
    full_rows = {r for r in range(88) if all((0, r, c) in pts for c in range(192))}
    assert any(r % 8 == 7 and r + 1 in full_rows for r in full_rows if r not in (0, 1, 86, 87))


def _network_op_names():
    names = {"rgb_head", "fusion_conv2+rgb@L0"}
    for i in range(LEVELS):
        for j in range(min(LEVELS - i, spec.SUB_LEVELS)):
            r = i + j
            names |= {f"fe_conv{2 * j + 1}@L{r}"} | ({f"fe_conv0@L{r}", f"fe_conv0+pool@L{r}"} if j == 0 else
                                                    {f"fe_conv{2 * j}@L{r}"})
    for l in range(LEVELS):
        names |= {f"flow_conv{k}@L{l}" for k in range(3)} | {f"flow_conv2+head@L{l}", f"flow_head@L{l}"}
    for i in range(FUSION - 1):
        names |= {f"fusion_up@L{i}", f"fusion_conv1@L{i}", f"fusion_conv2@L{i}"} | {f"fusion_up{k}@L{i}" for k in range(4)}
    return names


def test_wiring_rules_cover_every_conv_of_the_network_and_refuse_unknown_names():
    stages = set()
    for name in _network_op_names():
        rule_of(name)
        st = op_stage(name)
        assert st is None or 0 <= st < ST_COUNT, name
        stages.add(st)
        c = consumer_stage(name)
        assert c is None or (c in range(ST_COUNT)), name
    assert set(range(ST_COUNT)) <= stages          # every stage of the plan has a conv
    for bad in ("fe_conv8@L0", "fusion_conv3@L1", "fusion_up4@L0", "flow_conv3@L2", "new_layer@L0", "fe_conv1@L"):
        with pytest.raises(AssertionError, match="no wiring rule"):
            rule_of(bad)
    # the plan's wiring: the conv pairs of the image-level-0 sub-tree have a stage each, deeper image levels share one
    assert [op_stage(f"fe_conv{k}@L{k // 2}") for k in range(8)] == [0, 0, 1, 1, 2, 2, 3, 3]
    assert op_stage("fe_conv3@L2") == fe_stage(1, 3) == 4 and op_stage("fe_conv7@L6") == 6
    assert consumer_stage("fusion_conv2@L2") == op_stage("fusion_up@L1") and consumer_stage("fusion_conv2@L0") is None
    assert consumer_stage("fe_conv0@L0") == op_stage("fe_conv1@L0") and consumer_stage("flow_conv2@L0") is None


def test_single_pass_fraction_tells_the_products_apart():
    """The discriminator on synthetic operands: a three-pass product accumulated in fp32 carries none of the single-pass
    deviation, a single-pass one all of it, one that dropped a_lo.w_hi about its share of the low-order terms."""
    rng = np.random.default_rng(3)
    a = leaky(rng.standard_normal((1, 6, 6, 256))).astype(np.float32)
    k = (rng.standard_normal((3, 3, 256, 16)) * 0.02).astype(np.float32)
    ah, al = split_w(a, "fp16")
    pix = all_pixels(1, 6, 6)
    ref3, _, ref1 = conv_at(Src(ah, al), taps_3x3(k), *pix, "three", "fp16")
    wh, wl = split_w(np.concatenate([w for _, _, w in taps_3x3(k)]), "fp16")
    cols = lambda p: np.concatenate([np.pad(p, ((0, 0), (1, 1), (1, 1), (0, 0)))[:, ky:ky + 6, kx:kx + 6]
                                     for kx in range(3) for ky in range(3)], -1).reshape(36, -1)
    A_hi, A_lo = cols(ah), cols(al)
    f32 = lambda x, y: (x.astype(np.float32) @ y.astype(np.float32)).astype(np.float64)
    fractions = {}
    for name, got in (("three", f32(A_hi, wh + wl) + f32(A_lo, wh)), ("one", f32(A_hi, wh)),
                      ("no a_lo.w_hi", f32(A_hi, wh + wl))):
        rep = Report()
        rep.single_pass_fraction("conv", name, 3, got, ref3, ref1)
        fractions[name] = rep.frac["conv"][0]
    assert abs(fractions["three"]) < FRAC_MAX / 4
    assert fractions["one"] > 4 * FRAC_MAX and abs(fractions["one"] - 1) < 0.05
    assert FRAC_MAX < fractions["no a_lo.w_hi"] < 1 - FRAC_MAX
