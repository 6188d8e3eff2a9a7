"""Interpolation at arbitrary times (film_interpolate_times, Interpolator.interpolate_at) and the frame-rate conversion
built on it (eval_util.retime_schedule / retime_from_files, interpolator_cli --source_fps / --target_fps).

Frame i for time t_i is the reference graph with mid_time replaced by t_i: image 0 is warped with fp32(t * bwd), image 1
with fp32((1 - t) * fwd), 1 - t an fp32 subtraction.  At t = 0.5 both products are exact halvings, so frame i must equal
the ordinary call bit for bit; that is the main check.  The time-scaled reference graph is restated here twice: as a
subclass of the CPU oracle (only `model` changes, the scaling lines) and in float64 numpy on the helpers of
test_oracle_independent.py.
"""
import os

import numpy as np
import pytest
import torch

from fractions import Fraction

from frame_interpolation_b200 import eval_util, interpolator_cli, spec, synthetic, weights
from oracle import film_oracle as fo

F = spec.FUSION_PYRAMID_LEVELS


# ---------------------------------------------------------------------------------------------------------------------
# the time-scaled reference graph
# ---------------------------------------------------------------------------------------------------------------------
def time_factors(t):
    """(t, 1 - t) as the engine forms them: fp32 t, and 1 - t as one fp32 subtraction."""
    t32 = np.float32(t)
    return t32, np.float32(np.float32(1.0) - t32)


class TimeOracle(fo.Oracle):
    """`Oracle.model` with multiply_pyramid (util.py:85-103) at mid_time = t instead of 0.5 (interpolator.py:159-161)."""

    def model(self, x0, x1, aux=None, time=None):
        if time is None:
            return super().model(x0, x1, aux)
        s0, s1 = (torch.tensor(float(s), dtype=self.dtype) for s in time_factors(time))
        img_pyr = [fo.build_image_pyramid(x0), fo.build_image_pyramid(x1)]
        feat_pyr = [self.feature_pyramid(img_pyr[0]), self.feature_pyramid(img_pyr[1])]
        fwd_flow = fo.flow_pyramid_synthesis(self.pyramid_flow(feat_pyr[0], feat_pyr[1]))[:F]
        bwd_flow = fo.flow_pyramid_synthesis(self.pyramid_flow(feat_pyr[1], feat_pyr[0]))[:F]
        backward_flow = [f * s0 for f in bwd_flow]
        forward_flow = [f * s1 for f in fwd_flow]
        to_warp = [[torch.cat([img_pyr[k][l], feat_pyr[k][l]], dim=1) for l in range(F)] for k in range(2)]
        fwd_warped = [fo.warp(t, f) for t, f in zip(to_warp[0], backward_flow)]
        bwd_warped = [fo.warp(t, f) for t, f in zip(to_warp[1], forward_flow)]
        aligned = [torch.cat([a, b, c, d], dim=1)
                   for a, b, c, d in zip(fwd_warped, bwd_warped, backward_flow, forward_flow)]
        return self.fusion(aligned)[:, :3]


class TimeOracleInterpolator(fo.OracleInterpolator):
    def __init__(self, w, align=None, dtype=torch.float32):
        super().__init__(w, align, dtype=dtype)
        self._oracle = TimeOracle(w, dtype)

    def interpolate_at(self, x0, x1, times):
        """(H, W, 3) frames -> (n, H, W, 3), frame i at times[i]."""
        a, b = x0[np.newaxis], x1[np.newaxis]
        if self._align is not None:
            a, (oh, ow, h, w) = fo.pad_to_align(a, self._align)
            b, _ = fo.pad_to_align(b, self._align)
        t0 = torch.from_numpy(np.ascontiguousarray(a)).to(self._oracle.dtype).permute(0, 3, 1, 2)
        t1 = torch.from_numpy(np.ascontiguousarray(b)).to(self._oracle.dtype).permute(0, 3, 1, 2)
        outs = []
        with torch.no_grad():
            for t in times:
                o = self._oracle.model(t0, t1, time=t).permute(0, 2, 3, 1).numpy()[0]
                outs.append(o[oh:oh + h, ow:ow + w] if self._align is not None else o)
        return np.stack(outs)


def film_at_numpy(w, x0, x1, t):
    """test_oracle_independent.film with the fusion flows scaled by (t, 1 - t): float64 numpy throughout."""
    import test_oracle_independent as ind
    g = lambda n: (w[n + "/kernel"].astype(np.float64), w[n + "/bias"].astype(np.float64))
    L = spec.PYRAMID_LEVELS

    def pyramid(im):
        p = [im]
        for _ in range(L - 1):
            p.append(ind.pool(p[-1]))
        return p

    def subtree(im, n):
        out, head = [], im
        for i in range(n):
            head = ind.conv_same(head, *g(f"feat_net/sub_extractor/cfeat_conv_{2 * i}"), True)
            head = ind.conv_same(head, *g(f"feat_net/sub_extractor/cfeat_conv_{2 * i + 1}"), True)
            out.append(head)
            if i < n - 1:
                head = ind.pool(head)
        return out

    def features(pyr):
        subs = [subtree(pyr[i], min(L - i, spec.SUB_LEVELS)) for i in range(L)]
        return [np.concatenate([subs[i - j][j] for j in range(min(i, spec.SUB_LEVELS - 1) + 1)], axis=-1) for i in range(L)]

    def predict(level, a, b):
        name = spec.FLOW_PREDICTOR_NAMES[min(level, spec.SPECIALIZED_LEVELS)]
        net = np.concatenate([a, b], axis=-1)
        for k in range(4):
            net = ind.conv_same(net, *g(f"predict_flow/{name}/conv_{k}"), True)
        return ind.conv_same(net, *g(f"predict_flow/{name}/conv_4"), False)

    def flows(fa, fb):
        v = predict(L - 1, fa[-1], fb[-1])
        out = [v]
        for i in range(L - 2, -1, -1):
            v = ind.resize_bilinear(2.0 * v, *fa[i].shape[:2])
            v = predict(i, fa[i], ind.warp(fb[i], v)) + v
            out.append(v)
        return out[::-1]

    s0, s1 = (float(s) for s in time_factors(t))
    p0, p1 = pyramid(x0), pyramid(x1)
    f0, f1 = features(p0), features(p1)
    fwd, bwd = flows(f0, f1), flows(f1, f0)
    aligned = []
    for l in range(F):
        b, f = s0 * bwd[l], s1 * fwd[l]
        aligned.append(np.concatenate([ind.warp(np.concatenate([p0[l], f0[l]], axis=-1), b),
                                       ind.warp(np.concatenate([p1[l], f1[l]], axis=-1), f), b, f], axis=-1))
    net = aligned[-1]
    for i in range(F - 2, -1, -1):
        net = ind.resize_nearest(net, *aligned[i].shape[:2])
        net = ind.conv_same(net, *g(f"fusion/level_{i}/conv_0"), False)
        net = np.concatenate([aligned[i], net], axis=-1)
        net = ind.conv_same(net, *g(f"fusion/level_{i}/conv_1"), True)
        net = ind.conv_same(net, *g(f"fusion/level_{i}/conv_2"), True)
    return ind.conv_same(net, *g("fusion/output_conv"), False)


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_oracle_at_half_is_the_oracle():
    w = weights.synthetic_weights()
    x0, x1 = synthetic.frame_pair(64, 64, seed=4, n_waves=6)
    want = fo.OracleInterpolator(w, align=64).interpolate(x0, x1, np.full((1,), 0.5, np.float32))[0]
    got = TimeOracleInterpolator(w, align=64).interpolate_at(x0[0], x1[0], [0.5])[0]
    assert np.array_equal(got, want)


def test_oracle_at_time_matches_float64_numpy():
    w = weights.synthetic_weights()
    x0, x1 = synthetic.frame_pair(64, 64, seed=4, n_waves=6)
    ref = TimeOracleInterpolator(w, align=64, dtype=torch.float64).interpolate_at(x0[0], x1[0], [0.3])[0]
    got = film_at_numpy(w, x0[0].astype(np.float64), x1[0].astype(np.float64), 0.3)
    assert np.abs(got - ref).max() < 1e-9, np.abs(got - ref).max()
    half = TimeOracleInterpolator(w, align=64, dtype=torch.float64).interpolate_at(x0[0], x1[0], [0.5])[0]
    assert np.abs(half - ref).max() > 1e-6   # the time reaches the output


def test_time_factors_are_fp32():
    assert time_factors(0.5) == (np.float32(0.5), np.float32(0.5))
    t, s = time_factors(0.3)
    assert t.dtype == np.float32 and s == np.float32(0.7) and float(s) != 0.7


def _ts(sched):
    return [t for _, t in sched]


def test_retime_schedule_exact_fractions():
    s = eval_util.retime_schedule(4, 24, 60)            # 3 s of 24 fps -> floor(3 * 60 / 24) + 1 = 8 frames
    assert s == [(0, 0), (0, Fraction(2, 5)), (0, Fraction(4, 5)), (1, Fraction(1, 5)), (1, Fraction(3, 5)),
                 (2, 0), (2, Fraction(2, 5)), (2, Fraction(4, 5))]
    assert all(isinstance(t, Fraction) for t in _ts(s))
    s = eval_util.retime_schedule(5, "30", "60")
    assert s == [(i // 2, Fraction(i % 2, 2)) for i in range(9)] and s[-1] == (4, 0)
    s = eval_util.retime_schedule(6, 25, 30)             # pos = j * 5 / 6
    assert _ts(s) == [Fraction(0), Fraction(5, 6), Fraction(2, 3), Fraction(1, 2), Fraction(1, 3), Fraction(1, 6),
                      Fraction(0)]
    assert [i for i, _ in s] == [0, 0, 1, 2, 3, 4, 5]
    s = eval_util.retime_schedule(6, 60, 24)             # pos = j * 5 / 2: every other input pair is skipped
    assert s == [(0, 0), (2, Fraction(1, 2)), (5, 0)]
    s = eval_util.retime_schedule(4, "24000/1001", 60)   # pos = j * 400 / 1001
    assert len(s) == 3 * 1001 // 400 + 1
    for j, (i, t) in enumerate(s):
        pos = Fraction(j * 400, 1001)
        assert i == pos.numerator // pos.denominator and t == pos - i and 0 <= t < 1
    assert eval_util.retime_schedule(1, 24, 60) == [(0, 0)]
    with pytest.raises(AssertionError):
        eval_util.retime_schedule(3, 0, 60)


class StandIn:
    """interpolate_at stand-in: the linear blend plus an offset, one record per call."""

    def __init__(self):
        self.calls = []

    def interpolate_at(self, a, b, times):
        self.calls.append(list(times))
        return np.stack([np.float32(1 - t) * a + np.float32(t) * b + np.float32(0.125) for t in times]).astype(np.float32)

    def __call__(self, x0, x1, dt):
        return self.interpolate_at(x0[0], x1[0], [0.5])


def _clip(tmp_path, n, h=8, w=8):
    d = tmp_path / "clip"
    d.mkdir()
    rng = np.random.default_rng(1)
    for i in range(n):
        eval_util.write_image(str(d / f"im{i}.png"), rng.random((h, w, 3)).astype(np.float32))
    return d, [str(d / f"im{i}.png") for i in range(n)]


def test_retime_calls_once_per_pair_that_needs_frames(tmp_path):
    _, names = _clip(tmp_path, 6)
    s = StandIn()
    frames = list(eval_util.retime_from_files(names, 60, 24, s))
    assert len(frames) == 3 and s.calls == [[0.5]]       # pairs 0, 1, 3, 4 need nothing
    np.testing.assert_array_equal(frames[0], eval_util.read_image(names[0]))
    np.testing.assert_array_equal(frames[2], eval_util.read_image(names[5]))
    s = StandIn()
    frames = list(eval_util.retime_from_files(names[:4], 24, 60, s))
    assert s.calls == [[0.4, 0.8], [0.2, 0.6], [0.4, 0.8]] and len(frames) == 8
    a, b = eval_util.read_image(names[1]), eval_util.read_image(names[2])
    np.testing.assert_array_equal(frames[3], s.interpolate_at(a, b, [0.2])[0])
    np.testing.assert_array_equal(frames[5], eval_util.read_image(names[2]))


def test_retime_30_to_60_is_one_recursion(tmp_path):
    _, names = _clip(tmp_path, 3)
    got = list(eval_util.retime_from_files(names, 30, 60, StandIn()))
    want = list(eval_util.interpolate_recursively_from_files(names, 1, StandIn()))
    assert len(got) == len(want) == 5
    for a, b in zip(got, want):
        np.testing.assert_array_equal(a, b)


def test_cli_retime_flags(tmp_path):
    a = interpolator_cli.build_parser().parse_args(["--pattern", "x", "--model_path", "m", "--source_fps", "24000/1001",
                                                    "--target_fps", "60"])
    assert eval_util.parse_rate(a.source_fps) == Fraction(24000, 1001) and eval_util.parse_rate(a.target_fps) == 60
    a = interpolator_cli.build_parser().parse_args(["--pattern", "x", "--model_path", "m"])
    assert a.source_fps is None and a.target_fps is None
    with pytest.raises(SystemExit):
        interpolator_cli.main(["--pattern", str(tmp_path), "--model_path", "m", "--source_fps", "24"])
    with pytest.raises(SystemExit):
        interpolator_cli.main(["--pattern", str(tmp_path), "--model_path", "m", "--source_fps", "24", "--target_fps",
                               "60", "--block_height", "2"])


def test_retime_directory_with_stand_in(tmp_path):
    d, names = _clip(tmp_path, 3)
    n = interpolator_cli.retime_directory(str(d), StandIn(), 24, 60, video=False)
    assert n == 6   # positions 0, 0.4, 0.8, 1.2, 1.6, 2
    out = sorted(os.listdir(d / "interpolated_frames"))
    assert out == [f"frame_{i:03d}.png" for i in range(6)]
    np.testing.assert_array_equal(eval_util.read_image(str(d / "interpolated_frames" / "frame_000.png")),
                                  eval_util.read_image(names[0]))


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _engine(path, align=64, **opts):
    from frame_interpolation_b200.interpolator import Interpolator
    eng = Interpolator(path, align=align)
    if align is None:
        eng.set_option("any_size", 1)
    for k, v in opts.items():
        eng.set_option(k, v)
    return eng


HALF_CASES = [(128, 128, 64, {}), (128, 128, 64, {"onepass_mask": 0}), (67, 95, None, {}), (67, 95, None, {"onepass_mask": 0})]


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,align,opts", HALF_CASES)
def test_half_is_the_ordinary_call(synthetic_weights, h, w, align, opts):
    x0, x1 = synthetic.frame_pair(h, w, seed=5)
    eng = _engine(synthetic_weights[0], align, **opts)
    try:
        want = np.array(eng(x0, x1, np.full((1,), 0.5, np.float32))[0])
        got = np.array(eng.interpolate_at(x0[0], x1[0], [0.5]))
        assert got.shape == (1, h, w, 3) and np.array_equal(got[0], want)
        got = np.array(eng.interpolate_at(x0[0], x1[0], [0.3, 0.5, 0.9, 0.5]))
        assert np.array_equal(got[1], want) and np.array_equal(got[3], want)
        alone = np.array(eng.interpolate_at(x0[0], x1[0], [0.3]))[0]
        assert np.array_equal(got[0], alone)          # no tail replay clobbers what the head left for the next one
        assert not np.array_equal(got[0], want) and not np.array_equal(got[2], got[0])
        again = np.array(eng(x0, x1, np.full((1,), 0.5, np.float32))[0])
        assert np.array_equal(again, want)            # the ordinary plan's scalar still holds 0.5
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("opts", [{"use_graph": 0}, {"use_lanes": 1}, {"time_ops": 1}, {"keep_debug": 1}])
def test_schedules_agree_bit_for_bit(synthetic_weights, opts):
    x0, x1 = synthetic.frame_pair(128, 192, seed=6)
    times = [0.25, 0.5, 0.8]
    ref = _engine(synthetic_weights[0])
    eng = _engine(synthetic_weights[0], **opts)
    try:
        want = np.array(ref.interpolate_at(x0[0], x1[0], times))
        assert ref.profile()["used_graph"] == 1
        got = np.array(eng.interpolate_at(x0[0], x1[0], times))
        assert np.array_equal(got[1], eng(x0, x1, np.full((1,), 0.5, np.float32))[0]), opts
        if not opts.get("use_lanes"):   # lanes pool the image pyramid in kernels of its own
            assert np.array_equal(got, want), opts
        if opts.get("time_ops"):
            table = eng.op_table()
            assert all(r["ms"] >= 0 for r in table) and len({r["name"] for r in table if r["name"]}) > 10
    finally:
        ref.close()
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("onepass_mask,tol", [(0, 1e-4), (None, 4e-4)])
def test_against_the_oracle(synthetic_weights, onepass_mask, tol):
    path, w = synthetic_weights
    x0, x1 = synthetic.frame_pair(120, 180, seed=3, n_waves=8)
    times = [0.25, 0.3, 0.8]
    eng = _engine(path, **({} if onepass_mask is None else {"onepass_mask": onepass_mask}))
    try:
        got = np.array(eng.interpolate_at(x0[0], x1[0], times)).astype(np.float64)
    finally:
        eng.close()
    ref = TimeOracleInterpolator(w, align=64).interpolate_at(x0[0], x1[0], times)
    err = np.abs(got - ref).max(axis=(1, 2, 3))
    print("max-abs vs oracle per time:", err)
    assert (err <= tol).all(), err


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,align", [(128, 192, 64), (67, 95, None)])
def test_fusion_gathers_of_the_last_time(synthetic_weights, h, w, align):
    """keep_debug: every fusion_warp@L<l> / fusion_side@L<l> of the last time against a float64 restatement built on
    the fp32-rounded t * bwd and (1 - t) * fwd, with the taps of test_gather_ops (bit-exact fp32 positions)."""
    from test_gather_ops import K_GATHER, ULP, ratios, warp_at
    from test_conv_layers import split_w, fmt_bits
    x0, x1 = synthetic.frame_pair(h, w, seed=8)
    t = 0.3
    s0, s1 = time_factors(t)
    eng = _engine(synthetic_weights[0], align, keep_debug=1)
    try:
        eng.interpolate_at(x0[0], x1[0], [0.9, t])
        fmt = "fp16" if "split=fp16" in eng.version else "bf16"
        p = fmt_bits(fmt)
        ph, pw, _, _ = spec.padded_shape(h, w, align)
        ops = {r["name"] for r in eng.op_table()}
        for l in range(F):
            assert f"fusion_warp@L{l}" in ops and f"fusion_side@L{l}" in ops
            H, W = ph >> l, pw >> l
            C = spec.feature_channels(l)
            rd = lambda n, shape: eng.debug_read(n).reshape(shape)
            fwd, bwd = rd(f"flow_fwd/{l}", (H, W, 2)), rd(f"flow_bwd/{l}", (H, W, 2))
            scaled = [(bwd * s0).astype(np.float32), (fwd * s1).astype(np.float32)]   # k = 0: image 0 by t * bwd
            y, x = np.divmod(np.arange(H * W), W)
            # side tensor: channels 6-9 bit for bit, 10-63 zero, 0-5 the warped images
            hi, lo = rd(f"out:fusion_side@L{l}.hi", (H, W, 64)), rd(f"out:fusion_side@L{l}.lo", (H, W, 64))
            for c, f in ((6, scaled[0]), (8, scaled[1])):
                wh, wl = split_w(f, fmt)
                assert np.array_equal(hi[..., c:c + 2], wh) and np.array_equal(lo[..., c:c + 2], wl), (l, c)
            assert not hi[..., 10:].any() and not lo[..., 10:].any()
            img = rd(f"img/{l}", (2, H, W, 3))
            for k in range(2):
                got = (hi + lo)[y, x, 3 * k:3 * k + 3].astype(np.float64)
                ref, M = warp_at(img[k], y, x, scaled[k][y, x])
                bound = K_GATHER * ULP * M + 2.0 ** -(2 * p - 1) * np.abs(ref) + 2.0 ** -25
                r = ratios(got, ref, bound)
                assert np.isfinite(got).all() and r.max() <= 1.0, (l, k, r.max())
                # features: hi-only destinations read and write the hi planes alone
                dh, dl = rd(f"warped{k}/{l}.hi", (H, W, C)), rd(f"warped{k}/{l}.lo", (H, W, C))
                hi_only = not dl.any()
                src = rd(f"feat{k}/{l}.hi", (H, W, C))
                if not hi_only:
                    src = src + rd(f"feat{k}/{l}.lo", (H, W, C))
                got = (dh + dl)[y, x].astype(np.float64)
                ref, M = warp_at(src, y, x, scaled[k][y, x])
                eps = 2.0 ** -p if hi_only else 2.0 ** -(2 * p - 1)
                r = ratios(got, ref, K_GATHER * ULP * M + eps * np.abs(ref) + 2.0 ** -25)
                assert np.isfinite(got).all() and r.max() <= 1.0, (l, k, hi_only, r.max())
    finally:
        eng.close()


@pytest.mark.gpu
def test_device_path_equals_host_path_on_pitched_views(synthetic_weights):
    h, w = 128, 192
    x0, x1 = synthetic.frame_pair(h, w, seed=9)
    times = [0.1, 0.5, 0.7]
    eng = _engine(synthetic_weights[0])
    try:
        want = np.array(eng.interpolate_at(x0[0], x1[0], times))
        pad_in, pad_out = 21, 9
        big = torch.zeros((2, h, w * 3 + pad_in), dtype=torch.float32, device="cuda")
        big[0, :, :w * 3] = torch.from_numpy(x0[0].reshape(h, w * 3))
        big[1, :, :w * 3] = torch.from_numpy(x1[0].reshape(h, w * 3))
        out = torch.full((len(times), h, w * 3 + pad_out), -7.0, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        eng.interpolate_at_device(big[0].data_ptr(), big[1].data_ptr(), times, h, w, out.data_ptr(),
                                  in_pitch=w * 3 + pad_in, out_pitch=w * 3 + pad_out)
        eng.synchronize()
        got = out.cpu().numpy()
        assert np.array_equal(got[:, :, :w * 3].reshape(len(times), h, w, 3), want)
        assert (got[:, :, w * 3:] == -7.0).all()
        assert eng.profile()["last_call_ms"] > 0
    finally:
        eng.close()


@pytest.mark.gpu
def test_argument_errors(synthetic_weights):
    x0, x1 = synthetic.frame_pair(64, 64, seed=1)
    eng = _engine(synthetic_weights[0])
    try:
        for bad, idx in (([], None), ([0.2, -0.1], 1), ([1.5], 0), ([0.5, 0.5, float("nan")], 2), ([float("inf")], 0)):
            with pytest.raises(AssertionError) as e:
                eng.interpolate_at(x0[0], x1[0], bad)
            if idx is not None:
                assert f"times[{idx}]" in str(e.value)
        assert np.array(eng.interpolate_at(x0[0], x1[0], [0.0, 1.0])).shape == (2, 64, 64, 3)
    finally:
        eng.close()
    from frame_interpolation_b200.interpolator import Interpolator
    tiled = Interpolator(synthetic_weights[0], align=64, block_shape=[2, 1])
    try:
        with pytest.raises(AssertionError):
            tiled.interpolate_at(x0[0], x1[0], [0.5])
    finally:
        tiled.close()


@pytest.mark.gpu
def test_profile_and_arena(synthetic_weights):
    h, w = 128, 192
    x0, x1 = synthetic.frame_pair(h, w, seed=2)
    dt = np.full((1,), 0.5, np.float32)
    fresh = _engine(synthetic_weights[0])
    eng = _engine(synthetic_weights[0])
    try:
        fresh(x0, x1, dt)
        p_fresh = fresh.profile()
        n_ops = len(fresh.op_table())
        for n in (1, 4):
            eng.interpolate_at(x0[0], x1[0], np.linspace(0.1, 0.9, n))
            p = eng.profile()
            m = spec.conv_macs(h, w)
            assert p["conv_flops"] == pytest.approx(2 * (m["feature_extractor"] + m["flow"] + n * m["fusion"]), rel=1e-12)
            table = eng.op_table()
            tail = len(table) - [r["name"] for r in table].index("fusion_warp@L0")
            assert len(table) == n_ops and p["kernel_launches"] == len(table) - tail + n * tail
            assert p["arena_bytes"] > p_fresh["arena_bytes"]   # the feature levels stay pinned
        eng(x0, x1, dt)
        p = eng.profile()
        assert p["arena_bytes"] == p_fresh["arena_bytes"] and p["kernel_launches"] == p_fresh["kernel_launches"]
        assert p["conv_flops"] == p_fresh["conv_flops"]
    finally:
        fresh.close()
        eng.close()


@pytest.mark.gpu
def test_cli_retime_end_to_end(tmp_path, synthetic_weights):
    d = tmp_path / "clip"
    d.mkdir()
    x0, x1 = synthetic.frame_pair(64, 96, seed=3)
    x2, _ = synthetic.frame_pair(64, 96, seed=4)
    for i, f in enumerate((x0[0], x1[0], x2[0])):
        eval_util.write_image(str(d / f"f{i}.png"), f)
    rc = interpolator_cli.main(["--pattern", str(d), "--model_path", synthetic_weights[0], "--source_fps", "24",
                                "--target_fps", "60"])
    assert rc == 0
    out = sorted(os.listdir(d / "interpolated_frames"))
    assert out == [f"frame_{i:03d}.png" for i in range(6)]   # positions 0, 0.4, 0.8, 1.2, 1.6, 2
    rd = lambda p: eval_util.read_image(str(p))
    np.testing.assert_array_equal(rd(d / "interpolated_frames" / "frame_000.png"), rd(d / "f0.png"))
    np.testing.assert_array_equal(rd(d / "interpolated_frames" / "frame_005.png"), rd(d / "f2.png"))
    assert not np.array_equal(rd(d / "interpolated_frames" / "frame_001.png"), rd(d / "f0.png"))
    from frame_interpolation_b200.interpolator import Interpolator
    eng = Interpolator(synthetic_weights[0], align=64)
    try:
        a, b = rd(d / "f1.png"), rd(d / "f2.png")
        want = eval_util.to_uint8(np.array(eng.interpolate_at(a, b, [np.float32(0.2)]))[0])
        np.testing.assert_array_equal(eval_util.to_uint8(rd(d / "interpolated_frames" / "frame_003.png")), want)
    finally:
        eng.close()
