"""Parity tests proper: the CUDA engine (through the C ABI / Interpolator drop-in) against the
CPU oracle and the committed golden vectors. Tolerance: north_star's max-abs <= 1e-3 on the
fp32 output. Two bars below it:
  PLAN  (4e-4): the default precision plan (single-pass fp16 MMAs on the stages the measured study allows,
                tools/precision_study.py);
  TIGHT (1e-4): every conv on the three-pass split product (option onepass_mask = 0): measures 3e-5 .. 7e-5."""
import ast
import glob
import os

import numpy as np
import pytest

from frame_interpolation_b200 import spec, synthetic, weights

pytestmark = pytest.mark.gpu

TOL = 1e-3          # the contract (BASELINE.json north_star)
PLAN = 4e-4         # default precision plan
TIGHT = 1e-4        # all-three-pass engine (onepass_mask = 0)
DT = np.full((1,), 0.5, np.float32)
GOLD = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "*.npz")))


@pytest.fixture(scope="module")
def engine(synthetic_weights):
    from frame_interpolation_b200.interpolator import Interpolator
    path, _ = synthetic_weights
    eng = Interpolator(path, align=64)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def engine3(synthetic_weights):
    """Engine with every conv on the three-pass split product (fp32-grade)."""
    from frame_interpolation_b200.interpolator import Interpolator
    eng = Interpolator(synthetic_weights[0], align=64)
    eng.set_option("onepass_mask", 0)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def oracle(synthetic_weights):
    import torch
    from oracle.film_oracle import OracleInterpolator
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    return OracleInterpolator(synthetic_weights[1], align=64)


def psnr(a, b):
    return 10 * np.log10(1.0 / max(np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2), 1e-30))


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p) for p in GOLD])
def test_engine_matches_golden_vectors(path, synthetic_weights):
    from frame_interpolation_b200.interpolator import Interpolator
    z = np.load(path)
    c = dict(h=int(str(z["h"])), w=int(str(z["w"])), seed=int(str(z["seed"])), align=int(str(z["align"])),
             block=ast.literal_eval(str(z["block"])))
    assert weights.digest(synthetic_weights[1]) == str(z["weights_sha256"])
    x0, x1 = synthetic.frame_pair(c["h"], c["w"], seed=c["seed"], n_waves=6)
    eng = Interpolator(synthetic_weights[0], align=c["align"], block_shape=c["block"])
    out = eng(x0, x1, DT)
    assert out.dtype == np.float32 and out.shape == z["image"].shape
    assert np.abs(out - z["image"]).max() < PLAN
    eng.set_option("onepass_mask", 0)
    assert np.abs(eng(x0, x1, DT) - z["image"]).max() < TIGHT
    eng.close()


@pytest.mark.parametrize("h,w,seed", [(64, 64, 0), (128, 192, 1), (256, 256, 2), (192, 320, 3), (100, 150, 4), (65, 129, 5)])
def test_engine_matches_oracle(engine, engine3, oracle, h, w, seed):
    x0, x1 = synthetic.frame_pair(h, w, seed=seed, n_waves=8)
    ref = oracle(x0, x1, DT)
    for eng, tol in ((engine, PLAN), (engine3, TIGHT)):
        out = eng(x0, x1, DT)
        err = np.abs(out.astype(np.float64) - ref).max()
        assert out.shape == ref.shape == (1, h, w, 3)
        assert err < tol, err
        assert psnr(out, ref) > 80.0                 # i.e. PSNR delta vs the reference << 0.01 dB


def test_intermediate_tensors_match_oracle(engine3, oracle):
    """Stage-by-stage parity (three-pass engine): feature pyramid, residual flows, flows, warped pyramids."""
    engine = engine3
    x0, x1 = synthetic.frame_pair(128, 128, seed=9, n_waves=8)
    engine.set_option("keep_debug", 1)        # intermediates live in recycled arena blocks otherwise
    engine.interpolate(x0, x1, DT)
    engine.set_option("keep_debug", 0)
    with pytest.raises(AssertionError, match="keep_debug"):
        engine.interpolate(x0, x1, DT)        # plan without keep_debug: intermediates are recycled ...
        engine.debug_read("feat0/0")          # ... and reading one is refused, not silently stale
    engine.set_option("keep_debug", 1)
    engine.interpolate(x0, x1, DT)
    engine.set_option("keep_debug", 0)
    aux = {}
    oracle.interpolate(x0, x1, DT, aux)

    def nhwc(t):
        return t[0].permute(1, 2, 0).contiguous().numpy().reshape(-1)
    for l in range(spec.PYRAMID_LEVELS):
        for k in range(2):
            got, want = engine.debug_read(f"feat{k}/{l}"), nhwc(aux["feature_pyramids"][k][l])
            assert np.abs(got - want).max() < 1e-3 * max(1.0, np.abs(want).max())
        assert np.abs(engine.debug_read(f"res_fwd/{l}") - nhwc(aux["forward_residual_flow_pyramid"][l])).max() < 5e-4
        assert np.abs(engine.debug_read(f"res_bwd/{l}") - nhwc(aux["backward_residual_flow_pyramid"][l])).max() < 5e-4
    for l in range(spec.FUSION_PYRAMID_LEVELS):
        assert np.abs(engine.debug_read(f"flow_fwd/{l}") - nhwc(aux["forward_flow_pyramid"][l])).max() < 5e-4
        assert np.abs(engine.debug_read(f"flow_bwd/{l}") - nhwc(aux["backward_flow_pyramid"][l])).max() < 5e-4
        C = spec.feature_channels(l)
        al = aux["aligned_pyramid"][l]
        scale = max(1.0, float(al.abs().max()))
        assert np.abs(engine.debug_read(f"warped0/{l}") - nhwc(al[:, 3:3 + C])).max() < 5e-4 * scale
        assert np.abs(engine.debug_read(f"warped1/{l}") - nhwc(al[:, 6 + C:6 + 2 * C])).max() < 5e-4 * scale


def test_tensor_core_path_agrees_with_cuda_core_validation_path(synthetic_weights):
    """Same packed weights, same schedule; wgmma implicit GEMM vs fp32 FMA kernels."""
    from frame_interpolation_b200.interpolator import Interpolator
    x0, x1 = synthetic.frame_pair(128, 192, seed=11, n_waves=8)
    a = Interpolator(synthetic_weights[0], align=64)
    a.set_option("onepass_mask", 0)
    b = Interpolator(synthetic_weights[0], align=64)
    b.set_option("conv_impl", 1)
    oa, ob = a(x0, x1, DT), b(x0, x1, DT)
    assert np.abs(oa - ob).max() < 1e-4
    a.close()
    b.close()


def test_dt_value_is_ignored_and_calls_are_deterministic(engine):
    x0, x1 = synthetic.frame_pair(128, 128, seed=2, n_waves=8)
    a = engine(x0, x1, np.full((1,), 0.5, np.float32))
    b = engine(x0, x1, np.full((1,), 0.1, np.float32))
    np.testing.assert_array_equal(a, b)


def test_batch_of_pairs(engine, oracle):
    p = [synthetic.frame_pair(64, 128, seed=s, n_waves=6) for s in (0, 1, 2)]
    x0 = np.concatenate([a for a, _ in p])
    x1 = np.concatenate([b for _, b in p])
    out = engine(x0, x1, np.full((3,), 0.5, np.float32))
    assert out.shape == (3, 64, 128, 3)
    for i in range(3):
        np.testing.assert_array_equal(out[i:i + 1], engine(x0[i:i + 1], x1[i:i + 1], DT))
    assert np.abs(out - oracle(x0, x1, np.full((3,), 0.5, np.float32))).max() < PLAN


def test_tiled_path_matches_oracle_tiled_path_and_per_tile_calls(synthetic_weights):
    from frame_interpolation_b200.interpolator import Interpolator, image_to_patches
    from oracle.film_oracle import OracleInterpolator
    x0, x1 = synthetic.frame_pair(200, 300, seed=12, n_waves=8)      # tiles 100x150 -> each padded to 128x192
    eng = Interpolator(synthetic_weights[0], align=64, block_shape=[2, 2])
    out = eng(x0, x1, DT)
    ref = OracleInterpolator(synthetic_weights[1], align=64, block_shape=[2, 2])(x0, x1, DT)
    assert out.shape == (1, 200, 300, 3)
    assert np.abs(out - ref).max() < PLAN
    # seams are part of the reference behaviour: every tile equals an independent call on that tile
    single = Interpolator(synthetic_weights[0], align=64)
    p0, p1 = image_to_patches(x0, [2, 2]), image_to_patches(x1, [2, 2])
    for t in range(4):
        r, c = divmod(t, 2)
        np.testing.assert_array_equal(out[0, r * 100:(r + 1) * 100, c * 150:(c + 1) * 150],
                                      single(p0[t][None], p1[t][None], DT)[0])
    with pytest.raises(AssertionError, match="should evenly divide"):
        Interpolator(synthetic_weights[0], align=64, block_shape=[3, 2])(x0, x1, DT)
    eng.close()
    single.close()


def test_argument_errors_mirror_the_reference(engine, synthetic_weights):
    from frame_interpolation_b200.interpolator import Interpolator
    x0, x1 = synthetic.frame_pair(64, 64, seed=0, n_waves=4)
    with pytest.raises(AssertionError):
        engine(x0[0], x1[0], DT)                                  # rank 3 (eval/interpolator.py:43)
    with pytest.raises(AssertionError, match="positive"):
        Interpolator(synthetic_weights[0], align=-8)(x0, x1, DT)  # eval/interpolator.py:44
    noalign = Interpolator(synthetic_weights[0], align=None)
    assert noalign(x0, x1, DT).shape == (1, 64, 64, 3)            # already 64-aligned: fine without padding
    x0b, x1b = synthetic.frame_pair(70, 64, seed=0, n_waves=4)
    # The reference graph accepts unaligned sizes (VALID pooling floors); this engine implements the 64-aligned
    # case only and says so with FILM_ERR_UNSUPPORTED -- a capability limit, not an argument error
    with pytest.raises(RuntimeError, match="multiple of 64"):
        noalign(x0b, x1b, DT)
    noalign.close()
    with pytest.raises(RuntimeError, match="weight"):
        Interpolator("/nonexistent/weights.filmw")


def test_device_pointer_path_bitwise_equals_host_path(engine):
    import torch
    x0, x1 = synthetic.frame_pair(120, 200, seed=7, n_waves=8)
    host = engine(x0, x1, DT)
    d0, d1 = torch.from_numpy(x0).cuda(), torch.from_numpy(x1).cuda()
    out = torch.empty_like(d0)
    torch.cuda.synchronize()
    engine.interpolate_device(d0.data_ptr(), d1.data_ptr(), 1, 120, 200, out.data_ptr())
    engine.synchronize()
    np.testing.assert_array_equal(out.cpu().numpy(), host)
    # strided views: a tile of a larger device frame in, a tile of a larger frame out
    big0 = torch.zeros(1, 240, 400, 3, device="cuda")
    big1 = torch.zeros(1, 240, 400, 3, device="cuda")
    bigo = torch.zeros(1, 240, 400, 3, device="cuda")
    big0[0, 120:, 200:] = d0[0]
    big1[0, 120:, 200:] = d1[0]
    torch.cuda.synchronize()
    off = (120 * 400 + 200) * 3 * 4
    engine.interpolate_device(big0.data_ptr() + off, big1.data_ptr() + off, 1, 120, 200, bigo.data_ptr() + off,
                              in_pitch=400 * 3, out_pitch=400 * 3)
    engine.synchronize()
    np.testing.assert_array_equal(bigo[0, 120:, 200:].cpu().numpy(), host[0])
    assert float(bigo[0, :120].abs().sum()) == 0.0


def test_profile_and_op_table(engine):
    x0, x1 = synthetic.frame_pair(128, 128, seed=1, n_waves=4)
    engine(x0, x1, DT)
    p = engine.profile()
    assert p["padded_h"] == 128 and p["kernel_launches"] > 90 and p["used_graph"] == 1
    assert abs(p["conv_flops"] - 2 * spec.conv_macs(128, 128)["total"]) / p["conv_flops"] < 1e-9
    tab = engine.op_table()
    assert sum(1 for r in tab if r["category"] == 0) > 60
    # tensor-core conv FLOPs in the table = all convs but cfeat_conv_0 and the 1x1 heads
    assert 0.95 < sum(r["ref_flops"] for r in tab if r["category"] == 0) / p["conv_flops"] <= 1.0


@pytest.mark.timeout(900)
def test_full_size_1080p_parity_and_properties(synthetic_weights):
    """BASELINE.json configs[1] at full size: 1080p against the oracle, plus size-independent
    properties (tiled 1x1 == untiled, determinism, pad/crop geometry)."""
    import torch
    from frame_interpolation_b200.interpolator import Interpolator
    from oracle.film_oracle import OracleInterpolator
    x0, x1 = synthetic.frame_pair(1080, 1920, seed=0, n_waves=6)
    eng = Interpolator(synthetic_weights[0], align=64)
    out = eng(x0, x1, DT)
    assert out.shape == (1, 1080, 1920, 3) and np.isfinite(out).all()
    np.testing.assert_array_equal(out, eng(x0, x1, DT))
    np.testing.assert_array_equal(out, Interpolator(synthetic_weights[0], align=64, block_shape=[1, 1])(x0, x1, DT))
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    ref = OracleInterpolator(synthetic_weights[1], align=64)(x0, x1, DT)
    err = np.abs(out.astype(np.float64) - ref).max()
    assert err < TOL, err
    assert err < PLAN, err                 # default precision plan: 2.4e-4 measured
    assert psnr(out, ref) > 80.0
    eng.set_option("onepass_mask", 0)      # every conv three-pass: 7e-5 measured
    err3 = np.abs(eng(x0, x1, DT).astype(np.float64) - ref).max()
    assert err3 < 1.5e-4, err3
    eng.close()


def test_device_resident_recursion_equals_host_recursion(engine):
    """film_interpolate_recursive (frames stay in HBM) vs eval/util.py-style recursion through __call__."""
    from frame_interpolation_b200 import eval_util
    x0, x1 = synthetic.frame_pair(90, 160, seed=21, n_waves=6)
    seq = engine.interpolate_recursively(x0[0], x1[0], 3)
    assert seq.shape == (9, 90, 160, 3)

    def rec(a, b, n):
        if n == 0:
            return [a]
        m = engine(a[None], b[None], DT)[0]
        return rec(a, m, n - 1) + rec(m, b, n - 1)
    want = rec(x0[0], x1[0], 3) + [x1[0]]
    for got, ref in zip(seq, want):
        np.testing.assert_array_equal(got, ref)
    # the scheduling helper picks the device-resident path for the engine and yields the same frames
    frames = list(eval_util.interpolate_recursively_from_memory([x0[0], x1[0], x0[0]], 2, engine))
    assert len(frames) == 2 * 4 + 1
    np.testing.assert_array_equal(frames[2], engine(x0, x1, DT)[0])
    np.testing.assert_array_equal(frames[4], x1[0])


def test_cli_end_to_end(tmp_path, synthetic_weights):
    from frame_interpolation_b200 import eval_util, interpolator_cli, interpolator_test
    d = tmp_path / "scene"
    d.mkdir()
    x0, x1 = synthetic.frame_pair(96, 128, seed=5, n_waves=6)
    eval_util.write_image(str(d / "a1.png"), x0[0])
    eval_util.write_image(str(d / "a2.png"), x1[0])
    assert interpolator_cli.main(["--pattern", str(tmp_path / "*"), "--model_path", synthetic_weights[0],
                                  "--times_to_interpolate", "2", "--block_height", "2", "--block_width", "2"]) == 0
    out = sorted(os.listdir(d / "interpolated_frames"))
    assert out == [f"frame_{i:03d}.png" for i in range(5)]
    mid = eval_util.read_image(str(d / "interpolated_frames" / "frame_002.png"))
    assert interpolator_test.main(["--frame1", str(d / "a1.png"), "--frame2", str(d / "a2.png"), "--model_path",
                                   synthetic_weights[0], "--block_height", "2", "--block_width", "2",
                                   "--output_frame", str(tmp_path / "mid.png")]) == 0
    np.testing.assert_array_equal(mid, eval_util.read_image(str(tmp_path / "mid.png")))


@pytest.mark.parametrize("option,value", [("conv3x3_2cta", 0), ("conv3x3_2cta", 1), ("conv3x3_2cta", 2), ("conv3x3_v2", 0),
                                          ("conv3x3_halo", 0), ("conv3x3_halo", 1), ("conv3x3_halo", 2), ("conv3x3_halo", 3),
                                          ("fe_conv0_tc", 1), ("fuse_rgb_head", 0),
                                          ("mma_straight", 0), ("plane_skip", 0), ("arena_reuse", 0), ("fuse_flow_head", 0), ("fuse_flow_head", 2)])
def test_kernel_variants_agree(synthetic_weights, oracle, option, value):
    """Every conv kernel variant (generic, persistent, CTA-pair clusters on all eligible layers, wide-halo boxes off /
    pair-only / 64-channel chunks only; the default is wide halo on every persistent layer) meets the same bar."""
    from frame_interpolation_b200.interpolator import Interpolator
    x0, x1 = synthetic.frame_pair(256, 320, seed=13, n_waves=8)
    ref = oracle(x0, x1, DT)
    eng = Interpolator(synthetic_weights[0], align=64)
    eng.set_option(option, value)
    out = eng(x0, x1, DT)
    assert np.abs(out.astype(np.float64) - ref).max() < PLAN
    default = Interpolator(synthetic_weights[0], align=64)
    # same precision plan, different kernels: accumulation-order differences of ~1e-6 flip fp16 roundings inside the
    # single-pass stages, so two plan-mode results agree to the plan's own noise, not to 1e-6
    assert np.abs(out - default(x0, x1, DT)).max() < 2.5e-4
    for e in (eng, default):
        e.set_option("onepass_mask", 0)
    out3 = eng(x0, x1, DT)
    assert np.abs(out3.astype(np.float64) - ref).max() < TIGHT
    assert np.abs(out3 - default(x0, x1, DT)).max() < 5e-5
    eng.close()
    default.close()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("h,w", [(700, 1500)])
def test_streamed_weight_rings_at_wide_tile_sizes(synthetic_weights, oracle, h, w):
    """Padded 704x1536: the 256->512 / 512->512 feature convs of image level 1 (44x96, B = 2) fill one wave of SMs only
    with 4x32 tiles, where the three-pass weight taps (64 KiB each) leave room for little shared memory. Every streamed
    weight ring must still have two slots; three-pass everywhere is the tightest case."""
    from frame_interpolation_b200.interpolator import Interpolator
    x0, x1 = synthetic.frame_pair(h, w, seed=23, n_waves=8)
    eng = Interpolator(synthetic_weights[0], align=64)
    eng.set_option("onepass_mask", 0)
    out = eng(x0, x1, DT)
    eng.close()
    err = np.abs(out.astype(np.float64) - oracle(x0, x1, DT)).max()
    assert err < TIGHT, err


def test_results_live_in_distinct_pinned_buffers(engine):
    """Results are returned in pooled page-locked buffers; a buffer must never be recycled while the
    caller still holds the array (or a view of it)."""
    import gc
    a0, a1 = synthetic.frame_pair(64, 64, seed=1, n_waves=4)
    b0, b1 = synthetic.frame_pair(64, 64, seed=2, n_waves=4)
    ra = engine(a0, a1, DT)
    keep = ra.copy()
    view = ra[0, 10:20]
    rb = engine(b0, b1, DT)
    assert ra.ctypes.data != rb.ctypes.data
    np.testing.assert_array_equal(ra, keep)
    del ra
    gc.collect()
    rc = engine(b0, b1, DT)                      # the buffer behind `view` is still owned by the caller
    np.testing.assert_array_equal(view, keep[0, 10:20])
    np.testing.assert_array_equal(rc, rb)
    del view, rb, rc
    gc.collect()
    for _ in range(8):                           # steady state: buffers are recycled, results stay right
        np.testing.assert_array_equal(engine(a0, a1, DT), keep)


def test_clear_cache_drops_plans_and_results_are_reproduced(synthetic_weights):
    """Plans (CUDA graph + activation arena) are cached per shape; clear_cache() frees them and the next call
    rebuilds the plan with identical results."""
    from frame_interpolation_b200.interpolator import Interpolator
    eng = Interpolator(synthetic_weights[0], align=64)
    x0, x1 = synthetic.frame_pair(128, 192, seed=21, n_waves=8)
    y0, y1 = synthetic.frame_pair(64, 64, seed=22, n_waves=8)
    a, b = eng(x0, x1, DT).copy(), eng(y0, y1, DT).copy()
    assert eng.profile()["arena_bytes"] > 0
    eng.clear_cache()
    np.testing.assert_array_equal(eng(y0, y1, DT), b)      # same shape -> same plan -> same bits
    np.testing.assert_array_equal(eng(x0, x1, DT), a)
    eng.close()


def _flow_bias_weights(tmp_path, base, bias_xy, tag):
    """Synthetic weights whose flow predictors output a CONSTANT residual: conv_4 kernel = 0, bias = bias_xy.
    The flow pyramid is then known in closed form (v_l = 2 * up(v_{l+1}) + b) and can be made as large as wanted."""
    from frame_interpolation_b200 import weights as W
    w = {k: np.array(v, copy=True) for k, v in base.items()}
    for p in ("flow_predictor_0", "flow_predictor_1", "flow_predictor_2", "flow_predictor_shared"):
        w[f"predict_flow/{p}/conv_4/kernel"][...] = 0.0
        w[f"predict_flow/{p}/conv_4/bias"][...] = np.asarray(bias_xy, np.float32)
    path = str(tmp_path / f"flowbias_{tag}.filmw")
    W.save(path, w)
    return path, w


@pytest.mark.parametrize("bias_xy,tag", [((3.0, -2.0), "integer_landings"), ((2.75, 1.5), "twice_the_frame"),
                                         ((-0.4375, 0.3125), "fractional_negative")])
def test_warp_kernels_edge_cases(tmp_path, synthetic_weights, bias_xy, tag):
    """The gather kernels against `dense_image_warp` (models/film_net/util.py:48-82 + the TFA 0.15 rule: per axis
    floor = min(max(0, floor(q)), size - 2), alpha = clip(q - floor, 0, 1)) where a naive clamp would differ:
    flows far larger than the frame (|v_0| = 127 * |b|: 381 px on a 128 x 192 frame), integer flows landing exactly
    on pixels, on the border and on size - 1, negative coordinates; at every level, both stages (flow-stage warp by
    the upsampled flow, fusion-stage warp by 0.5 * flow). The kernels are isolated from the convs by feeding the
    ORACLE's warp with the engine's own features and flows."""
    import torch
    from frame_interpolation_b200.interpolator import Interpolator
    from oracle import film_oracle as O
    path, w = _flow_bias_weights(tmp_path, synthetic_weights[1], bias_xy, tag)
    h, wd = 128, 192
    x0, x1 = synthetic.frame_pair(h, wd, seed=31, n_waves=8)
    eng = Interpolator(path, align=64)
    eng.set_option("onepass_mask", 0)
    eng.set_option("keep_debug", 1)
    eng(x0, x1, DT)
    sizes = spec.level_sizes(h, wd)

    def t_nchw(flat, hh, ww, c):
        return torch.from_numpy(flat.reshape(1, hh, ww, c)).permute(0, 3, 1, 2).contiguous()

    # closed-form flow pyramid: v_6 = b, v_l = 2 * v_{l+1} + b  (bilinear upsampling of a constant is the constant)
    v = np.asarray(bias_xy, np.float64)
    expect = {}
    for l in reversed(range(spec.PYRAMID_LEVELS)):
        expect[l] = v.copy()
        v = 2 * v + np.asarray(bias_xy, np.float64)
    assert max(abs(expect[0])) > 30
    for l in range(spec.PYRAMID_LEVELS):
        hh, ww = sizes[l]
        C = spec.feature_channels(l)
        for name in (f"flow_fwd/{l}", f"flow_bwd/{l}"):
            got = eng.debug_read(name).reshape(hh, ww, 2)
            assert np.abs(got - expect[l].astype(np.float32)).max() <= 1e-5 * max(1.0, abs(expect[l]).max()), (name, tag)
        feats = [t_nchw(eng.debug_read(f"feat{k}/{l}"), hh, ww, C) for k in range(2)]
        fscale = max(1.0, float(max(f.abs().max() for f in feats)))
        if l < spec.PYRAMID_LEVELS - 1:
            # flow-stage warp: direction d warps the features of image 1 - d by the upsampled flow of direction d
            for d in range(2):
                vup = t_nchw(eng.debug_read(f"flow_vup{d}/{l}"), hh, ww, 2)
                want = O.warp(feats[1 - d], vup)[0].permute(1, 2, 0).reshape(-1).numpy()
                got = eng.debug_read(f"flow_warped{d}/{l}")
                assert np.abs(got - want).max() <= 1e-5 * fscale, (l, d, tag)
        if l < spec.FUSION_PYRAMID_LEVELS:
            # fusion-stage warp: image k by 0.5 * flow of direction 1 - k (interpolator.py:163-178)
            flows = [t_nchw(eng.debug_read(n), hh, ww, 2) for n in (f"flow_fwd/{l}", f"flow_bwd/{l}")]
            for k in range(2):
                want = O.warp(feats[k], 0.5 * flows[1 - k])[0].permute(1, 2, 0).reshape(-1).numpy()
                got = eng.debug_read(f"warped{k}/{l}")
                assert np.abs(got - want).max() <= 1e-5 * fscale, (l, k, tag)
    # and the whole network still matches the oracle with these weights
    ref = O.OracleInterpolator(w, align=64)(x0, x1, DT)
    assert np.abs(eng(x0, x1, DT).astype(np.float64) - ref).max() < TIGHT
    eng.close()


@pytest.mark.timeout(900)
def test_4k_tiled_2x2_at_real_tile_size(synthetic_weights):
    """BASELINE.json configs[2] at its real size: 3840x2160, block 2x2 -> four 1080x1920 tiles, each padded on its own
    to 1088x1920 (eval/interpolator.py:192-206). One tile is checked against the oracle, all four against independent
    engine calls on the tile (seams are reference behaviour), and the stitch geometry against the tile order."""
    import torch
    from frame_interpolation_b200.interpolator import Interpolator, image_to_patches
    from oracle.film_oracle import OracleInterpolator
    x0, x1 = synthetic.frame_pair(2160, 3840, seed=5, n_waves=8)
    eng = Interpolator(synthetic_weights[0], align=64, block_shape=[2, 2])
    out = eng(x0, x1, DT)
    assert out.shape == (1, 2160, 3840, 3) and np.isfinite(out).all()
    single = Interpolator(synthetic_weights[0], align=64)
    p0, p1 = image_to_patches(x0, [2, 2]), image_to_patches(x1, [2, 2])
    for t in range(4):
        r, c = divmod(t, 2)
        np.testing.assert_array_equal(out[0, r * 1080:(r + 1) * 1080, c * 1920:(c + 1) * 1920],
                                      single(p0[t][None], p1[t][None], DT)[0])
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    t = 3                                                       # bottom-right tile
    ref = OracleInterpolator(synthetic_weights[1], align=64)(p0[t][None], p1[t][None], DT)
    err = np.abs(out[0, 1080:, 1920:].astype(np.float64) - ref[0]).max()
    assert err < PLAN, err
    eng.close()
    single.close()


@pytest.mark.parametrize("h,w", [(96, 160), (65, 129)])
def test_u8_front_and_back_end_bit_identical_to_the_host_conversions(engine, h, w):
    """film_interpolate_u8 / _recursive_u8: uint8 frames cross PCIe, `/255` (eval/util.py:38-41) and
    `clip(x*255,0,255)+0.5 -> uint8` (eval/util.py:51-52) run on the device. Must equal the float path wrapped in the
    host-side conversions bit for bit (65x129: frame slots that are not 16-byte aligned take the scalar kernels)."""
    from frame_interpolation_b200 import eval_util
    x0, x1 = synthetic.frame_pair(h, w, seed=17, n_waves=8)
    u0, u1 = eval_util.to_uint8(x0), eval_util.to_uint8(x1)
    f0 = u0.astype(np.float32) / np.float32(255.0)
    f1 = u1.astype(np.float32) / np.float32(255.0)
    got = engine.interpolate_u8(u0, u1)
    assert got.dtype == np.uint8 and got.shape == u0.shape
    np.testing.assert_array_equal(got, eval_util.to_uint8(engine(f0, f1, DT)))
    seq = engine.interpolate_recursively_u8(u0[0], u1[0], 3)
    assert seq.shape == (9, h, w, 3) and seq.dtype == np.uint8
    np.testing.assert_array_equal(seq, eval_util.to_uint8(engine.interpolate_recursively(f0[0], f1[0], 3)))
    np.testing.assert_array_equal(seq[0], u0[0])
    np.testing.assert_array_equal(seq[-1], u1[0])
