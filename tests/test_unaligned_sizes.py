"""Frame sizes that are not multiples of 64 (option any_size = 1), as the reference graph runs them.

At such sizes some pyramid levels have odd heights or widths: their 2x2 pools floor (the fused pool of the persistent
3x3 conv must clip its last row / column), and a decoder level that is not exactly twice the coarser one takes the
nearest resize as a gather of its own followed by a plain 2x2 SAME conv (k_resize_nearest + fusion_up on the generic
kernel).  The CPU tests pin the oracle at such sizes; the GPU tests hold the engine to it at the bars of
test_engine_gpu.py."""
import os

import numpy as np
import pytest
import torch

from frame_interpolation_b200 import spec, synthetic, weights

PLAN = 4e-4         # default precision plan
TIGHT = 1e-4        # every conv three-pass (onepass_mask = 0)
DT = np.full((1,), 0.5, np.float32)


def _nearest_index(dst, n_in, n_out):
    """TF2 NEAREST with half-pixel centres, floor((dst + 0.5) * in / out), in exact integer arithmetic."""
    return np.minimum((2 * dst + 1) * n_in // (2 * n_out), n_in - 1)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle at odd sizes
# ---------------------------------------------------------------------------------------------------------------------
def test_independent_restatement_agrees_with_the_oracle_at_an_unaligned_size():
    from oracle.film_oracle import OracleInterpolator
    from test_oracle_independent import film   # pytest puts this directory on sys.path
    w = weights.synthetic_weights()
    x0, x1 = synthetic.frame_pair(65, 97, seed=4, n_waves=6)   # levels 65x97, 32x48, ...: odd at level 0 only
    ref = OracleInterpolator(w, align=None, dtype=torch.float64).interpolate(x0, x1, DT)[0]
    got = film(w, x0[0].astype(np.float64), x1[0].astype(np.float64))
    assert got.shape == ref.shape == (65, 97, 3)
    assert np.abs(got - ref).max() < 1e-9, np.abs(got - ref).max()


@pytest.mark.parametrize("n_in,n_out", [(3, 7), (67, 135), (17, 35), (2, 5), (5, 10)])
def test_oracle_resize_nearest_follows_the_integer_rule(n_in, n_out):
    from oracle.film_oracle import resize_nearest
    x = torch.arange(n_in * n_in, dtype=torch.float64).view(1, 1, n_in, n_in)
    got = resize_nearest(x, (n_out, n_out))[0, 0].numpy().astype(np.int64)
    idx = _nearest_index(np.arange(n_out), n_in, n_out)
    np.testing.assert_array_equal(got, idx[:, None] * n_in + idx[None, :])


def test_integer_rule_matches_float64_on_every_pyramid_ratio():
    """Every ratio a pyramid produces (out = 2 in or 2 in + 1) up to 8K: the float64 expression of the oracle and the
    integer one of the engine's k_resize_nearest pick the same source pixel."""
    for n_in in range(1, 2200):
        for n_out in (2 * n_in, 2 * n_in + 1):
            d = np.arange(n_out)
            f = np.minimum(np.floor((d.astype(np.float64) + 0.5) * (n_in / n_out)).astype(np.int64), n_in - 1)
            np.testing.assert_array_equal(f, _nearest_index(d, n_in, n_out))


def test_level_sizes_of_the_issue_shapes():
    """Which levels take the non-2x decoder path and which pooled levels are odd (align=None)."""
    def non2x(h, w):
        s = spec.level_sizes(h, w)
        return [i for i in range(spec.FUSION_PYRAMID_LEVELS - 1)
                if s[i] != (2 * s[i + 1][0], 2 * s[i + 1][1])]
    assert non2x(1080, 1920) == [3]
    assert non2x(720, 1280) == []
    assert non2x(270, 480) == [1, 2, 3]
    assert non2x(100, 150) == [1, 2]
    assert non2x(65, 129) == [0]
    assert non2x(128, 192) == []


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the engine against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def oracles(synthetic_weights):
    from oracle.film_oracle import OracleInterpolator
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    return {a: OracleInterpolator(synthetic_weights[1], align=a) for a in (None, 32)}


def _engine(synthetic_weights, align=None, onepass_mask=None, block_shape=None):
    from frame_interpolation_b200.interpolator import Interpolator
    eng = Interpolator(synthetic_weights[0], align=align, block_shape=block_shape)
    eng.set_option("any_size", 1)
    if onepass_mask is not None:
        eng.set_option("onepass_mask", onepass_mask)
    return eng


def _resize_levels(eng):
    return sorted(int(r["name"].split("@L")[1]) for r in eng.op_table() if r["name"].startswith("fusion_resize@"))


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,align,resized", [(100, 150, None, [1, 2]), (65, 129, None, [0]),
                                                (270, 480, None, [1, 2, 3]), (100, 150, 32, [])])
def test_unaligned_sizes_match_the_oracle(synthetic_weights, oracles, h, w, align, resized):
    x0, x1 = synthetic.frame_pair(h, w, seed=31, n_waves=8)
    ref = oracles[align](x0, x1, DT)
    for mask, tol in ((None, PLAN), (0, TIGHT)):
        eng = _engine(synthetic_weights, align, mask)
        try:
            out = eng(x0, x1, DT)
            assert out.shape == ref.shape == (1, h, w, 3)
            err = np.abs(out.astype(np.float64) - ref).max()
            assert err < tol, (mask, err)
            # the resize path ran exactly on the non-2x levels, with its conv on the generic kernel
            assert _resize_levels(eng) == resized
            forms = {r["name"]: r["form"] for r in eng.op_table() if r["category"] == 0}
            for i in resized:
                assert forms[f"fusion_up@L{i}"] == "tc"
            p = eng.profile()
            ph, pw, _, _ = spec.padded_shape(h, w, align)
            assert (p["padded_h"], p["padded_w"]) == (ph, pw)
            assert abs(p["conv_flops"] - 2 * spec.conv_macs(ph, pw)["total"]) / p["conv_flops"] < 1e-9
        finally:
            eng.close()


@pytest.mark.gpu
def test_pixels_on_n_pool_clips_odd_levels(synthetic_weights, oracles):
    """Every eligible 64 -> 64 layer on the pixels-on-N form, so its fused pool meets the odd levels of 100x150."""
    x0, x1 = synthetic.frame_pair(100, 150, seed=33, n_waves=8)
    ref = oracles[None](x0, x1, DT)
    eng = _engine(synthetic_weights, None, 0)
    try:
        eng.set_option("conv3x3_pxn", 2)
        out = eng(x0, x1, DT)
        forms = {r["name"]: r["form"] for r in eng.op_table() if r["category"] == 0}
        assert forms["fe_conv1@L1"] == "3x3_pxn"   # 50x75 pooled to 25x37
        assert np.abs(out.astype(np.float64) - ref).max() < TIGHT
    finally:
        eng.close()


@pytest.mark.gpu
def test_intermediate_tensors_match_oracle_at_odd_levels(synthetic_weights, oracles):
    """Three-pass engine at 100x150 (levels 100x150, 50x75, 25x37, 12x18, 6x9, 3x4, 1x2): the feature pyramid (fused
    pools on the odd levels), residual flows, flows and warped pyramids."""
    x0, x1 = synthetic.frame_pair(100, 150, seed=9, n_waves=8)
    eng = _engine(synthetic_weights, None, 0)
    try:
        eng.set_option("keep_debug", 1)
        eng.interpolate(x0, x1, DT)
        aux = {}
        oracles[None].interpolate(x0, x1, DT, aux)

        def nhwc(t):
            return t[0].permute(1, 2, 0).contiguous().numpy().reshape(-1)
        for l in range(spec.PYRAMID_LEVELS):
            for k in range(2):
                got, want = eng.debug_read(f"feat{k}/{l}"), nhwc(aux["feature_pyramids"][k][l])
                assert got.shape == want.shape
                assert np.abs(got - want).max() < 1e-3 * max(1.0, np.abs(want).max()), (k, l)
            assert np.abs(eng.debug_read(f"res_fwd/{l}") - nhwc(aux["forward_residual_flow_pyramid"][l])).max() < 5e-4
            assert np.abs(eng.debug_read(f"res_bwd/{l}") - nhwc(aux["backward_residual_flow_pyramid"][l])).max() < 5e-4
        for l in range(spec.FUSION_PYRAMID_LEVELS):
            assert np.abs(eng.debug_read(f"flow_fwd/{l}") - nhwc(aux["forward_flow_pyramid"][l])).max() < 5e-4
            assert np.abs(eng.debug_read(f"flow_bwd/{l}") - nhwc(aux["backward_flow_pyramid"][l])).max() < 5e-4
            C = spec.feature_channels(l)
            al = aux["aligned_pyramid"][l]
            scale = max(1.0, float(al.abs().max()))
            assert np.abs(eng.debug_read(f"warped0/{l}") - nhwc(al[:, 3:3 + C])).max() < 5e-4 * scale
            assert np.abs(eng.debug_read(f"warped1/{l}") - nhwc(al[:, 6 + C:6 + 2 * C])).max() < 5e-4 * scale
    finally:
        eng.close()


@pytest.mark.gpu
def test_tiled_recursive_and_u8_entries_at_unaligned_sizes(synthetic_weights):
    from frame_interpolation_b200 import eval_util
    from frame_interpolation_b200.interpolator import image_to_patches
    from oracle.film_oracle import OracleInterpolator
    x0, x1 = synthetic.frame_pair(200, 300, seed=12, n_waves=8)      # tiles of 100x150, run unpadded
    tiled = _engine(synthetic_weights, block_shape=[2, 2])
    single = _engine(synthetic_weights)
    try:
        out = tiled(x0, x1, DT)
        ref = OracleInterpolator(synthetic_weights[1], align=None, block_shape=[2, 2])(x0, x1, DT)
        assert out.shape == (1, 200, 300, 3)
        assert np.abs(out - ref).max() < PLAN
        p0, p1 = image_to_patches(x0, [2, 2]), image_to_patches(x1, [2, 2])
        for t in range(4):
            r, c = divmod(t, 2)
            np.testing.assert_array_equal(out[0, r * 100:(r + 1) * 100, c * 150:(c + 1) * 150],
                                          single(p0[t][None], p1[t][None], DT)[0])
        # device-resident recursion == recursion through __call__
        a, b = p0[0], p1[0]
        seq = single.interpolate_recursively(a, b, 2)
        assert seq.shape == (5, 100, 150, 3)

        def rec(u, v, n):
            if n == 0:
                return [u]
            m = single(u[None], v[None], DT)[0]
            return rec(u, m, n - 1) + rec(m, v, n - 1)
        for got, want in zip(seq, rec(a, b, 2) + [b]):
            np.testing.assert_array_equal(got, want)
        # 8-bit entry
        u0, u1 = eval_util.to_uint8(p0[:1]), eval_util.to_uint8(p1[:1])
        got = single.interpolate_u8(u0, u1)
        f0, f1 = (u.astype(np.float32) / np.float32(255.0) for u in (u0, u1))
        np.testing.assert_array_equal(got, eval_util.to_uint8(single(f0, f1, DT)))
    finally:
        tiled.close()
        single.close()


@pytest.mark.gpu
def test_any_size_option_semantics(synthetic_weights):
    from frame_interpolation_b200.interpolator import Interpolator
    eng = Interpolator(synthetic_weights[0], align=None)
    try:
        assert eng.get_option("any_size") == 0
        x0, x1 = synthetic.frame_pair(70, 64, seed=0, n_waves=4)
        with pytest.raises(RuntimeError, match="multiple of 64"):
            eng(x0, x1, DT)
        eng.set_option("any_size", 1)
        assert eng.get_option("any_size") == 1
        assert eng(x0, x1, DT).shape == (1, 70, 64, 3)
        # back to 0 on the same handle: the cached plan of 70x64 must not keep serving it
        eng.set_option("any_size", 0)
        with pytest.raises(RuntimeError, match="multiple of 64"):
            eng(x0, x1, DT)
        # too small even with the option: the level-5 grid would be under 2x2
        eng.set_option("any_size", 1)
        s0, s1 = synthetic.frame_pair(40, 100, seed=0, n_waves=4)
        with pytest.raises(AssertionError, match="too small"):
            eng(s0, s1, DT)
        # an aligned size runs the same plan either way
        a0, a1 = synthetic.frame_pair(128, 192, seed=3, n_waves=8)
        eng.set_option("any_size", 0)
        off = eng(a0, a1, DT).copy()
        n_off = eng.profile()["kernel_launches"]
        eng.set_option("any_size", 1)
        on = eng(a0, a1, DT)
        np.testing.assert_array_equal(on, off)
        assert eng.profile()["kernel_launches"] == n_off
        assert _resize_levels(eng) == []
    finally:
        eng.close()
