"""Closed-form checks of the third-party op semantics the oracle restates (TF SAME / VALID padding, half-pixel bilinear
and NEAREST resize, TFA dense_image_warp with its border clamp, concat orders). CPU only."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import film_oracle as fo


def test_conv_same_3x3_identity_kernel():
    x = torch.randn(1, 2, 5, 7)
    k = torch.zeros(3, 3, 2, 2)
    k[1, 1, 0, 0] = 1.0
    k[1, 1, 1, 1] = 1.0
    y = fo.conv2d_same(x, k, torch.zeros(2), activation=False)
    assert torch.equal(y, x)


def test_conv_same_2x2_pads_bottom_right_only():
    # TF SAME with an even kernel puts the extra pixel AFTER: out[y,x] = sum_k w[ky,kx] * in[y+ky, x+kx]
    x = torch.arange(12, dtype=torch.float32).view(1, 1, 3, 4)
    k = torch.zeros(2, 2, 1, 1)
    k[1, 1, 0, 0] = 1.0   # picks in[y+1, x+1]
    y = fo.conv2d_same(x, k, torch.zeros(1), activation=False)
    want = torch.zeros_like(x)
    want[..., :2, :3] = x[..., 1:, 1:]
    assert torch.equal(y, want)
    k = torch.zeros(2, 2, 1, 1)
    k[0, 0, 0, 0] = 1.0   # picks in[y, x]: no shift, nothing padded on top/left
    assert torch.equal(fo.conv2d_same(x, k, torch.zeros(1), False), x)


def test_conv_matches_manual_loops():
    rng = np.random.default_rng(0)
    x = rng.standard_normal((1, 3, 4, 5)).astype(np.float32)
    k = rng.standard_normal((3, 3, 3, 2)).astype(np.float32)
    b = rng.standard_normal(2).astype(np.float32)
    y = fo.conv2d_same(torch.from_numpy(x), torch.from_numpy(k), torch.from_numpy(b), True).numpy()
    xp = np.pad(x, ((0, 0), (0, 0), (1, 1), (1, 1)))
    want = np.zeros((1, 2, 4, 5), np.float64)
    for o in range(2):
        for yy in range(4):
            for xx in range(5):
                acc = b[o]
                for ky in range(3):
                    for kx in range(3):
                        for c in range(3):
                            acc += xp[0, c, yy + ky, xx + kx] * k[ky, kx, c, o]
                want[0, o, yy, xx] = acc if acc >= 0 else 0.2 * acc
    np.testing.assert_allclose(y, want, rtol=1e-5, atol=1e-5)


def test_leaky_relu_slope():
    x = torch.tensor([-2.0, -0.0, 0.0, 3.0])
    assert torch.equal(fo.leaky_relu(x), torch.tensor([-0.4, -0.0, 0.0, 3.0]))


def test_avg_pool_drops_odd_row_and_col():
    x = torch.arange(35, dtype=torch.float32).view(1, 1, 5, 7)
    y = fo.avg_pool_2x2(x)
    assert y.shape == (1, 1, 2, 3)
    assert y[0, 0, 0, 0] == (0 + 1 + 7 + 8) / 4
    assert torch.allclose(y, F.avg_pool2d(x, 2, 2))


def test_image_pyramid_levels():
    pyr = fo.build_image_pyramid(torch.rand(1, 3, 128, 192))
    assert [tuple(p.shape[-2:]) for p in pyr] == [(128, 192), (64, 96), (32, 48), (16, 24), (8, 12), (4, 6), (2, 3)]


def test_resize_bilinear_2x_half_pixel_centres():
    x = torch.tensor([[0.0, 1.0, 2.0, 3.0]]).view(1, 1, 1, 4).repeat(1, 1, 2, 1)
    y = fo.resize_bilinear(x, (4, 8))
    # src = (dst + .5)/2 - .5 -> -0.25, .25, .75, 1.25, ... clamped at the borders
    want = torch.tensor([0.0, 0.25, 0.75, 1.25, 1.75, 2.25, 2.75, 3.0])
    assert torch.allclose(y[0, 0, 0], want)
    z = torch.rand(2, 3, 5, 6)
    assert torch.allclose(fo.resize_bilinear(z, (10, 12)),
                          F.interpolate(z, size=(10, 12), mode="bilinear", align_corners=False), atol=1e-6)


def test_resize_bilinear_general_ratio_against_formula():
    z = torch.rand(1, 1, 3, 5, dtype=torch.float64)
    out = fo.resize_bilinear(z, (7, 9))
    for oy in range(7):
        for ox in range(9):
            sy, sx = (oy + 0.5) * 3 / 7 - 0.5, (ox + 0.5) * 5 / 9 - 0.5
            y0, x0 = max(int(np.floor(sy)), 0), max(int(np.floor(sx)), 0)
            y1, x1 = min(int(np.ceil(sy)), 2), min(int(np.ceil(sx)), 4)
            wy, wx = sy - np.floor(sy), sx - np.floor(sx)
            top = z[0, 0, y0, x0] + (z[0, 0, y0, x1] - z[0, 0, y0, x0]) * wx
            bot = z[0, 0, y1, x0] + (z[0, 0, y1, x1] - z[0, 0, y1, x0]) * wx
            assert abs(float(out[0, 0, oy, ox]) - float(top + (bot - top) * wy)) < 1e-12


def test_resize_nearest_2x_is_repeat():
    z = torch.rand(1, 2, 3, 4)
    y = fo.resize_nearest(z, (6, 8))
    assert torch.equal(y, z.repeat_interleave(2, 2).repeat_interleave(2, 3))


def test_warp_zero_flow_is_identity():
    img = torch.rand(1, 4, 6, 7)
    out = fo.warp(img, torch.zeros(1, 2, 6, 7))
    assert torch.allclose(out, img)


def test_warp_integer_shift_and_axis_order():
    # flow channel 0 is x, channel 1 is y: out[y,x] = img[y + fy, x + fx]
    img = torch.arange(30, dtype=torch.float32).view(1, 1, 5, 6)
    flow = torch.zeros(1, 2, 5, 6)
    flow[:, 0] = 1.0   # x + 1
    out = fo.warp(img, flow)
    assert torch.equal(out[..., :, :5], img[..., :, 1:])
    assert torch.equal(out[..., :, 5], img[..., :, 5])          # clamped at the right border
    flow = torch.zeros(1, 2, 5, 6)
    flow[:, 1] = -2.0  # y - 2
    out = fo.warp(img, flow)
    assert torch.equal(out[..., 2:, :], img[..., :3, :])
    assert torch.equal(out[..., 0, :], img[..., 0, :])          # clamped at the top border


def test_warp_matches_grid_sample_border_align_corners():
    torch.manual_seed(0)
    img = torch.rand(2, 3, 9, 11)
    flow = 6.0 * torch.randn(2, 2, 9, 11)      # includes far out-of-bounds queries
    out = fo.warp(img, flow)
    gy, gx = torch.meshgrid(torch.arange(9.0), torch.arange(11.0), indexing="ij")
    qx = (gx + flow[:, 0]) * 2 / (11 - 1) - 1
    qy = (gy + flow[:, 1]) * 2 / (9 - 1) - 1
    ref = F.grid_sample(img, torch.stack([qx, qy], -1), mode="bilinear", padding_mode="border", align_corners=True)
    assert torch.allclose(out, ref, atol=2e-5)


def test_flow_synthesis_equals_estimator_accumulation():
    torch.manual_seed(1)
    res = [torch.randn(1, 2, 8 >> l if (8 >> l) else 1, 8 >> l if (8 >> l) else 1) for l in range(3)]
    res = [torch.randn(1, 2, 16, 16), torch.randn(1, 2, 8, 8), torch.randn(1, 2, 4, 4)]
    pyr = fo.flow_pyramid_synthesis(res)
    v = res[2]
    assert torch.equal(pyr[2], v)
    v = res[1] + fo.resize_bilinear(2 * v, (8, 8))
    assert torch.equal(pyr[1], v)
    v = res[0] + fo.resize_bilinear(2 * v, (16, 16))
    assert torch.equal(pyr[0], v)


def test_pad_to_align_centres_with_floor_offset():
    x = np.ones((1, 1080, 1920, 3), np.float32)
    p, (oh, ow, h, w) = fo.pad_to_align(x, 64)
    assert p.shape == (1, 1088, 1920, 3) and (oh, ow, h, w) == (4, 0, 1080, 1920)
    assert p[0, :4].sum() == 0 and p[0, 1084:].sum() == 0 and p[0, 4:1084].min() == 1
    x = np.ones((1, 5, 7, 3), np.float32)
    p, (oh, ow, h, w) = fo.pad_to_align(x, 4)
    assert p.shape == (1, 8, 8, 3) and (oh, ow) == (1, 0)       # 3 // 2 = 1, 1 // 2 = 0
    with pytest.raises(AssertionError):
        fo.pad_to_align(np.ones((5, 7, 3), np.float32), 4)
    with pytest.raises(AssertionError):
        fo.pad_to_align(x, 0)


def test_patches_round_trip_and_tile_order():
    img = np.arange(1 * 4 * 6 * 3, dtype=np.float32).reshape(1, 4, 6, 3)
    p = fo.image_to_patches(img, [2, 3])
    assert p.shape == (6, 2, 2, 3)
    # tile index r * bw + c, tile (r,c)[i,j] = image[r*ph + i, c*pw + j]
    np.testing.assert_array_equal(p[4], img[0, 2:4, 2:4])
    np.testing.assert_array_equal(fo.patches_to_image(p, [2, 3]), img)
    with pytest.raises(AssertionError):
        fo.image_to_patches(img, [3, 3])
