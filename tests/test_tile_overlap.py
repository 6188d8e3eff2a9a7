"""Overlapped tiles with a feathered stitch (engine option tile_overlap = v).

Every tile is interpolated on a window that reaches v pixels past each interior tile boundary and neighbouring results
are cross-faded over the 2v pixels around the boundary.  The CPU tests pin the geometry (`spec.tile_windows`), the numpy
statement of the stitch (`spec.stitch_overlapped`) against a brute-force restatement of the rule kept in this file, and
the host-side sharding; the GPU tests hold k_stitch_feather and the overlapped branch of film_interpolate_tiled to
them.  With the option at 0 nothing may change, bit for bit."""
import ctypes
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from frame_interpolation_b200 import parallel, spec, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = np.full((1,), 0.5, np.float32)
TOL = 1e-3
# (frame height, frame width, block_h, block_w, overlap)
GEOMETRIES = [(128, 192, 2, 2, 16), (64, 96, 1, 3, 8), (192, 288, 3, 3, 16), (512, 768, 4, 4, 32)]


# ---------------------------------------------------------------------------------------------------------------------
# The rule, restated by brute force: per axis a (length, blocks) matrix of the weight each window has at each pixel
# ---------------------------------------------------------------------------------------------------------------------
def _axis_weights(length, blocks, v):
    p = length // blocks
    wgt = np.zeros((length, blocks), np.float64)
    for x in range(length):
        wgt[x, x // p] = 1.0                       # outside every ramp: the tile whose core contains the pixel
        if blocks > 1 and v > 0:
            for k in range(1, blocks):
                c = k * p
                if c - v <= x < c + v:
                    t = (x + 0.5 - (c - v)) / (2 * v)
                    wgt[x] = 0.0
                    wgt[x, k - 1], wgt[x, k] = 1.0 - t, t
    return wgt


def _stitch_reference(tiles, h, w, block_shape, v):
    """Separable weighted sum of the windows over every pixel, float64: (1, h, w, C)."""
    bh, bw = block_shape
    origins, (qh, qw) = spec.tile_windows(h, w, block_shape, v)
    wy, wx = _axis_weights(h, bh, v), _axis_weights(w, bw, v)
    tiles = np.asarray(tiles, np.float64)
    out = np.zeros((h, w, tiles.shape[-1]), np.float64)
    for t, (oy, ox) in enumerate(origins):
        full = np.zeros_like(out)
        full[oy:oy + qh, ox:ox + qw] = tiles[t]
        out += wy[:, t // bw, None, None] * wx[None, :, t % bw, None] * full
    return out[np.newaxis]


class OverlapOracle:
    """The CPU oracle with overlapped tiles: every window of `spec.tile_windows` through OracleInterpolator.interpolate
    (padded to `align` on its own, like a tile), stitched by `_stitch_reference`.  tile_overlap = 0 is the oracle's own
    tiled path."""

    def __init__(self, weights, align=None, block_shape=None, tile_overlap=0, dtype=torch.float32):
        from oracle.film_oracle import OracleInterpolator
        self._orc = OracleInterpolator(weights, align=align, block_shape=block_shape, dtype=dtype)
        self._block_shape, self._v = block_shape, tile_overlap

    def __call__(self, x0, x1, dt):
        if not self._v:
            return self._orc(x0, x1, dt)
        _, h, w, _ = x0.shape
        origins, (qh, qw) = spec.tile_windows(h, w, self._block_shape, self._v)
        outs = [self._orc.interpolate(x0[:, y:y + qh, x:x + qw], x1[:, y:y + qh, x:x + qw], dt)[0] for y, x in origins]
        return _stitch_reference(np.stack(outs), h, w, self._block_shape, self._v)


def fake_engine(x0, x1, dt):
    # position-dependent so that any window-origin or ordering mistake changes the result
    ramp = np.arange(x0.shape[1] * x0.shape[2], dtype=np.float32).reshape(1, x0.shape[1], x0.shape[2], 1)
    return 0.5 * (x0 + x1) + 1e-3 * ramp


def fake_engine_dev(x0, x1, out):
    h, w, _ = x0.shape
    out.copy_(0.5 * (x0 + x1) + 1e-3 * torch.arange(h * w, dtype=torch.float32).view(h, w, 1))


fake_engine_dev.stitch = parallel.stitch_tiles_host


def _fake_overlapped(x0, x1, block_shape, v):
    _, h, w, _ = x0.shape
    origins, (qh, qw) = spec.tile_windows(h, w, block_shape, v)
    outs = [fake_engine(x0[:, y:y + qh, x:x + qw], x1[:, y:y + qh, x:x + qw], DT)[0] for y, x in origins]
    return spec.stitch_overlapped(np.stack(outs), h, w, block_shape, v).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w,bh,bw,v", GEOMETRIES)
def test_window_geometry(h, w, bh, bw, v):
    origins, (qh, qw) = spec.tile_windows(h, w, [bh, bw], v)
    ph, pw = h // bh, w // bw
    assert len(origins) == bh * bw
    # one shape for every window: the core plus v on both sides of an axis that is cut at all
    assert (qh, qw) == (ph + (2 * v if bh > 1 else 0), pw + (2 * v if bw > 1 else 0))
    for t, (oy, ox) in enumerate(origins):
        r, c = divmod(t, bw)
        assert 0 <= oy and oy + qh <= h and 0 <= ox and ox + qw <= w          # inside the frame
        # the core plus v on interior sides
        assert oy <= max(r * ph - v, 0) and oy + qh >= min((r + 1) * ph + v, h)
        assert ox <= max(c * pw - v, 0) and ox + qw >= min((c + 1) * pw + v, w)
    oy, ox = [origins[r * bw][0] for r in range(bh)], [origins[c][1] for c in range(bw)]
    for length, blocks, org, q in ((h, bh, oy, qh), (w, bw, ox, qw)):
        wgt = _axis_weights(length, blocks, v)
        np.testing.assert_allclose(wgt.sum(axis=1), 1.0, rtol=0, atol=1e-15)
        assert ((wgt != 0).sum(axis=1) <= 2).all()
        assert blocks == 1 or ((wgt != 0).sum(axis=1) == 2).sum() == 2 * v * (blocks - 1)
        # a window is only ever read where it has pixels
        for k in range(blocks):
            x = np.nonzero(wgt[:, k])[0]
            assert org[k] <= x.min() and x.max() < org[k] + q


@pytest.mark.parametrize("h,w,bh,bw,v", GEOMETRIES + [(30, 42, 2, 3, 5), (12, 18, 3, 3, 0), (64, 64, 2, 2, 16)])
def test_stitch_of_crops_of_one_image_returns_the_image(h, w, bh, bw, v):
    g = np.random.default_rng(h * w + v).random((h, w, 3))
    origins, (qh, qw) = spec.tile_windows(h, w, [bh, bw], v)
    tiles = np.stack([g[y:y + qh, x:x + qw] for y, x in origins])
    assert np.abs(spec.stitch_overlapped(tiles, h, w, [bh, bw], v)[0] - g).max() <= 1e-12
    assert np.abs(_stitch_reference(tiles, h, w, [bh, bw], v)[0] - g).max() <= 1e-12


@pytest.mark.parametrize("h,w,bh,bw,v", GEOMETRIES[:3] + [(30, 42, 2, 3, 5), (64, 64, 2, 2, 16)])
def test_stitch_of_unrelated_tiles_follows_the_rule(h, w, bh, bw, v):
    """Random windows that disagree everywhere: the lerp form against the brute-force weighted sum."""
    _, (qh, qw) = spec.tile_windows(h, w, [bh, bw], v)
    tiles = np.random.default_rng(7).random((bh * bw, qh, qw, 3))
    got = spec.stitch_overlapped(tiles, h, w, [bh, bw], v)
    assert got.shape == (1, h, w, 3) and got.dtype == np.float64
    assert np.abs(got - _stitch_reference(tiles, h, w, [bh, bw], v)).max() <= 1e-12
    # the last column before a boundary and the first after it differ by one ramp step, not by a seam
    pw = w // bw
    if bw > 1:
        origins, _ = spec.tile_windows(h, w, [bh, bw], v)
        a = tiles[0][0, pw - 1 - origins[0][1]]
        b = tiles[1][0, pw - 1 - origins[1][1]]
        t = (v - 0.5) / (2 * v)
        np.testing.assert_allclose(got[0, 0, pw - 1], a + t * (b - a), rtol=0, atol=1e-12)


def test_zero_overlap_is_the_reference_tiling(synthetic_weights):
    from frame_interpolation_b200.interpolator import image_to_patches, patches_to_image
    g = np.random.default_rng(3).random((1, 12, 18, 3))
    np.testing.assert_array_equal(spec.stitch_overlapped(image_to_patches(g, [3, 3]), 12, 18, [3, 3], 0), g)
    np.testing.assert_array_equal(patches_to_image(image_to_patches(g, [3, 3]), [3, 3]), g)
    gold = np.load(os.path.join(ROOT, "tests", "golden", "g128_tiled2x2.npz"))
    x0, x1 = synthetic.frame_pair(128, 128, seed=7, n_waves=6)
    out = OverlapOracle(synthetic_weights[1], align=64, block_shape=[2, 2], tile_overlap=0)(x0, x1, DT)
    assert np.abs(out - gold["image"]).max() < 1e-5


@pytest.mark.parametrize("h,w,bh,bw,v,axis", [(128, 192, 2, 2, 33, "height"), (128, 64, 1, 2, 17, "width"),
                                               (96, 96, 3, 3, 17, "height")])
def test_overlap_of_more_than_half_a_tile_is_refused(h, w, bh, bw, v, axis):
    with pytest.raises(AssertionError, match=axis):
        spec.tile_windows(h, w, [bh, bw], v)
    spec.tile_windows(h, w, [bh, bw], min(h // bh if bh > 1 else h, w // bw if bw > 1 else w) // 2)


def test_host_sharding_with_overlap_matches_the_stitch_of_the_same_results():
    rng = np.random.default_rng(0)
    x0, x1 = (rng.random((1, 24, 36, 3), dtype=np.float32) for _ in range(2))
    for block, v in (([3, 3], 4), ([2, 2], 6), ([1, 3], 5)):
        want = _fake_overlapped(x0, x1, block, v)
        got = parallel.interpolate_tiled(fake_engine, x0, x1, block, overlap=v)
        assert got.dtype == np.float32
        np.testing.assert_array_equal(got, want)
        t0, t1 = torch.from_numpy(x0), torch.from_numpy(x1)
        np.testing.assert_array_equal(parallel.interpolate_tiled_device(fake_engine_dev, t0, t1, block, overlap=v).numpy(), want)
    # a window is a row-pitched view of the frame, never a copy; overlap 0 is the tile
    t0 = torch.from_numpy(x0)
    v = parallel.window_view(t0, [3, 3], 4, 4)
    assert v.shape == (16, 20, 3) and v.stride(0) == 36 * 3 and v.data_ptr() == t0[0, 4, 8].data_ptr()
    assert parallel.window_view(t0, [3, 3], 8, 4).data_ptr() == t0[0, 8, 16].data_ptr()      # shifted inward
    assert parallel.window_view(t0, [3, 3], 4, 0).data_ptr() == parallel.tile_view(t0, [3, 3], 4).data_ptr()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(0)
    x0, x1 = (rng.random((1, 24, 36, 3), dtype=np.float32) for _ in range(2))
    res = {"host": parallel.interpolate_tiled(fake_engine, x0, x1, [3, 3], overlap=4),
           "dev": parallel.interpolate_tiled_device(fake_engine_dev, torch.from_numpy(x0), torch.from_numpy(x1), [3, 3],
                                                    overlap=4).numpy()}
    q.put((rank, res))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(240)
def test_two_ranks_with_overlap_bitwise_equal_serial():
    """9 windows over 2 ranks (5 / 4): the rank-major slots reach the stitch through the slot table."""
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=150) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    rng = np.random.default_rng(0)
    x0, x1 = (rng.random((1, 24, 36, 3), dtype=np.float32) for _ in range(2))
    want = _fake_overlapped(x0, x1, [3, 3], 4)
    for r in range(world):
        np.testing.assert_array_equal(got[r]["host"], want)
        np.testing.assert_array_equal(got[r]["dev"], want)


def test_library_exports_the_stitch_entry_point(built_lib):
    from frame_interpolation_b200 import _lib
    assert "film_stitch_tiles_device" in _lib.EXPORTS
    assert hasattr(ctypes.CDLL(built_lib), "film_stitch_tiles_device")
    with open(os.path.join(ROOT, "include", "film_b200.h")) as f:
        header = f.read()
    assert "FILM_API int film_stitch_tiles_device(" in header
    assert '"tile_overlap"' in header


def test_cli_flag():
    from frame_interpolation_b200 import interpolator_cli
    p = interpolator_cli.build_parser()
    assert p.parse_args(["--pattern", "x", "--model_path", "synthetic"]).tile_overlap == 0
    assert p.parse_args(["--pattern", "x", "--model_path", "synthetic", "--tile_overlap", "32"]).tile_overlap == 32


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _engine(synthetic_weights, align=64, block_shape=None, overlap=None, any_size=False):
    from frame_interpolation_b200.interpolator import Interpolator
    eng = Interpolator(synthetic_weights[0], align=align, block_shape=block_shape)
    if any_size:
        eng.set_option("any_size", 1)
    if overlap is not None:
        eng.set_option("tile_overlap", overlap)
    return eng


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,block,v,align,window", [
    (128, 192, [2, 2], 16, 64, (128, 128)),      # 96x128 windows padded to 128x128
    (128, 288, [1, 3], 16, 64, (128, 128)),      # one axis unblended
    (192, 288, [3, 3], 16, 64, (128, 128)),      # an interior tile, four-tile corners
    (200, 300, [2, 2], 10, None, (120, 170)),    # unpadded windows that are not 64-aligned
])
def test_engine_matches_the_oracle(synthetic_weights, h, w, block, v, align, window):
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    x0, x1 = synthetic.frame_pair(h, w, seed=21, n_waves=8)
    ref = OverlapOracle(synthetic_weights[1], align=align, block_shape=block, tile_overlap=v)(x0, x1, DT)
    eng = _engine(synthetic_weights, align, block, v, any_size=align is None)
    try:
        out = eng(x0, x1, DT)
        assert out.shape == ref.shape == (1, h, w, 3)
        err = np.abs(out.astype(np.float64) - ref).max()
        assert err <= TOL, err
        p = eng.profile()
        assert (p["padded_h"], p["padded_w"]) == window
        # the mode is not the reference's tiling: the pasted result differs in the ramps
        eng.set_option("tile_overlap", 0)
        assert np.abs(eng(x0, x1, DT) - out).max() > 0
    finally:
        eng.close()


@pytest.mark.gpu
def test_overlap_back_to_zero_is_bitwise_the_untouched_path(synthetic_weights):
    from frame_interpolation_b200.parallel import device_engine, interpolate_tiled_device
    x0, x1 = synthetic.frame_pair(128, 192, seed=22, n_waves=8)
    d0, d1 = torch.from_numpy(x0).cuda(), torch.from_numpy(x1).cuda()
    used = _engine(synthetic_weights, 64, [2, 2], 16)
    fresh = _engine(synthetic_weights, 64, [2, 2])
    try:
        used(x0, x1, DT)
        interpolate_tiled_device(device_engine(used), d0, d1, [2, 2], overlap=16)
        used.set_option("tile_overlap", 0)
        np.testing.assert_array_equal(used(x0, x1, DT), fresh(x0, x1, DT))
        a = interpolate_tiled_device(device_engine(used), d0, d1, [2, 2]).cpu().numpy()
        b = interpolate_tiled_device(device_engine(fresh), d0, d1, [2, 2]).cpu().numpy()
        np.testing.assert_array_equal(a, b)
        np.testing.assert_array_equal(a, fresh(x0, x1, DT))
    finally:
        used.close()
        fresh.close()


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,bh,bw,v", [(128, 192, 2, 2, 16), (192, 288, 3, 3, 16), (30, 42, 2, 3, 5), (64, 100, 1, 2, 25),
                                         (96, 64, 4, 1, 12)])
def test_stitch_kernel_alone(synthetic_weights, h, w, bh, bw, v):
    """Random windows, a permuted slot table into a buffer with spare slots, an output pitch larger than a row."""
    nt = bh * bw
    _, (qh, qw) = spec.tile_windows(h, w, [bh, bw], v)
    rng = np.random.default_rng(h + w + v)
    tiles = rng.random((nt, qh, qw, 3), dtype=np.float32)
    slots = [int(s) for s in rng.permutation(nt + 3)[:nt]]
    stride = qh * qw * 3 + 5                                   # slots need not be densely packed
    buf = np.full(((nt + 3) * stride,), np.nan, np.float32)
    for t, s in enumerate(slots):
        buf[s * stride:s * stride + qh * qw * 3] = tiles[t].ravel()
    want = spec.stitch_overlapped(tiles, h, w, [bh, bw], v)[0]
    d_buf = torch.from_numpy(buf).cuda()
    pitch = w * 3 + 7
    eng = _engine(synthetic_weights)
    try:
        runs = []
        for _ in range(2):
            d_out = torch.full((h, pitch), -7.0, dtype=torch.float32, device="cuda")
            eng.stitch_tiles_device(d_buf.data_ptr(), stride, h, w, [bh, bw], v, d_out.data_ptr(), slot_of_tile=slots,
                                    out_pitch=pitch)
            eng.synchronize()
            runs.append(d_out.cpu().numpy())
        np.testing.assert_array_equal(runs[0], runs[1])
        assert (runs[0][:, w * 3:] == -7.0).all()               # nothing written past a row
        assert np.abs(runs[0][:, :w * 3].reshape(h, w, 3) - want).max() <= 1e-6
        # identity slot table, dense rows
        d_tiles = torch.from_numpy(tiles).cuda()
        d_out = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
        eng.stitch_tiles_device(d_tiles.data_ptr(), qh * qw * 3, h, w, [bh, bw], v, d_out.data_ptr())
        eng.synchronize()
        np.testing.assert_array_equal(d_out.cpu().numpy(), runs[0][:, :w * 3].reshape(h, w, 3))
        with pytest.raises(AssertionError, match="tile_stride"):
            eng.stitch_tiles_device(d_tiles.data_ptr(), qh * qw * 3 - 1, h, w, [bh, bw], v, d_out.data_ptr())
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,block,v", [(128, 192, [2, 2], 16), (192, 288, [3, 3], 16)])
def test_device_resident_path_is_bitwise_the_host_call(synthetic_weights, h, w, block, v):
    from frame_interpolation_b200.parallel import device_engine, interpolate_tiled_device
    x0, x1 = synthetic.frame_pair(h, w, seed=23, n_waves=8)
    eng = _engine(synthetic_weights, 64, block, v)
    try:
        host = eng(x0, x1, DT).copy()
        dev = interpolate_tiled_device(device_engine(eng), torch.from_numpy(x0).cuda(), torch.from_numpy(x1).cuda(), block,
                                       overlap=v)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(dev.cpu().numpy(), host)
    finally:
        eng.close()


@pytest.mark.gpu
def test_option_semantics(synthetic_weights):
    eng = _engine(synthetic_weights, 64, [2, 2])
    try:
        assert eng.get_option("tile_overlap") == 0
        for v, want in ((16, 16), (-3, 0), (1, 1), (0, 0)):
            eng.set_option("tile_overlap", v)
            assert eng.get_option("tile_overlap") == want
        x0, x1 = synthetic.frame_pair(128, 192, seed=24, n_waves=8)
        eng.set_option("tile_overlap", 33)                     # tiles of 64x96
        with pytest.raises(AssertionError, match="height"):
            eng(x0, x1, DT)
        assert "height" in eng._lib.film_last_error(eng._handle).decode()
        y0, y1 = synthetic.frame_pair(192, 128, seed=24, n_waves=8)   # tiles of 96x64
        eng.set_option("tile_overlap", 40)
        with pytest.raises(AssertionError, match="width"):
            eng(y0, y1, DT)
        eng.set_option("tile_overlap", 32)                     # 2v == p on the height: still allowed
        assert eng(x0, x1, DT).shape == (1, 128, 192, 3)
    finally:
        eng.close()


@pytest.mark.gpu
def test_one_plan_serves_every_window_of_a_frame(synthetic_weights):
    """2x2 tiles of a 128x128 frame and 4x4 tiles of a 256x256 frame have the same 96x96 window: the same plan."""
    small = synthetic.frame_pair(128, 128, seed=25, n_waves=8)
    large = synthetic.frame_pair(256, 256, seed=25, n_waves=8)
    e2 = _engine(synthetic_weights, 64, [2, 2], 16)
    e4 = _engine(synthetic_weights, 64, [4, 4], 16)
    try:
        e2(*small, DT)
        e4(*large, DT)
        p2, p4 = e2.profile(), e4.profile()
        assert p2["arena_bytes"] == p4["arena_bytes"] > 0
        assert (p2["padded_h"], p2["padded_w"]) == (p4["padded_h"], p4["padded_w"]) == (128, 128)
    finally:
        e2.close()
        e4.close()
