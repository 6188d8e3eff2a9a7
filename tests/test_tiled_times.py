"""Interpolation at arbitrary times on tiles (film_interpolate_times_tiled, Interpolator.interpolate_at_tiled,
parallel.interpolate_at_tiled_device) and tiled retiming in interpolator_cli.

Frame i is the tiled interpolation of film_interpolate_tiled with every window's mid_time replaced by t_i: every window
of `spec.tile_windows` runs one head and one tail per time of the times plan, and per time the window results are
stitched by k_stitch_feather (a paste at tile_overlap 0).  What the tests pin:
1. at t = 0.5 frame i is film_interpolate_tiled, bit for bit;
2. at overlap 0, tile k of frame i is `interpolate_at` on tile k's crop, bit for bit;
3. at overlap > 0, frame i is the device stitch of `interpolate_at` on the window crops, bit for bit;
4. block [1, 1] is `interpolate_at`, bit for bit.
"""
import ctypes
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from frame_interpolation_b200 import eval_util, interpolator_cli, parallel, spec, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = np.full((1,), 0.5, np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# CPU stand-in for device_engine: a position- and time-dependent blend, so that a wrong window, slot or time shows
# ---------------------------------------------------------------------------------------------------------------------
def _blend(x0, x1, t):
    h, w, _ = x0.shape
    ramp = torch.arange(h * w, dtype=torch.float32).view(h, w, 1)
    t32 = torch.tensor(t, dtype=torch.float32)
    return (1 - t32) * x0 + t32 * x1 + 1e-3 * ramp * (t32 + 0.25)


def fake_at(x0, x1, times, out):
    for i, t in enumerate(times):
        out[i].copy_(_blend(x0, x1, t))


class _FakeDev:
    at = staticmethod(fake_at)
    stitch = staticmethod(parallel.stitch_tiles_host)


def serial_composition(x0, x1, times, block, v):
    """`at` on every window crop, then spec.stitch_overlapped per time, rounded to float32: (n, H, W, 3)."""
    _, h, w, _ = x0.shape
    origins, (qh, qw) = spec.tile_windows(h, w, block, v)
    wins = []
    for y, x in origins:
        o = torch.empty((len(times), qh, qw, 3))
        fake_at(x0[0, y:y + qh, x:x + qw], x1[0, y:y + qh, x:x + qw], times, o)
        wins.append(o.numpy())
    wins = np.stack(wins)                       # (tiles, n, qh, qw, 3)
    return np.stack([spec.stitch_overlapped(wins[:, i], h, w, block, v)[0].astype(np.float32)
                     for i in range(len(times))])


def _pair(h, w, seed=0):
    rng = np.random.default_rng(seed)
    return tuple(torch.from_numpy(rng.random((1, h, w, 3), dtype=np.float32)) for _ in range(2))


# (frame h, frame w, block, overlap): 9 and 16 tiles, so 2 and 3 ranks get uneven shares
SHARD_CASES = [(24, 36, [3, 3], 4), (24, 36, [3, 3], 0), (32, 48, [4, 4], 3), (32, 48, [4, 4], 0), (24, 36, [1, 3], 5)]
TIMES = [0.2, 0.5, 0.85]


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_library_exports_the_entry_point(built_lib):
    from frame_interpolation_b200 import _lib
    assert "film_interpolate_times_tiled" in _lib.EXPORTS
    assert hasattr(ctypes.CDLL(built_lib), "film_interpolate_times_tiled")
    with open(os.path.join(ROOT, "include", "film_b200.h")) as f:
        header = f.read()
    assert "FILM_API int film_interpolate_times_tiled(" in header


@pytest.mark.parametrize("h,w,block,v", SHARD_CASES)
def test_one_rank_is_the_serial_composition(h, w, block, v):
    x0, x1 = _pair(h, w)
    want = serial_composition(x0, x1, TIMES, block, v)
    got = parallel.interpolate_at_tiled_device(_FakeDev, x0, x1, TIMES, block, overlap=v)
    assert got.shape == (len(TIMES), h, w, 3) and got.dtype == torch.float32
    np.testing.assert_array_equal(got.numpy(), want)
    # the time reaches every frame, and the frames differ from one another
    assert not np.array_equal(want[0], want[1]) and not np.array_equal(want[1], want[2])
    # (H, W, 3) frames and a caller's output buffer
    out = torch.full((len(TIMES), h, w, 3), -7.0)
    res = parallel.interpolate_at_tiled_device(_FakeDev, x0[0], x1[0], TIMES, block, out=out, overlap=v)
    assert res is out
    np.testing.assert_array_equal(out.numpy(), want)


def test_overlap_zero_pastes_the_tiles():
    from frame_interpolation_b200.interpolator import patches_to_image
    x0, x1 = _pair(24, 36, seed=3)
    got = parallel.interpolate_at_tiled_device(_FakeDev, x0, x1, TIMES, [3, 3]).numpy()
    _, (qh, qw) = spec.tile_windows(24, 36, [3, 3], 0)
    for i, t in enumerate(TIMES):
        tiles = np.stack([_blend(parallel.tile_view(x0, [3, 3], k), parallel.tile_view(x1, [3, 3], k), t).numpy()
                          for k in range(9)])
        np.testing.assert_array_equal(got[i], patches_to_image(tiles, [3, 3])[0])


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    res = {}
    for h, w, block, v in SHARD_CASES:
        x0, x1 = _pair(h, w)
        res[(h, w, tuple(block), v)] = parallel.interpolate_at_tiled_device(_FakeDev, x0, x1, TIMES, block,
                                                                            overlap=v).numpy()
    q.put((rank, res))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("world", [2, 3])
def test_ranks_bitwise_equal_serial(world):
    """9 and 16 tiles over 2 and 3 ranks (5/4, 3/3/3, 8/8, 6/5/5): one all-gather, then per time the rank-major slots of
    that time reach the stitch through the slot table, read in place from the gather buffer."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=200) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for h, w, block, v in SHARD_CASES:
        x0, x1 = _pair(h, w)
        want = serial_composition(x0, x1, TIMES, block, v)
        for r in range(world):
            np.testing.assert_array_equal(got[r][(h, w, tuple(block), v)], want, err_msg=f"rank {r} {h}x{w} {block} {v}")


class AtStandIn:
    """`interpolate_at` / `interpolate_at_tiled` stand-in: a linear blend with a different offset per method."""

    def __init__(self):
        self.calls = []

    def _blend(self, name, off, a, b, times):
        self.calls.append((name, list(times)))
        return np.stack([np.float32(1 - t) * a + np.float32(t) * b + np.float32(off) for t in times]).astype(np.float32)

    def interpolate_at(self, a, b, times):
        return self._blend("at", 0.125, a, b, times)

    def interpolate_at_tiled(self, a, b, times):
        return self._blend("tiled", 0.25, a, b, times)


def _clip(tmp_path, n, h=8, w=8):
    d = tmp_path / "clip"
    d.mkdir()
    rng = np.random.default_rng(1)
    for i in range(n):
        eval_util.write_image(str(d / f"im{i}.png"), rng.random((h, w, 3)).astype(np.float32))
    return d, [str(d / f"im{i}.png") for i in range(n)]


def test_retime_sends_each_pairs_times_to_at(tmp_path):
    _, names = _clip(tmp_path, 4)
    s = AtStandIn()
    frames = list(eval_util.retime_from_files(names, 24, 60, s, at=s.interpolate_at_tiled))
    assert s.calls == [("tiled", [0.4, 0.8]), ("tiled", [0.2, 0.6]), ("tiled", [0.4, 0.8])] and len(frames) == 8
    a, b = eval_util.read_image(names[1]), eval_util.read_image(names[2])
    np.testing.assert_array_equal(frames[3], s.interpolate_at_tiled(a, b, [0.2])[0])
    np.testing.assert_array_equal(frames[5], eval_util.read_image(names[2]))
    s = AtStandIn()
    list(eval_util.retime_from_files(names, 24, 60, s))
    assert [c[0] for c in s.calls] == ["at"] * 3


def test_cli_routes_tiles_with_overlap_to_at(tmp_path, monkeypatch):
    d, names = _clip(tmp_path, 3)
    s = AtStandIn()
    n = interpolator_cli.retime_directory(str(d), s, 24, 60, video=False, at=s.interpolate_at_tiled)
    assert n == 6 and [c[0] for c in s.calls] == ["tiled", "tiled"]
    out = d / "interpolated_frames"
    want = s.interpolate_at_tiled(eval_util.read_image(names[0]), eval_util.read_image(names[1]), [0.4])[0]
    np.testing.assert_array_equal(eval_util.to_uint8(eval_util.read_image(str(out / "frame_001.png"))),
                                  eval_util.to_uint8(want))

    made = []

    class FakeInterpolator(AtStandIn):
        def __init__(self, model_path, align, block_shape, device=0):
            super().__init__()
            self.block_shape, self.options = block_shape, {}
            made.append(self)

        def set_option(self, name, value):
            self.options[name] = value

    monkeypatch.setattr(interpolator_cli, "Interpolator", FakeInterpolator)
    base = ["--pattern", str(d), "--model_path", "m", "--source_fps", "24", "--target_fps", "60"]
    assert interpolator_cli.main(base + ["--block_height", "2", "--block_width", "2", "--tile_overlap", "8"]) == 0
    assert made[-1].block_shape == [2, 2] and made[-1].options == {"tile_overlap": 8}
    assert [c[0] for c in made[-1].calls] == ["tiled", "tiled"]
    assert interpolator_cli.main(base) == 0                       # untiled: interpolate_at, as before
    assert [c[0] for c in made[-1].calls] == ["at", "at"]
    n_made = len(made)
    for tiles in (["--block_height", "2"], ["--block_width", "3", "--tile_overlap", "0"]):
        with pytest.raises(SystemExit):
            interpolator_cli.main(base + tiles)
    assert len(made) == n_made                                    # refused before any engine is created


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _engine(path, align=64, block_shape=None, overlap=None, **opts):
    from frame_interpolation_b200.interpolator import Interpolator
    eng = Interpolator(path, align=align, block_shape=block_shape)
    if align is None:
        eng.set_option("any_size", 1)
    if overlap is not None:
        eng.set_option("tile_overlap", overlap)
    for k, v in opts.items():
        eng.set_option(k, v)
    return eng


HALF_CASES = [
    (128, 192, [2, 2], 0, 64, {}),
    (128, 192, [2, 2], 0, 64, {"onepass_mask": 0}),
    (128, 192, [2, 2], 16, 64, {}),
    (128, 192, [2, 2], 16, 64, {"onepass_mask": 0}),
    (192, 288, [3, 3], 16, 64, {}),
    (128, 288, [1, 3], 16, 64, {}),
    (200, 300, [2, 2], 10, None, {}),
]


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,block,v,align,opts", HALF_CASES)
def test_half_is_the_tiled_call(synthetic_weights, h, w, block, v, align, opts):
    """Property 1; later tails and later windows leave what earlier ones produced alone."""
    x0, x1 = synthetic.frame_pair(h, w, seed=31, n_waves=8)
    eng = _engine(synthetic_weights[0], align, block, v, **opts)
    try:
        want = np.array(eng(x0, x1, DT)[0])
        got = np.array(eng.interpolate_at_tiled(x0[0], x1[0], [0.3, 0.5, 0.9, 0.5]))
        assert got.shape == (4, h, w, 3)
        assert np.array_equal(got[1], want) and np.array_equal(got[3], want)
        alone = np.array(eng.interpolate_at_tiled(x0[0], x1[0], [0.3]))[0]
        assert np.array_equal(got[0], alone)
        assert not np.array_equal(got[0], want) and not np.array_equal(got[2], got[0])
        assert np.array_equal(np.array(eng(x0, x1, DT)[0]), want)      # the ordinary tiled call is untouched
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("t", [0.2, 0.7])
def test_overlap_zero_tiles_are_interpolate_at_on_the_crops(synthetic_weights, t):
    """Property 2: a tile of the result is `interpolate_at` of an untiled engine on the tile's crop."""
    from frame_interpolation_b200.interpolator import image_to_patches
    h, w, block = 128, 192, [2, 2]
    x0, x1 = synthetic.frame_pair(h, w, seed=32, n_waves=8)
    tiled = _engine(synthetic_weights[0], 64, block)
    plain = _engine(synthetic_weights[0], 64)
    try:
        got = np.array(tiled.interpolate_at_tiled(x0[0], x1[0], [0.5, t]))[1]
        tiles = image_to_patches(got, block)
        p0, p1 = image_to_patches(x0[0], block), image_to_patches(x1[0], block)
        for k in range(4):
            want = np.array(plain.interpolate_at(p0[k], p1[k], [t]))[0]
            assert np.array_equal(tiles[k], want), k
    finally:
        tiled.close()
        plain.close()


@pytest.mark.gpu
def test_overlap_is_the_device_stitch_of_interpolate_at(synthetic_weights):
    """Property 3 at v = 16: `interpolate_at` on every window crop, then film_stitch_tiles_device per time."""
    h, w, block, v = 192, 288, [3, 3], 16
    times = [0.15, 0.6]
    x0, x1 = synthetic.frame_pair(h, w, seed=33, n_waves=8)
    tiled = _engine(synthetic_weights[0], 64, block, v)
    plain = _engine(synthetic_weights[0], 64)
    try:
        got = np.array(tiled.interpolate_at_tiled(x0[0], x1[0], times))
        origins, (qh, qw) = spec.tile_windows(h, w, block, v)
        wins = np.stack([np.array(plain.interpolate_at(x0[0, y:y + qh, x:x + qw], x1[0, y:y + qh, x:x + qw], times))
                         for y, x in origins])                    # (tiles, n, qh, qw, 3)
        for i in range(len(times)):
            d_tiles = torch.from_numpy(np.ascontiguousarray(wins[:, i])).cuda()
            d_out = torch.empty((h, w, 3), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            plain.stitch_tiles_device(d_tiles.data_ptr(), qh * qw * 3, h, w, block, v, d_out.data_ptr())
            plain.synchronize()
            assert np.array_equal(got[i], d_out.cpu().numpy()), i
    finally:
        tiled.close()
        plain.close()


@pytest.mark.gpu
@pytest.mark.parametrize("block", [None, [1, 1]])
def test_one_tile_is_interpolate_at(synthetic_weights, block):
    """Property 4."""
    x0, x1 = synthetic.frame_pair(128, 192, seed=34, n_waves=8)
    times = [0.1, 0.5, 0.75]
    eng = _engine(synthetic_weights[0], 64, block, 16)
    try:
        got = np.array(eng.interpolate_at_tiled(x0[0], x1[0], times))
        assert np.array_equal(got, np.array(eng.interpolate_at(x0[0], x1[0], times)))
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("onepass_mask,tol", [(0, 1e-4), (None, 4e-4)])
def test_against_the_oracle(synthetic_weights, onepass_mask, tol):
    """TimeOracle on every window, then spec.stitch_overlapped per time, float64 throughout the stitch."""
    from test_time_interpolation import TimeOracleInterpolator
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    path, wts = synthetic_weights
    h, w, block, v = 128, 192, [2, 2], 16
    times = [0.25, 0.8]
    x0, x1 = synthetic.frame_pair(h, w, seed=35, n_waves=8)
    eng = _engine(path, 64, block, v, **({} if onepass_mask is None else {"onepass_mask": onepass_mask}))
    try:
        got = np.array(eng.interpolate_at_tiled(x0[0], x1[0], times)).astype(np.float64)
    finally:
        eng.close()
    orc = TimeOracleInterpolator(wts, align=64)
    origins, (qh, qw) = spec.tile_windows(h, w, block, v)
    wins = np.stack([orc.interpolate_at(x0[0, y:y + qh, x:x + qw], x1[0, y:y + qh, x:x + qw], times)
                     for y, x in origins])
    ref = np.stack([spec.stitch_overlapped(wins[:, i], h, w, block, v)[0] for i in range(len(times))])
    err = np.abs(got - ref).max(axis=(1, 2, 3))
    print("max-abs vs oracle per time:", err)
    assert (err <= tol).all(), err


@pytest.mark.gpu
@pytest.mark.parametrize("opts", [{"use_graph": 0}, {"time_ops": 1}, {"keep_debug": 1}, {"use_lanes": 1}])
def test_schedules_agree_bit_for_bit(synthetic_weights, opts):
    h, w, block, v = 128, 192, [2, 2], 16
    x0, x1 = synthetic.frame_pair(h, w, seed=36, n_waves=8)
    times = [0.25, 0.5, 0.8]
    ref = _engine(synthetic_weights[0], 64, block, v)
    eng = _engine(synthetic_weights[0], 64, block, v, **opts)
    try:
        want = np.array(ref.interpolate_at_tiled(x0[0], x1[0], times))
        assert ref.profile()["used_graph"] == 1
        got = np.array(eng.interpolate_at_tiled(x0[0], x1[0], times))
        assert np.array_equal(got[1], np.array(eng(x0, x1, DT)[0])), opts
        if not opts.get("use_lanes"):   # lanes pool the image pyramid in kernels of their own
            assert np.array_equal(got, want), opts
        if opts.get("time_ops"):
            table = eng.op_table()
            assert all(r["ms"] >= 0 for r in table) and len({r["name"] for r in table if r["name"]}) > 10
        if opts.get("keep_debug"):
            # readable after the call: the last window's tensors, at the padded window shape
            eng.interpolate_at_tiled(x0[0], x1[0], times)
            assert eng.debug_read("flow_fwd/0").size == 128 * 128 * 2
    finally:
        ref.close()
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("v", [0, 16])
def test_device_path_equals_the_host_call(synthetic_weights, v):
    """parallel.interpolate_at_tiled_device at world size 1 on an untiled engine, against interpolate_at_tiled."""
    h, w, block = 128, 192, [2, 2]
    times = [0.3, 0.5, 0.65]
    x0, x1 = synthetic.frame_pair(h, w, seed=37, n_waves=8)
    tiled = _engine(synthetic_weights[0], 64, block, v)
    plain = _engine(synthetic_weights[0], 64)
    try:
        want = np.array(tiled.interpolate_at_tiled(x0[0], x1[0], times))
        got = parallel.interpolate_at_tiled_device(parallel.device_engine(plain), torch.from_numpy(x0).cuda(),
                                                   torch.from_numpy(x1).cuda(), times, block, overlap=v)
        torch.cuda.synchronize()
        assert got.shape == (3, h, w, 3)
        assert np.array_equal(got.cpu().numpy(), want)
    finally:
        tiled.close()
        plain.close()


@pytest.mark.gpu
def test_profile_and_plans(synthetic_weights):
    h, w, block, v = 128, 192, [2, 2], 16           # 96x128 windows, padded to 128x128
    x0, x1 = synthetic.frame_pair(h, w, seed=38, n_waves=8)
    eng = _engine(synthetic_weights[0], 64, block, v)
    try:
        want_tiled = np.array(eng(x0, x1, DT)[0])
        p_tiled = eng.profile()
        n_ops = len(eng.op_table())
        for n in (1, 3):
            eng.interpolate_at_tiled(x0[0], x1[0], np.linspace(0.1, 0.9, n))
            p = eng.profile()
            assert (p["padded_h"], p["padded_w"]) == (128, 128)
            m = spec.conv_macs(128, 128)
            assert p["conv_flops"] == pytest.approx(4 * 2 * (m["feature_extractor"] + m["flow"] + n * m["fusion"]),
                                                    rel=1e-12)
            table = eng.op_table()
            tail = len(table) - [r["name"] for r in table].index("fusion_warp@L0")
            assert len(table) == n_ops and p["kernel_launches"] == 4 * (len(table) - tail + n * tail)
            assert p["last_call_ms"] > 0
        p_times = eng.profile()
        assert p_times["arena_bytes"] > p_tiled["arena_bytes"]
        # a later ordinary tiled call is unchanged
        assert np.array_equal(np.array(eng(x0, x1, DT)[0]), want_tiled)
        p = eng.profile()
        assert p["arena_bytes"] == p_tiled["arena_bytes"] and p["kernel_launches"] == p_tiled["kernel_launches"]
        assert p["conv_flops"] == p_tiled["conv_flops"]
    finally:
        eng.close()
    # a 2x2 frame and a 4x4 frame with the same 96x96 window share one times plan
    small = synthetic.frame_pair(128, 128, seed=39, n_waves=8)
    large = synthetic.frame_pair(256, 256, seed=39, n_waves=8)
    e2 = _engine(synthetic_weights[0], 64, [2, 2], 16)
    e4 = _engine(synthetic_weights[0], 64, [4, 4], 16)
    try:
        e2.interpolate_at_tiled(small[0][0], small[1][0], [0.4])
        e4.interpolate_at_tiled(large[0][0], large[1][0], [0.4])
        p2, p4 = e2.profile(), e4.profile()
        assert p2["arena_bytes"] == p4["arena_bytes"] > 0
        assert (p2["padded_h"], p2["padded_w"]) == (p4["padded_h"], p4["padded_w"]) == (128, 128)
    finally:
        e2.close()
        e4.close()


@pytest.mark.gpu
def test_argument_errors(synthetic_weights):
    x0, x1 = synthetic.frame_pair(128, 192, seed=40, n_waves=8)
    eng = _engine(synthetic_weights[0], 64, [2, 2], 16)
    try:
        for bad, idx in (([], None), ([0.2, -0.1], 1), ([1.5], 0), ([0.5, 0.5, float("nan")], 2)):
            with pytest.raises(AssertionError) as e:
                eng.interpolate_at_tiled(x0[0], x1[0], bad)
            assert (f"times[{idx}]" if idx is not None else "n_times") in str(e.value)
        eng.set_option("tile_overlap", 33)                 # tiles of 64x96: 2v > 64 on the height
        with pytest.raises(AssertionError, match="height"):
            eng.interpolate_at_tiled(x0[0], x1[0], [0.5])
        eng.set_option("tile_overlap", 16)
        y0, y1 = synthetic.frame_pair(128, 191, seed=40, n_waves=8)
        with pytest.raises(AssertionError, match="block_width"):
            eng.interpolate_at_tiled(y0[0], y1[0], [0.5])
        assert np.array(eng.interpolate_at_tiled(x0[0], x1[0], [0.0, 1.0])).shape == (2, 128, 192, 3)
    finally:
        eng.close()


@pytest.mark.gpu
def test_cli_tiled_retime_end_to_end(tmp_path, synthetic_weights):
    d = tmp_path / "clip"
    d.mkdir()
    x0, x1 = synthetic.frame_pair(64, 96, seed=3)
    x2, _ = synthetic.frame_pair(64, 96, seed=4)
    for i, f in enumerate((x0[0], x1[0], x2[0])):
        eval_util.write_image(str(d / f"f{i}.png"), f)
    rc = interpolator_cli.main(["--pattern", str(d), "--model_path", synthetic_weights[0], "--block_height", "2",
                                "--block_width", "2", "--tile_overlap", "8", "--source_fps", "24", "--target_fps", "60"])
    assert rc == 0
    out = sorted(os.listdir(d / "interpolated_frames"))
    assert out == [f"frame_{i:03d}.png" for i in range(6)]   # positions 0, 0.4, 0.8, 1.2, 1.6, 2
    rd = lambda p: eval_util.read_image(str(p))
    np.testing.assert_array_equal(rd(d / "interpolated_frames" / "frame_000.png"), rd(d / "f0.png"))
    np.testing.assert_array_equal(rd(d / "interpolated_frames" / "frame_005.png"), rd(d / "f2.png"))
    eng = _engine(synthetic_weights[0], 64, [2, 2], 8)
    try:
        a, b = rd(d / "f1.png"), rd(d / "f2.png")
        want = eval_util.to_uint8(np.array(eng.interpolate_at_tiled(a, b, [np.float32(0.2)]))[0])
        np.testing.assert_array_equal(eval_util.to_uint8(rd(d / "interpolated_frames" / "frame_003.png")), want)
    finally:
        eng.close()
