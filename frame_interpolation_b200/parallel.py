"""Multi-GPU sharding of the FILM hot path (one process per GPU, torch.distributed).

The path shards into independent units:

* frame pairs  -- `interpolate_pairs`: contiguous block partition of N independent
  (x0, x1) pairs over ranks, weights replicated, ONE all-gather of the outputs so every
  rank (or a single writer) holds the full sequence.
* tiles        -- `interpolate_tiled`: the reference's `--block_height/--block_width`
  tiles (eval/interpolator.py:192-206) are independent by construction (no halo, each
  tile padded on its own), so tile t goes to rank t % world; ONE all-gather reassembles
  the stitched frame (NCCL over NVLink on GPUs; gloo on CPU for the host-logic tests).
  With `overlap` > 0 every tile runs on its window of `spec.tile_windows` and the gathered
  results are cross-faded instead of pasted (engine option tile_overlap).
  `interpolate_at_tiled_device` is the same for the frames of one pair at several times.
* recursion    -- `interpolate_recursively`: eval/util.py:62-91's binary dependency tree
  scheduled level-synchronously: the 2^(k-1) calls of level k are sharded, new mid-frames
  are all-gathered so every rank holds the parents of level k+1; the output order is the
  generator's in-order traversal.

There is no model parallelism (34 M parameters) and no collective inside the network.
`engine` is any callable `(x0, x1, dt) -> mid` on numpy NHWC batches -- the real
`Interpolator` in production, a stand-in in the CPU (gloo) tests of this host logic.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

from . import spec

Engine = Callable[[np.ndarray, np.ndarray, np.ndarray], np.ndarray]


def block_partition(n_items: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous [start, stop) share of `rank`; the first n % world ranks get one extra."""
    base, rem = divmod(n_items, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def round_robin(n_items: int, world: int, rank: int) -> List[int]:
    return list(range(rank, n_items, world))


def _dist():
    import torch.distributed as dist
    return dist


def _world_rank(group=None) -> Tuple[int, int]:
    dist = _dist()
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(group), dist.get_rank(group)
    return 1, 0


def _all_gather_padded(local: np.ndarray, counts: Sequence[int], device=None, group=None) -> np.ndarray:
    """All-gathers `local` (n_local, ...) where ranks hold different n_local (`counts`).
    One collective: every rank pads to max(counts) rows, all_gather_into_tensor, then the
    padding is dropped. Returns the concatenation in rank order."""
    import torch
    dist = _dist()
    world, rank = _world_rank(group)
    if world == 1:
        return local
    item_shape = local.shape[1:]
    m = max(counts)
    buf = torch.zeros((m,) + tuple(item_shape), dtype=torch.float32, device=device or "cpu")
    if local.shape[0]:
        buf[: local.shape[0]] = torch.from_numpy(np.ascontiguousarray(local)).to(buf.device)
    out = torch.empty((world * m,) + tuple(item_shape), dtype=torch.float32, device=buf.device)
    dist.all_gather_into_tensor(out, buf, group=group)
    out = out.cpu().numpy().reshape((world, m) + tuple(item_shape))
    return np.concatenate([out[r, : counts[r]] for r in range(world)], axis=0)


def interpolate_pairs(engine: Engine, x0: np.ndarray, x1: np.ndarray, device=None, group=None,
                      gather: bool = True) -> np.ndarray:
    """Mid-frames of N independent pairs (x0[i], x1[i]), sharded over ranks.

    x0, x1: (N, H, W, 3). Returns (N, H, W, 3) on every rank when `gather`, else only the
    local block (N_local, H, W, 3)."""
    world, rank = _world_rank(group)
    n = x0.shape[0]
    lo, hi = block_partition(n, world, rank)
    outs = [engine(x0[i:i + 1], x1[i:i + 1], np.full((1,), 0.5, np.float32)) for i in range(lo, hi)]
    local = np.concatenate(outs, axis=0) if outs else np.zeros((0,) + x0.shape[1:], np.float32)
    if not gather or world == 1:
        return local
    counts = [block_partition(n, world, r)[1] - block_partition(n, world, r)[0] for r in range(world)]
    return _all_gather_padded(local, counts, device, group)


def interpolate_tiled(engine: Engine, x0: np.ndarray, x1: np.ndarray, block_shape: Sequence[int],
                      device=None, group=None, overlap: int = 0) -> np.ndarray:
    """The reference's tiled path with tiles sharded round-robin over ranks and one
    all-gather to reassemble (eval/interpolator.py:192-206 runs them sequentially).
    overlap > 0: every tile runs on its window of `spec.tile_windows` and the results are cross-faded
    (`spec.stitch_overlapped`, rounded to float32) instead of pasted."""
    from .interpolator import image_to_patches, patches_to_image
    world, rank = _world_rank(group)
    bh, bw = int(block_shape[0]), int(block_shape[1])
    if overlap:
        origins, (qh, qw) = spec.tile_windows(x0.shape[1], x0.shape[2], [bh, bw], overlap)
        p0, p1 = (np.stack([x[0, y:y + qh, c:c + qw] for y, c in origins]) for x in (x0, x1))
    else:
        p0 = image_to_patches(x0, [bh, bw])
        p1 = image_to_patches(x1, [bh, bw])
    nt = bh * bw
    mine = round_robin(nt, world, rank)
    dt = np.full((1,), 0.5, np.float32)
    outs = [engine(p0[t][np.newaxis], p1[t][np.newaxis], dt) for t in mine]
    local = np.concatenate(outs, axis=0) if outs else np.zeros((0,) + p0.shape[1:], np.float32)
    if world > 1:
        counts = [len(round_robin(nt, world, r)) for r in range(world)]
        gathered = _all_gather_padded(local, counts, device, group)
        # rank-major order -> tile order
        order = [t for r in range(world) for t in round_robin(nt, world, r)]
        tiles = np.empty_like(gathered)
        tiles[order] = gathered
    else:
        tiles = local
    if overlap:
        return spec.stitch_overlapped(tiles, x0.shape[1], x0.shape[2], [bh, bw], overlap).astype(np.float32)
    return patches_to_image(tiles, [bh, bw])


def interpolate_recursively(engine: Engine, frame0: np.ndarray, frame1: np.ndarray,
                            times_to_interpolate: int, device=None, group=None) -> List[np.ndarray]:
    """All 2^n - 1 mid-frames between two (H, W, 3) frames plus the end points, in display
    order -- the sequence `_recursive_generator` (eval/util.py:62-91) yields, followed by
    frame1 (eval/util.py:118-123). Level-synchronous over ranks: at level k the 2^(k-1)
    independent calls are block-partitioned and their results all-gathered."""
    world, rank = _world_rank(group)
    frames = [np.asarray(frame0, np.float32), np.asarray(frame1, np.float32)]
    for _ in range(times_to_interpolate):
        a = np.stack(frames[:-1])
        b = np.stack(frames[1:])
        mids = interpolate_pairs(engine, a, b, device, group, gather=True)
        nxt = []
        for i in range(len(frames) - 1):
            nxt.append(frames[i])
            nxt.append(mids[i])
        nxt.append(frames[-1])
        frames = nxt
    return frames


# =========================================================================================
# Device-resident data path (GPUs): frames, tiles and gather buffers are torch tensors in
# HBM; the network writes straight into the NCCL all-gather buffer; nothing goes through
# host memory between the network call and the collective.
# =========================================================================================
# `engine_dev(x0, x1, out)`: x0, x1, out are (H, W, 3) float32 tensor VIEWS (row pitch =
# stride(0) floats, inner two dims dense); computes the mid-frame of (x0, x1) into `out`
# asynchronously on the current stream. `device_engine(Interpolator)` builds it from the
# real engine (film_interpolate_device takes row pitches, so a tile of a larger frame and
# a slot of a gather buffer are passed without copies); the gloo tests use a CPU stand-in.

def device_engine(interp):
    """Adapts an `Interpolator` to the `engine_dev(x0, x1, out)` tensor-view interface.

    Stream semantics: the call is ordered after everything already enqueued on torch's CURRENT stream and everything
    enqueued on the current stream afterwards (NCCL collectives, copies) is ordered after it. The engine runs on a
    dedicated side stream joined to the current one with events, because torch's default stream is the NULL handle,
    which `film_interpolate_device` reads as "use the engine's own stream"."""
    import torch
    side = {}

    def run(x0, x1, out):
        h, w, c = x0.shape
        for t in (x0, x1, out):
            assert t.dtype == torch.float32 and t.is_cuda and t.shape == (h, w, 3)
            assert t.stride(2) == 1 and t.stride(1) == 3, "inner dims must be dense (row-pitched view)"
        assert x0.stride(0) == x1.stride(0), "x0 and x1 must share the row pitch"
        dev = x0.device
        if dev not in side:
            side[dev] = torch.cuda.Stream(device=dev)
        es, cur = side[dev], torch.cuda.current_stream(dev)
        es.wait_stream(cur)
        interp.interpolate_device(x0.data_ptr(), x1.data_ptr(), 1, h, w, out.data_ptr(),
                                  in_pitch=x0.stride(0), out_pitch=out.stride(0), stream=es.cuda_stream)
        cur.wait_stream(es)
        for t in (x0, x1, out):
            t.record_stream(es)

    def at(x0, x1, times, out):
        """Frames of (x0, x1) at `times` (`Interpolator.interpolate_at_device`) into the dense (n, H, W, 3) tensor `out`,
        frame i at out[i]; same stream semantics as the network call. The Interpolator must be untiled."""
        h, w, _ = x0.shape
        n = len(times)
        for t in (x0, x1):
            assert t.dtype == torch.float32 and t.is_cuda and t.shape == (h, w, 3)
            assert t.stride(2) == 1 and t.stride(1) == 3, "inner dims must be dense (row-pitched view)"
        assert x0.stride(0) == x1.stride(0), "x0 and x1 must share the row pitch"
        assert out.dtype == torch.float32 and out.is_cuda and out.shape == (n, h, w, 3) and out.is_contiguous()
        dev = x0.device
        if dev not in side:
            side[dev] = torch.cuda.Stream(device=dev)
        es, cur = side[dev], torch.cuda.current_stream(dev)
        es.wait_stream(cur)
        interp.interpolate_at_device(x0.data_ptr(), x1.data_ptr(), times, h, w, out.data_ptr(), in_pitch=x0.stride(0),
                                     out_pitch=w * 3, stream=es.cuda_stream)
        cur.wait_stream(es)
        for t in (x0, x1, out):
            t.record_stream(es)

    def stitch(tiles, slot_of_tile, block_shape, overlap, out):
        """Feathered stitch (film_stitch_tiles_device) of the window results in `tiles` (slots, q_h, q_w, 3), tile t in
        slot slot_of_tile[t], into the (H, W, 3) view `out`; same stream semantics as the network call. The inner three
        dims of `tiles` must be dense; the slots may be further apart (tile_stride = tiles.stride(0)), so a per-time
        slice of a gather buffer is read in place."""
        h, w, _ = out.shape
        qh, qw = tiles.shape[-3], tiles.shape[-2]
        if tiles.dim() != 4:
            assert tiles.is_contiguous(), "tiles must be (slots, q_h, q_w, 3) or contiguous"
            tiles = tiles.view(-1, qh, qw, 3)
        assert tiles.dtype == out.dtype == torch.float32 and tiles.is_cuda
        assert tiles.stride(3) == 1 and tiles.stride(2) == 3 and tiles.stride(1) == qw * 3, "inner dims must be dense"
        assert (qh, qw) == spec.tile_windows(h, w, block_shape, overlap)[1], "tiles do not have the window shape"
        assert max(slot_of_tile) < tiles.shape[0], "slot outside the tile buffer"
        assert out.stride(2) == 1 and out.stride(1) == 3, "inner dims must be dense (row-pitched view)"
        dev = out.device
        if dev not in side:
            side[dev] = torch.cuda.Stream(device=dev)
        es, cur = side[dev], torch.cuda.current_stream(dev)
        es.wait_stream(cur)
        interp.stitch_tiles_device(tiles.data_ptr(), max(tiles.stride(0), qh * qw * 3), h, w, block_shape, overlap,
                                   out.data_ptr(), slot_of_tile=slot_of_tile, out_pitch=out.stride(0),
                                   stream=es.cuda_stream)
        cur.wait_stream(es)
        for t in (tiles, out):
            t.record_stream(es)
    run.at = at
    run.stitch = stitch
    return run


def stitch_tiles_host(tiles, slot_of_tile, block_shape, overlap, out):
    """The `stitch` of a CPU stand-in for `device_engine` (host-logic tests): `spec.stitch_overlapped` on CPU tensors."""
    import torch
    qh, qw = tiles.shape[-3], tiles.shape[-2]
    t = tiles.reshape(-1, qh, qw, 3)[list(slot_of_tile)].numpy()
    res = spec.stitch_overlapped(t, out.shape[0], out.shape[1], block_shape, overlap)[0]
    out.copy_(torch.from_numpy(res.astype(np.float32)))


def _all_gather_slots(buf, group=None):
    """ONE in-place all-gather: `buf` is (world, m, ...) on every rank, rank r has filled
    buf[r]; afterwards every rank holds every slot. The send buffer IS the rank's slice of
    the receive buffer (NCCL in-place all-gather), so nothing is staged."""
    dist = _dist()
    world, rank = _world_rank(group)
    if world > 1:
        dist.all_gather_into_tensor(buf.view(-1), buf[rank].reshape(-1), group=group)
    return buf


def window_view(frame, block_shape, t, overlap):
    """Window of tile t (row-major; `spec.tile_windows`) of a (1, H, W, 3) or (H, W, 3) tensor as a strided view."""
    f = frame[0] if frame.dim() == 4 else frame
    origins, (qh, qw) = spec.tile_windows(f.shape[0], f.shape[1], block_shape, overlap)
    y, x = origins[t]
    return f[y:y + qh, x:x + qw]


def tile_view(frame, block_shape, t):
    """Tile t (row-major, eval/interpolator.py:66-99) of a (1, H, W, 3) or (H, W, 3) tensor as a strided view."""
    return window_view(frame, block_shape, t, 0)


def interpolate_tiled_device(engine_dev, x0, x1, block_shape, group=None, out=None, gather_buf=None, overlap=0):
    """Tiled path with tiles sharded round-robin over ranks, device-resident end to end.

    x0, x1: (1, H, W, 3) tensors resident on every rank's device. Rank r computes tiles
    r, r + world, ... and the network writes each of them directly into slot [r, j] of the
    all-gather buffer; ONE NCCL all-gather; one device copy stitches the rank-major slots
    into the (1, H, W, 3) frame (`out`, allocated if None). Returns `out`.

    overlap > 0: the slots have the window shape of `spec.tile_windows`, every tile runs on its window, and
    `engine_dev.stitch` (the feathered stitch kernel behind `device_engine`; `stitch_tiles_host` for a CPU stand-in)
    reads the rank-major slots in place through a slot table."""
    import torch
    world, rank = _world_rank(group)
    bh, bw = int(block_shape[0]), int(block_shape[1])
    nt = bh * bw
    _, h, w, _ = x0.shape
    ph, pw = spec.tile_windows(h, w, [bh, bw], overlap)[1]
    m = (nt + world - 1) // world
    if gather_buf is None:
        gather_buf = torch.empty((world, m, ph, pw, 3), dtype=torch.float32, device=x0.device)
    for j, t in enumerate(round_robin(nt, world, rank)):
        engine_dev(window_view(x0, block_shape, t, overlap), window_view(x1, block_shape, t, overlap), gather_buf[rank, j])
    _all_gather_slots(gather_buf, group)
    if out is None:
        out = torch.empty((1, h, w, 3), dtype=torch.float32, device=x0.device)
    if overlap:
        # slot [r, j] holds tile j * world + r
        engine_dev.stitch(gather_buf.view(world * m, ph, pw, 3), [(t % world) * m + t // world for t in range(nt)],
                          [bh, bw], overlap, out[0])
        return out
    # slot [r, j] holds tile j * world + r -> tile-major order, then patches_to_image as one strided copy
    tiles = gather_buf.transpose(0, 1).reshape(world * m, ph, pw, 3)[:nt]
    out.view(bh, ph, bw, pw, 3).copy_(tiles.view(bh, bw, ph, pw, 3).permute(0, 2, 1, 3, 4))
    return out


def interpolate_at_tiled_device(engine_dev, x0, x1, times, block_shape, group=None, out=None, gather_buf=None, overlap=0):
    """The times form of `interpolate_tiled_device`: frames of one pair at every t in `times`, tiled, device-resident.

    x0, x1: (1, H, W, 3) or (H, W, 3) tensors resident on every rank's device. Tiles go round-robin over ranks; rank r
    runs `engine_dev.at` (one head and n tails, `device_engine` over an untiled Interpolator) on the windows of
    `spec.tile_windows` of its tiles, straight into slot [r, j] of the (world, m, n, q_h, q_w, 3) gather buffer; ONE
    all-gather; then one `engine_dev.stitch` per time reads that time's slots in place through the slot table (a paste
    at overlap 0). Returns `out`, (n, H, W, 3), allocated if None."""
    import torch
    world, rank = _world_rank(group)
    bh, bw = int(block_shape[0]), int(block_shape[1])
    nt, n = bh * bw, len(times)
    h, w = x0.shape[-3], x0.shape[-2]
    qh, qw = spec.tile_windows(h, w, [bh, bw], overlap)[1]
    m = (nt + world - 1) // world
    if gather_buf is None:
        gather_buf = torch.empty((world, m, n, qh, qw, 3), dtype=torch.float32, device=x0.device)
    for j, t in enumerate(round_robin(nt, world, rank)):
        engine_dev.at(window_view(x0, block_shape, t, overlap), window_view(x1, block_shape, t, overlap), times,
                      gather_buf[rank, j])
    _all_gather_slots(gather_buf, group)
    if out is None:
        out = torch.empty((n, h, w, 3), dtype=torch.float32, device=x0.device)
    slots = [(t % world) * m + t // world for t in range(nt)]   # slot [r, j] holds tile j * world + r
    per_time = gather_buf.view(world * m, n, qh, qw, 3)
    for i in range(n):
        engine_dev.stitch(per_time[:, i], slots, [bh, bw], overlap, out[i])
    return out


def interpolate_pairs_device(engine_dev, x0, x1, group=None, gather_buf=None):
    """Mid-frames of N independent pairs (x0[i], x1[i]) -- (N, H, W, 3) tensors resident on
    every rank -- block-partitioned over ranks, one in-place all-gather. Returns (N, H, W, 3)."""
    import torch
    world, rank = _world_rank(group)
    n, h, w, _ = x0.shape
    m = (n + world - 1) // world
    if gather_buf is None:
        gather_buf = torch.empty((world, m, h, w, 3), dtype=torch.float32, device=x0.device)
    lo, hi = block_partition(n, world, rank)
    for j, i in enumerate(range(lo, hi)):
        engine_dev(x0[i], x1[i], gather_buf[rank, j])
    _all_gather_slots(gather_buf, group)
    if world == 1:
        return gather_buf[0, :n]
    parts = [gather_buf[r, : block_partition(n, world, r)[1] - block_partition(n, world, r)[0]] for r in range(world)]
    return torch.cat(parts, dim=0)


def interpolate_recursively_device(engine_dev, frame0, frame1, times_to_interpolate, group=None):
    """Level-synchronous recursion (eval/util.py:62-91) with every frame resident in HBM on
    every rank: returns the (2^n + 1, H, W, 3) display-order sequence. At level k the
    2^(k-1) independent calls read their parents from the sequence buffer, write into the
    level's gather buffer, are all-gathered in place (device to device over NVLink) and
    scattered to their positions in the sequence."""
    import torch
    world, rank = _world_rank(group)
    n = (1 << int(times_to_interpolate)) + 1
    h, w, _ = frame0.shape
    seq = torch.empty((n, h, w, 3), dtype=torch.float32, device=frame0.device)
    seq[0].copy_(frame0)
    seq[n - 1].copy_(frame1)
    step = (n - 1) // 2
    while step >= 1:
        idx = list(range(step, n - 1, 2 * step))           # positions of this level's mid-frames
        cnt = len(idx)
        m = (cnt + world - 1) // world
        buf = torch.empty((world, m, h, w, 3), dtype=torch.float32, device=seq.device)
        lo, hi = block_partition(cnt, world, rank)
        for j, k in enumerate(range(lo, hi)):
            i = idx[k]
            engine_dev(seq[i - step], seq[i + step], buf[rank, j])
        _all_gather_slots(buf, group)
        for r in range(world):
            rlo, rhi = block_partition(cnt, world, r)
            if rhi > rlo:
                # idx[rlo:rhi] is an arithmetic progression: one strided copy per rank
                seq[idx[rlo]:idx[rhi - 1] + 1:2 * step].copy_(buf[r, : rhi - rlo])
        step //= 2
    return seq
