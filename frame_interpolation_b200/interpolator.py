"""Drop-in for the reference's `eval/interpolator.py` on top of the H100 engine.

Same class name, constructor arguments, methods, argument meaning and error behaviour
as `eval.interpolator.Interpolator` (reference eval/interpolator.py:129-209):

    Interpolator(model_path, align=None, block_shape=None)
    .interpolate(x0, x1, dt) -> np.ndarray      # eval/interpolator.py:152-176
    .__call__(x0, x1, dt)    -> np.ndarray      # eval/interpolator.py:178-209 (tiled if prod(block_shape) > 1)

`model_path` names a FILMW1 weight file (frame_interpolation_b200/weights.py) instead of
a TF2 SavedModel directory; the string "synthetic" (or "synthetic:<seed>") selects the
seeded synthetic Style-architecture weights used by the tests and benchmarks.

All arithmetic runs in libfilm_b200.so (hand-written sm_90a kernels) through the C ABI
of include/film_b200.h. No TensorFlow, no torch, no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional

import numpy as np

from . import _lib, weights as _weights


def _fptr(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def image_to_patches(image: np.ndarray, block_shape: List[int]) -> np.ndarray:
    """eval/interpolator.py:66-99 (host-side helper kept for API parity)."""
    block_height, block_width = block_shape
    height, width, channel = image.shape[-3:]
    patch_height, patch_width = height // block_height, width // block_width
    assert height == (patch_height * block_height), \
        'block_height=%d should evenly divide height=%d.' % (block_height, height)
    assert width == (patch_width * block_width), \
        'block_width=%d should evenly divide width=%d.' % (block_width, width)
    x = np.reshape(image, (block_height, patch_height, block_width, patch_width, channel))
    x = np.transpose(x, (0, 2, 1, 3, 4))
    return np.ascontiguousarray(np.reshape(x, (block_height * block_width, patch_height, patch_width, channel)))


def patches_to_image(patches: np.ndarray, block_shape: List[int]) -> np.ndarray:
    """eval/interpolator.py:102-126."""
    block_height, block_width = block_shape
    patch_height, patch_width, channel = patches.shape[-3:]
    x = np.reshape(patches, (block_height, block_width, patch_height, patch_width, channel))
    x = np.transpose(x, (0, 2, 1, 3, 4))
    return np.ascontiguousarray(np.reshape(x, (1, block_height * patch_height, block_width * patch_width, channel)))


class _PinnedPool:
    """Pinned (page-locked) result buffers. A returned ndarray owns its buffer through a
    finalizer: when the caller drops the array the buffer goes back to the pool (at most
    `keep` idle buffers per size are retained, the rest are freed)."""

    def __init__(self, lib, keep: int = 4):
        self._lib = lib
        self._keep = keep
        self._idle = {}

    def _release(self, nbytes: int, ptr: int) -> None:
        idle = self._idle.setdefault(nbytes, [])
        if len(idle) < self._keep:
            idle.append(ptr)
        else:
            self._lib.film_host_free(C.c_void_p(ptr))

    def empty(self, shape) -> np.ndarray:
        import weakref
        n = int(np.prod(shape))
        nbytes = n * 4
        idle = self._idle.get(nbytes)
        ptr = idle.pop() if idle else self._lib.film_host_alloc(nbytes)
        if not ptr:
            return np.empty(shape, np.float32)           # pinned allocation failed: plain memory still works
        buf = (C.c_float * n).from_address(ptr)
        arr = np.ctypeslib.as_array(buf).reshape(shape)
        weakref.finalize(buf, self._release, nbytes, ptr)  # `buf` lives as long as any view of `arr`
        return arr

    def close(self) -> None:
        for ptrs in self._idle.values():
            for ptr in ptrs:
                self._lib.film_host_free(C.c_void_p(ptr))
        self._idle = {}


class Interpolator:
    """A class for generating interpolated frames between two input frames (H100 engine)."""

    def __init__(self, model_path: str, align: Optional[int] = None,
                 block_shape: Optional[List[int]] = None, device: int = 0) -> None:
        self._lib = _lib.load()
        if model_path is None:
            # the reference fails without a SavedModel; silently substituting random weights would produce
            # plausible-looking garbage frames
            raise ValueError("model_path is required: a FILMW1 weight file (tf_bundle.convert_saved_model), or the "
                             "explicit string 'synthetic[:seed]' for seeded random weights (tests / benchmarks only)")
        if str(model_path).startswith("synthetic"):
            seed = 1234
            if ":" in str(model_path):
                seed = int(str(model_path).split(":", 1)[1])
            model_path = _weights.ensure_synthetic_file(seed=seed)
        self._handle = C.c_void_p()
        st = self._lib.film_create(C.byref(self._handle), str(model_path).encode(), int(device))
        if st != 0:
            msg = self._lib.film_last_error(None).decode()
            self._handle = C.c_void_p()
            raise RuntimeError(f"film_create failed (status {st}): {msg}")
        self._align = align or None
        self._block_shape = block_shape or None
        self.device = int(device)
        self._pool = _PinnedPool(self._lib)

    # -- lifecycle ------------------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "_handle", None) is not None and self._handle.value:
            self._lib.film_destroy(self._handle)
            self._handle = C.c_void_p()
            if getattr(self, "_pool", None) is not None:
                self._pool.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st: int) -> None:
        if st == 0:
            return
        msg = self._lib.film_last_error(self._handle).decode()
        if st == 1:
            # the reference raises AssertionError from its shape / divisibility asserts
            raise AssertionError(msg)
        raise RuntimeError(f"film engine error (status {st}): {msg}")

    @staticmethod
    def _prep(x0, x1, dt):
        # eval/interpolator.py:43-44
        assert np.ndim(x0) == 4 and np.ndim(x1) == 4, "expected (batch, height, width, channels)"
        x0 = np.ascontiguousarray(x0, dtype=np.float32)
        x1 = np.ascontiguousarray(x1, dtype=np.float32)
        assert x0.shape == x1.shape, "x0 and x1 must have the same shape"
        assert x0.shape[-1] == 3, "expected 3 colour channels"
        dt = np.ascontiguousarray(dt, dtype=np.float32).reshape(-1)
        assert dt.shape[0] == x0.shape[0], "dt must have one entry per batch element"
        return x0, x1, dt

    # -- reference API --------------------------------------------------------------
    def interpolate(self, x0: np.ndarray, x1: np.ndarray, dt: np.ndarray) -> np.ndarray:
        """Generates an interpolated frame between given two batches of frames.

        x0, x1: (batch, height, width, 3) float32; dt: (batch,), ignored by the network
        exactly like the reference (models/film_net/interpolator.py:102). Returns the
        unclipped (batch, height, width, 3) float32 mid-frame.
        """
        if self._align is not None:
            assert self._align > 0, 'align must be a positive number.'
        x0, x1, dt = self._prep(x0, x1, dt)
        b, h, w, _ = x0.shape
        out = self._pool.empty(x0.shape)
        st = self._lib.film_interpolate(self._handle, _fptr(x0), _fptr(x1), _fptr(dt), b, h, w,
                                        int(self._align or 0), _fptr(out))
        self._check(st)
        return out

    def __call__(self, x0: np.ndarray, x1: np.ndarray, dt: np.ndarray) -> np.ndarray:
        if self._block_shape is not None and np.prod(self._block_shape) > 1:
            if self._align is not None:
                assert self._align > 0, 'align must be a positive number.'
            x0, x1, dt = self._prep(x0, x1, dt)
            # the reference's reshape at eval/interpolator.py:97-98 is only valid for batch 1
            assert x0.shape[0] == 1, "tiled interpolation expects batch size 1"
            _, h, w, _ = x0.shape
            bh, bw = int(self._block_shape[0]), int(self._block_shape[1])
            out = self._pool.empty(x0.shape)
            st = self._lib.film_interpolate_tiled(self._handle, _fptr(x0), _fptr(x1), _fptr(dt), h, w,
                                                  int(self._align or 0), bh, bw, _fptr(out))
            self._check(st)
            return out
        return self.interpolate(x0, x1, dt)

    # -- engine extras (no reference counterpart) ------------------------------------
    def interpolate_device(self, d_x0: int, d_x1: int, batch: int, height: int, width: int,
                           d_out: int, in_pitch: Optional[int] = None,
                           out_pitch: Optional[int] = None, stream: int = 0) -> None:
        """Device-pointer path (raw addresses, e.g. torch.Tensor.data_ptr()); asynchronous."""
        in_pitch = in_pitch or width * 3
        out_pitch = out_pitch or width * 3
        st = self._lib.film_interpolate_device(self._handle, C.c_void_p(d_x0), C.c_void_p(d_x1), batch,
                                               height, width, in_pitch, int(self._align or 0),
                                               C.c_void_p(d_out), out_pitch, C.c_void_p(stream))
        self._check(st)

    def stitch_tiles_device(self, d_tiles: int, tile_stride: int, height: int, width: int, block_shape: List[int],
                            overlap: int, d_out: int, slot_of_tile: Optional[List[int]] = None,
                            out_pitch: Optional[int] = None, stream: int = 0) -> None:
        """Feathered stitch of overlapped window results on the device (film_stitch_tiles_device; geometry in
        `spec.tile_windows`); asynchronous. Tile t is read at d_tiles + slot_of_tile[t] * tile_stride floats (identity
        if None); the (height, width, 3) frame is written at d_out with row pitch `out_pitch` floats."""
        bh, bw = int(block_shape[0]), int(block_shape[1])
        slots = None
        if slot_of_tile is not None:
            assert len(slot_of_tile) == bh * bw, "slot_of_tile needs one entry per tile"
            slots = (C.c_int * (bh * bw))(*[int(s) for s in slot_of_tile])
        st = self._lib.film_stitch_tiles_device(self._handle, C.c_void_p(d_tiles), int(tile_stride), slots, int(height),
                                                int(width), bh, bw, int(overlap), C.c_void_p(d_out),
                                                int(out_pitch or width * 3), C.c_void_p(stream))
        self._check(st)

    def interpolate_recursively(self, frame0: np.ndarray, frame1: np.ndarray,
                                times_to_interpolate: int) -> np.ndarray:
        """All frames between two (H, W, 3) frames, end points included, in display order:
        (2**times + 1, H, W, 3). The recursion of eval/util.py:62-91 runs with every
        intermediate frame resident on the device (film_interpolate_recursive). Only for the
        untiled path; bit-identical to recursive calls of `__call__`."""
        if self._align is not None:
            assert self._align > 0, 'align must be a positive number.'
        assert self._block_shape is None or np.prod(self._block_shape) <= 1, \
            "device-resident recursion is the untiled path"
        f0 = np.ascontiguousarray(frame0, dtype=np.float32)
        f1 = np.ascontiguousarray(frame1, dtype=np.float32)
        assert f0.ndim == 3 and f0.shape == f1.shape and f0.shape[-1] == 3, "expected two (H, W, 3) frames"
        h, w, _ = f0.shape
        n = (1 << int(times_to_interpolate)) + 1
        out = self._pool.empty((n, h, w, 3))
        st = self._lib.film_interpolate_recursive(self._handle, _fptr(f0), _fptr(f1), h, w,
                                                  int(self._align or 0), int(times_to_interpolate), _fptr(out))
        self._check(st)
        return out

    @staticmethod
    def _times(times) -> np.ndarray:
        return np.ascontiguousarray(np.asarray(times, dtype=np.float32).reshape(-1))

    def interpolate_at(self, frame0: np.ndarray, frame1: np.ndarray, times) -> np.ndarray:
        """Frames at arbitrary times between two (H, W, 3) frames: (len(times), H, W, 3) float32, frame i at times[i]
        (each finite, 0 <= t <= 1). Frame i is the reference graph with its mid_time 0.5 replaced by times[i]
        (film_interpolate_times): the features and both flow pyramids are computed once, the time-scaled warps and the
        fusion decoder once per time. Bit-identical to `__call__` at t = 0.5; away from 0.5 the quality depends on the
        weights, which the reference trained at t = 0.5 only. Untiled path: a tiled engine uses `interpolate_at_tiled`."""
        if self._align is not None:
            assert self._align > 0, 'align must be a positive number.'
        assert self._block_shape is None or np.prod(self._block_shape) <= 1, "interpolation at times is the untiled path"
        f0, f1, t = self._times_args(frame0, frame1, times)
        h, w, _ = f0.shape
        out = self._pool.empty((max(t.shape[0], 1), h, w, 3))
        st = self._lib.film_interpolate_times(self._handle, _fptr(f0), _fptr(f1), _fptr(t), t.shape[0], h, w,
                                              int(self._align or 0), _fptr(out))
        self._check(st)
        return out

    def interpolate_at_tiled(self, frame0: np.ndarray, frame1: np.ndarray, times) -> np.ndarray:
        """`interpolate_at` on the engine's tiles (block_shape, None meaning [1, 1], and option tile_overlap):
        (len(times), H, W, 3) float32, frame i what `__call__` computes on the tiles with every window's mid_time
        replaced by times[i] (film_interpolate_times_tiled). One head and n tails per window, one stitch per time.
        Bit-identical to `__call__` at t = 0.5; at tile_overlap 0, tile k of frame i is `interpolate_at` on tile k's
        crop."""
        if self._align is not None:
            assert self._align > 0, 'align must be a positive number.'
        f0, f1, t = self._times_args(frame0, frame1, times)
        h, w, _ = f0.shape
        bh, bw = (int(self._block_shape[0]), int(self._block_shape[1])) if self._block_shape is not None else (1, 1)
        out = self._pool.empty((max(t.shape[0], 1), h, w, 3))
        st = self._lib.film_interpolate_times_tiled(self._handle, _fptr(f0), _fptr(f1), _fptr(t), t.shape[0], h, w,
                                                    int(self._align or 0), bh, bw, _fptr(out))
        self._check(st)
        return out

    def _times_args(self, frame0, frame1, times):
        f0 = np.ascontiguousarray(frame0, dtype=np.float32)
        f1 = np.ascontiguousarray(frame1, dtype=np.float32)
        assert f0.ndim == 3 and f0.shape == f1.shape and f0.shape[-1] == 3, "expected two (H, W, 3) frames"
        return f0, f1, self._times(times)

    def interpolate_at_device(self, d_x0: int, d_x1: int, times, height: int, width: int, d_out: int,
                              in_pitch: Optional[int] = None, out_pitch: Optional[int] = None, stream: int = 0) -> None:
        """`interpolate_at` on device pointers (raw addresses, e.g. torch.Tensor.data_ptr()); asynchronous. Frame i is
        written at d_out + i * height * out_pitch floats; `times` is read before the call returns."""
        assert self._block_shape is None or np.prod(self._block_shape) <= 1, "interpolation at times is the untiled path"
        t = self._times(times)
        in_pitch = in_pitch or width * 3
        out_pitch = out_pitch or width * 3
        st = self._lib.film_interpolate_times_device(self._handle, C.c_void_p(d_x0), C.c_void_p(d_x1), _fptr(t),
                                                     t.shape[0], height, width, in_pitch, int(self._align or 0),
                                                     C.c_void_p(d_out), out_pitch, C.c_void_p(stream))
        self._check(st)

    def interpolate_u8(self, x0: np.ndarray, x1: np.ndarray) -> np.ndarray:
        """8-bit in / 8-bit out: (B, H, W, 3) uint8 frames; the /255 of `read_image` (eval/util.py:38-41) and the
        quantisation of `write_image` (eval/util.py:51-52) run on the device, so PCIe carries a quarter of the bytes.
        Bit-identical to `to_uint8(self(x0 / 255, x1 / 255, dt))`. Untiled path."""
        if self._align is not None:
            assert self._align > 0, 'align must be a positive number.'
        assert np.ndim(x0) == 4 and np.ndim(x1) == 4, "expected (batch, height, width, channels)"
        x0 = np.ascontiguousarray(x0, dtype=np.uint8)
        x1 = np.ascontiguousarray(x1, dtype=np.uint8)
        assert x0.shape == x1.shape and x0.shape[-1] == 3
        b, h, w, _ = x0.shape
        out = np.empty(x0.shape, np.uint8)
        up = C.POINTER(C.c_uint8)
        st = self._lib.film_interpolate_u8(self._handle, x0.ctypes.data_as(up), x1.ctypes.data_as(up), b, h, w,
                                           int(self._align or 0), out.ctypes.data_as(up))
        self._check(st)
        return out

    def interpolate_recursively_u8(self, frame0: np.ndarray, frame1: np.ndarray, times_to_interpolate: int) -> np.ndarray:
        """`interpolate_recursively` with uint8 frames at the boundary: (2**times + 1, H, W, 3) uint8, end points included.
        The recursion runs on the unquantised float32 mid-frames (eval/util.py:85-91); only the returned frames are quantised."""
        if self._align is not None:
            assert self._align > 0, 'align must be a positive number.'
        f0 = np.ascontiguousarray(frame0, dtype=np.uint8)
        f1 = np.ascontiguousarray(frame1, dtype=np.uint8)
        assert f0.ndim == 3 and f0.shape == f1.shape and f0.shape[-1] == 3, "expected two (H, W, 3) uint8 frames"
        h, w, _ = f0.shape
        n = (1 << int(times_to_interpolate)) + 1
        out = np.empty((n, h, w, 3), np.uint8)
        up = C.POINTER(C.c_uint8)
        st = self._lib.film_interpolate_recursive_u8(self._handle, f0.ctypes.data_as(up), f1.ctypes.data_as(up), h, w,
                                                     int(self._align or 0), int(times_to_interpolate), out.ctypes.data_as(up))
        self._check(st)
        return out

    def synchronize(self) -> None:
        self._check(self._lib.film_synchronize(self._handle))

    def set_option(self, name: str, value: int) -> None:
        self._check(self._lib.film_set_option(self._handle, name.encode(), int(value)))

    def get_option(self, name: str) -> int:
        v = C.c_int()
        self._check(self._lib.film_get_option(self._handle, name.encode(), C.byref(v)))
        return int(v.value)

    def stage_names(self) -> List[str]:
        """Stages of the precision plan; index = bit in the "onepass_mask" option."""
        out = []
        for i in range(self._lib.film_stage_count()):
            buf = C.create_string_buffer(32)
            self._lib.film_stage_name(i, buf, 32)
            out.append(buf.value.decode())
        return out

    def clear_cache(self) -> None:
        """Drops every cached per-shape plan (CUDA graph + activation arena) of this engine; the next call of a
        shape rebuilds it. For services that see many resolutions: plans are never evicted otherwise."""
        self.set_option("clear_plans", 1)

    def profile(self) -> dict:
        p = _lib.FilmProfile()
        self._check(self._lib.film_profile(self._handle, C.byref(p)))
        return {k: getattr(p, k) for k, _ in p._fields_ if k != "reserved"}

    def debug_read(self, name: str) -> np.ndarray:
        n = C.c_int64()
        self._check(self._lib.film_debug_read(self._handle, name.encode(), None, C.byref(n)))
        out = np.empty(n.value, np.float32)
        self._check(self._lib.film_debug_read(self._handle, name.encode(), _fptr(out), C.byref(n)))
        return out

    def op_table(self) -> List[dict]:
        """Per-kernel table of the last call (ms filled when option time_ops=1)."""
        n = C.c_int64()
        self._check(self._lib.film_op_table(self._handle, None, 0, C.byref(n)))
        buf = C.create_string_buffer(n.value)
        self._check(self._lib.film_op_table(self._handle, buf, n.value, C.byref(n)))
        rows = buf.value.decode().strip().split("\n")
        keys = rows[0].split(",")
        out = []
        for r in rows[1:]:
            v = r.split(",")
            out.append({"idx": int(v[0]), "category": int(v[1]), "name": v[2], "ms": float(v[3]),
                        "ref_flops": float(v[4]), "alg_bytes": float(v[5]), "form": v[6],
                        "passes": int(v[7]) if v[7] else None})
        return out

    @property
    def version(self) -> str:
        return self._lib.film_version().decode()
