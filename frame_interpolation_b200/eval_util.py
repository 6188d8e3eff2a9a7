"""Frame scheduling and image I/O on top of the engine's `Interpolator`.

Counterpart of the reference's `eval/util.py:29-153` without TensorFlow:
  read_image / write_image                    eval/util.py:29-59   (cv2 instead of tf.io)
  interpolate_recursively_from_files/_memory  eval/util.py:94-153
The yielded sequence is the reference's: for every consecutive input pair the in-order
traversal of the mid-point tree (first frame included, second excluded), then the last frame.

When the interpolator is the untiled engine, each pair's whole tree is evaluated by ONE
device-resident call (`Interpolator.interpolate_recursively`): intermediate frames never leave
HBM, which removes the per-mid-frame H2D + D2H + sync the reference pays
(eval/interpolator.py:171,176). Any other callable `(x0, x1, dt) -> mid` takes the generic path.

Frame-rate conversion (no reference counterpart): `retime_schedule` places every output frame of the target rate
in a pair of input frames at an exact fractional time, and `retime_from_files` renders the sequence with one
`interpolate_at` call per pair that needs frames.
"""
from __future__ import annotations

import os
import shutil
from fractions import Fraction
from typing import Callable, Iterable, Iterator, List, Sequence, Tuple, Union

import numpy as np

_UINT8_MAX_F = 255.0


def read_image(filename: str) -> np.ndarray:
    """8-bit sRGB image file -> float32 (H, W, 3) RGB in [0, 1]."""
    import cv2
    # BGR, uint8, alpha dropped, gray replicated; EXIF orientation ignored like tf.io.decode_image does
    data = cv2.imread(filename, cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION)
    if data is None:
        raise FileNotFoundError(f"cannot read image {filename}")
    rgb = np.ascontiguousarray(data[..., ::-1])
    return rgb.astype(np.float32) / np.float32(_UINT8_MAX_F)


def to_uint8(image: np.ndarray) -> np.ndarray:
    """The reference's quantisation (eval/util.py:51-52): clip(x*255, 0, 255) + 0.5, truncated."""
    scaled = np.clip(image * _UINT8_MAX_F, 0.0, _UINT8_MAX_F)
    return (scaled + 0.5).astype(np.uint8)


def write_image(filename: str, image: np.ndarray) -> None:
    """float32 (H, W, 3) RGB in [0, 1] -> .png (default) or .jpg by extension."""
    import cv2
    bgr = np.ascontiguousarray(to_uint8(image)[..., ::-1])
    ext = os.path.splitext(filename)[1].lower()
    if ext not in (".jpg", ".jpeg", ".png"):
        ok, buf = cv2.imencode(".png", bgr)
        if not ok:
            raise IOError(f"cannot encode {filename}")
        with open(filename, "wb") as f:
            f.write(buf.tobytes())
        return
    if not cv2.imwrite(filename, bgr):
        raise IOError(f"cannot write {filename}")


def _pair_sequence(frame_a: np.ndarray, frame_b: np.ndarray, times: int, interpolator: Callable,
                   on_frame=None) -> List[np.ndarray]:
    """Frames from frame_a (included) up to frame_b (excluded), 2**times of them, in display order."""
    fast = getattr(interpolator, "interpolate_recursively", None)
    tiled = getattr(interpolator, "_block_shape", None)
    if fast is not None and (tiled is None or int(np.prod(tiled)) <= 1) and times > 0:
        seq = fast(frame_a, frame_b, times)
        if on_frame:
            on_frame((1 << times) - 1)
        # copies, not views: `seq` is one page-locked (2^times + 1)-frame buffer of the engine's pool, and a caller
        # holding a single frame must not keep hundreds of MB of pinned memory alive
        return [np.array(seq[i]) for i in range(seq.shape[0] - 1)]
    # generic path: explicit stack instead of recursion, same calls and same order of results
    dt = np.full((1,), 0.5, np.float32)
    frames = [frame_a, frame_b]
    for _ in range(times):
        nxt = []
        for left, right in zip(frames[:-1], frames[1:]):
            nxt.append(left)
            nxt.append(interpolator(left[np.newaxis], right[np.newaxis], dt)[0])
            if on_frame:
                on_frame(1)
        nxt.append(frames[-1])
        frames = nxt
    return frames[:-1]


def interpolate_recursively_from_memory(frames: Sequence[np.ndarray], times_to_interpolate: int,
                                        interpolator: Callable, progress=None) -> Iterator[np.ndarray]:
    """Yields the interpolated sequence (inputs included) for in-memory (H, W, 3) frames."""
    for a, b in zip(frames[:-1], frames[1:]):
        yield from _pair_sequence(a, b, times_to_interpolate, interpolator, progress)
    yield frames[-1]


def interpolate_recursively_from_files(frames: Sequence[str], times_to_interpolate: int,
                                       interpolator: Callable, progress=None) -> Iterator[np.ndarray]:
    """Same, loading the input files on demand (each file is decoded once)."""
    prev = read_image(frames[0])
    for name in frames[1:]:
        cur = read_image(name)
        yield from _pair_sequence(prev, cur, times_to_interpolate, interpolator, progress)
        prev = cur
    yield prev


Rate = Union[int, str, Fraction]


def parse_rate(r: Rate) -> Fraction:
    """A frame rate as an exact fraction: 30, "30", "29.97" or "24000/1001"."""
    f = r if isinstance(r, Fraction) else Fraction(str(r))
    assert f > 0, f"frame rates must be positive, got {r!r}"
    return f


def retime_schedule(n_frames: int, source_fps: Rate, target_fps: Rate) -> List[Tuple[int, Fraction]]:
    """Output frame j of a clip of `n_frames` input frames converted from `source_fps` to `target_fps` sits at the
    input position pos = j * source / target, for j = 0 .. floor((n_frames - 1) * target / source). Entry j is
    (i, t): input pair (i, i + 1) at the exact time t = pos - i, i = floor(pos). t = 0 is input frame i itself
    (the last input frame has i = n_frames - 1)."""
    assert n_frames >= 1, "a clip needs at least one frame"
    step = parse_rate(source_fps) / parse_rate(target_fps)
    out = []
    pos = Fraction(0)
    while pos <= n_frames - 1:
        i = pos.numerator // pos.denominator
        out.append((i, pos - i))
        pos += step
    return out


def retime_from_files(frames: Sequence[str], source_fps: Rate, target_fps: Rate, interpolator,
                      progress=None, at: Callable | None = None) -> Iterator[np.ndarray]:
    """Yields the clip `frames` (image files) retimed from `source_fps` to `target_fps` (see `retime_schedule`).
    Every input pair that needs frames strictly between its ends gets ONE `at(frame_i, frame_i1, times)` call for all
    of them (default `interpolator.interpolate_at`; `interpolator.interpolate_at_tiled` for tiles); t = 0 yields the
    input frame without a network call. Only the current pair is held in memory, and each file is decoded once."""
    if at is None:
        at = interpolator.interpolate_at
    sched = retime_schedule(len(frames), source_fps, target_fps)
    cur_i, cur, nxt = -1, None, None
    k = 0
    while k < len(sched):
        i = sched[k][0]
        if i != cur_i:  # advance to pair i: reuse the decoded right frame of the previous pair when it is frame i
            cur = nxt if (nxt is not None and cur_i + 1 == i) else read_image(frames[i])
            nxt = None
            cur_i = i
        ts = []
        while k < len(sched) and sched[k][0] == i:
            ts.append(sched[k][1])
            k += 1
        inner = [t for t in ts if t != 0]
        mids = []
        if inner:
            nxt = read_image(frames[i + 1])
            mids = at(cur, nxt, [float(t) for t in inner])
            if progress:
                progress(len(inner))
        m = 0
        for t in ts:
            if t == 0:
                yield cur
            else:
                # a copy, not a view: the result is one page-locked buffer of the engine's pool
                yield np.array(mids[m])
                m += 1


def natural_sorted(names: Iterable[str]) -> List[str]:
    """natsort.natsorted stand-in: digit runs compare numerically."""
    import re

    def key(s):
        return [int(t) if t.isdigit() else t.lower() for t in re.split(r"(\d+)", s)]
    return sorted(names, key=key)


def get_ffmpeg_path() -> str:
    path = shutil.which("ffmpeg")
    if not path:
        raise RuntimeError("Program 'ffmpeg' is not found; it is only needed for --output_video.")
    return path
