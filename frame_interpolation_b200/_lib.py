"""ctypes binding of libfilm_b200.so (C ABI in include/film_b200.h).

The library is built in-tree by `frame_interpolation_b200.build`. Loading fails loudly
if it is missing: there is no Python / CPU fallback for the engine.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfilm_b200.so")

EXPORTS = [
    "film_create", "film_destroy", "film_interpolate", "film_interpolate_tiled",
    "film_interpolate_device", "film_interpolate_recursive", "film_host_alloc", "film_host_free",
    "film_synchronize", "film_profile", "film_set_option",
    "film_debug_read", "film_op_table", "film_last_error", "film_version",
    "film_get_option", "film_stage_count", "film_stage_name",
    "film_interpolate_u8", "film_interpolate_recursive_u8", "film_stitch_tiles_device",
    "film_interpolate_times", "film_interpolate_times_device", "film_interpolate_times_tiled",
]


class FilmProfile(C.Structure):
    _fields_ = [
        ("last_call_ms", C.c_double), ("last_h2d_ms", C.c_double), ("last_d2h_ms", C.c_double),
        ("conv_flops", C.c_double), ("mma_flops", C.c_double), ("warp_bytes", C.c_double),
        ("kernel_launches", C.c_int64), ("arena_bytes", C.c_int64),
        ("padded_h", C.c_int32), ("padded_w", C.c_int32), ("used_graph", C.c_int32),
        ("reserved", C.c_int32),
    ]


_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -m frame_interpolation_b200.build` "
            "(the FILM engine has no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    fp = C.POINTER(C.c_float)
    lib.film_create.argtypes = [C.POINTER(C.c_void_p), C.c_char_p, C.c_int]
    lib.film_create.restype = C.c_int
    lib.film_destroy.argtypes = [C.c_void_p]
    lib.film_destroy.restype = None
    lib.film_interpolate.argtypes = [C.c_void_p, fp, fp, fp, C.c_int, C.c_int, C.c_int, C.c_int, fp]
    lib.film_interpolate.restype = C.c_int
    lib.film_interpolate_tiled.argtypes = [C.c_void_p, fp, fp, fp, C.c_int, C.c_int, C.c_int,
                                           C.c_int, C.c_int, fp]
    lib.film_interpolate_tiled.restype = C.c_int
    lib.film_interpolate_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                            C.c_int, C.c_int64, C.c_int, C.c_void_p, C.c_int64,
                                            C.c_void_p]
    lib.film_interpolate_device.restype = C.c_int
    lib.film_stitch_tiles_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int), C.c_int, C.c_int,
                                             C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    lib.film_stitch_tiles_device.restype = C.c_int
    lib.film_interpolate_times.argtypes = [C.c_void_p, fp, fp, fp, C.c_int, C.c_int, C.c_int, C.c_int, fp]
    lib.film_interpolate_times.restype = C.c_int
    lib.film_interpolate_times_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, fp, C.c_int, C.c_int, C.c_int,
                                                  C.c_int64, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    lib.film_interpolate_times_device.restype = C.c_int
    lib.film_interpolate_times_tiled.argtypes = [C.c_void_p, fp, fp, fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                                 C.c_int, fp]
    lib.film_interpolate_times_tiled.restype = C.c_int
    lib.film_interpolate_recursive.argtypes = [C.c_void_p, fp, fp, C.c_int, C.c_int, C.c_int, C.c_int, fp]
    lib.film_interpolate_recursive.restype = C.c_int
    up = C.POINTER(C.c_uint8)
    lib.film_interpolate_u8.argtypes = [C.c_void_p, up, up, C.c_int, C.c_int, C.c_int, C.c_int, up]
    lib.film_interpolate_u8.restype = C.c_int
    lib.film_interpolate_recursive_u8.argtypes = [C.c_void_p, up, up, C.c_int, C.c_int, C.c_int, C.c_int, up]
    lib.film_interpolate_recursive_u8.restype = C.c_int
    lib.film_host_alloc.argtypes = [C.c_size_t]
    lib.film_host_alloc.restype = C.c_void_p
    lib.film_host_free.argtypes = [C.c_void_p]
    lib.film_host_free.restype = None
    lib.film_synchronize.argtypes = [C.c_void_p]
    lib.film_synchronize.restype = C.c_int
    lib.film_profile.argtypes = [C.c_void_p, C.POINTER(FilmProfile)]
    lib.film_profile.restype = C.c_int
    lib.film_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
    lib.film_set_option.restype = C.c_int
    lib.film_get_option.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_int)]
    lib.film_get_option.restype = C.c_int
    lib.film_stage_count.argtypes = []
    lib.film_stage_count.restype = C.c_int
    lib.film_stage_name.argtypes = [C.c_int, C.c_char_p, C.c_int]
    lib.film_stage_name.restype = C.c_int
    lib.film_debug_read.argtypes = [C.c_void_p, C.c_char_p, fp, C.POINTER(C.c_int64)]
    lib.film_debug_read.restype = C.c_int
    lib.film_op_table.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.POINTER(C.c_int64)]
    lib.film_op_table.restype = C.c_int
    lib.film_last_error.argtypes = [C.c_void_p]
    lib.film_last_error.restype = C.c_char_p
    lib.film_version.argtypes = []
    lib.film_version.restype = C.c_char_p
    _lib = lib
    return lib
