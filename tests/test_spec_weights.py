"""Architecture tables, weight file format and the C-ABI surface. CPU only."""
import os
import re

import numpy as np
import pytest

from frame_interpolation_b200 import spec, weights

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_channel_tables_match_survey():
    assert [spec.feature_channels(l) for l in range(7)] == [64, 192, 448, 960, 960, 960, 960]
    assert [spec.aligned_channels(l) for l in range(5)] == [138, 394, 906, 1930, 1930]
    assert [spec.fusion_filters(l) for l in range(4)] == [64, 128, 256, 512]


def test_parameter_count():
    n = sum(int(np.prod(s)) for _, s in spec.weight_table())
    assert n == 34_436_667            # 34.44 M


def test_conv_macs_match_survey_table():
    m = spec.conv_macs(1088, 1920)
    assert round(m["total"] / 1e9, 1) == 4435.1
    assert round(m["feature_extractor"] / 1e9, 1) == 1137.5
    assert round(m["flow"] / 1e9, 1) == 1380.9
    assert round(m["fusion"] / 1e9, 1) == 1916.7
    assert round(spec.conv_macs(768, 1280)["total"] / 1e9, 1) == 2087.1
    assert round(spec.conv_macs(256, 256)["total"] / 1e9, 1) == 139.1


def test_padded_shape():
    assert spec.padded_shape(1080, 1920, 64) == (1088, 1920, 4, 0)
    assert spec.padded_shape(720, 1280, 64) == (768, 1280, 24, 0)
    assert spec.padded_shape(768, 1024, 64) == (768, 1024, 0, 0)
    assert spec.padded_shape(100, 150, None) == (100, 150, 0, 0)


def test_weight_file_round_trip(tmp_path):
    w = weights.synthetic_weights(7)
    p = str(tmp_path / "w.filmw")
    weights.save(p, w)
    r = weights.load(p)
    assert weights.digest(r) == weights.digest(w)
    assert weights.digest(weights.synthetic_weights(7)) == weights.digest(w)      # deterministic
    assert weights.digest(weights.synthetic_weights(8)) != weights.digest(w)
    bad = dict(w)
    bad["fusion/output_conv/bias"] = np.zeros(4, np.float32)
    with pytest.raises(ValueError):
        weights.save(str(tmp_path / "bad.filmw"), bad)
    with open(p, "r+b") as f:
        f.write(b"XXXX")
    with pytest.raises(ValueError):
        weights.load(p)


def test_saved_model_name_mapping():
    w = weights.synthetic_weights(3)
    # emulate SavedModel naming: fusion convs are auto-named conv2d, conv2d_1, ... in creation order
    named = {}
    k = 0
    for name, _ in spec.weight_table():
        if not name.endswith("/kernel"):
            continue
        base = name[:-len("/kernel")]
        if base.startswith("fusion/"):
            tf_name = "fusion/conv2d" + ("" if k == 0 else f"_{k}")
            k += 1
        else:
            tf_name = base
        named[tf_name + "/kernel:0"] = w[base + "/kernel"]
        named[tf_name + "/bias:0"] = w[base + "/bias"]
    assert k == 13
    mapped = weights.from_named_arrays(named)
    assert weights.digest(mapped) == weights.digest(w)


def test_library_exports_every_declared_symbol(built_lib):
    """The C-ABI library loads without a GPU and exports every FILM_API symbol of include/*.h."""
    import ctypes
    hdr = open(os.path.join(ROOT, "include", "film_b200.h")).read()
    declared = re.findall(r"FILM_API\s+[\w\s\*]+?\b(film_\w+)\s*\(", hdr)
    assert len(declared) >= 12
    lib = ctypes.CDLL(built_lib)
    for name in declared:
        assert hasattr(lib, name), name
    from frame_interpolation_b200 import _lib
    assert sorted(_lib.EXPORTS) == sorted(set(declared))
    lib.film_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.film_version()


def test_precision_plan_stage_table(built_lib):
    """The stages of the precision plan are part of the C ABI (bit positions of option "onepass_mask"): 7 feature-extractor
    groups, 7 flow levels, 4 fusion levels x 3 convs, in that order; readable without a GPU."""
    import ctypes
    lib = ctypes.CDLL(built_lib)
    n = lib.film_stage_count()
    assert n == 26
    names = []
    for i in range(n):
        buf = ctypes.create_string_buffer(32)
        assert lib.film_stage_name(i, buf, 32) == 0
        names.append(buf.value.decode())
    assert names[:7] == ["fe_i0_k01", "fe_i0_k23", "fe_i0_k45", "fe_i0_k67", "fe_i1", "fe_i2", "fe_i3p"]
    assert names[7:14] == [f"flow_L{l}" for l in range(7)]
    assert names[14:] == [f"fus{l}_c{c}" for l in range(4) for c in range(3)]
    buf = ctypes.create_string_buffer(4)
    assert lib.film_stage_name(n, buf, 4) != 0 and lib.film_stage_name(-1, buf, 4) != 0      # out of range -> status 1
    assert lib.film_stage_name(0, buf, 4) == 0 and buf.value == b"fe_"                      # truncated, NUL-terminated


def test_engine_fails_loudly_without_gpu(built_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from frame_interpolation_b200.interpolator import Interpolator
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        Interpolator("synthetic", align=64)


def test_product_package_never_imports_oracle():
    pkg = os.path.join(ROOT, "frame_interpolation_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "film_oracle" not in src and "from oracle" not in src and "import oracle" not in src, f
