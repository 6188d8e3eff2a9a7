"""Pixels on the wgmma N dimension for the Cout = 32 layers (option conv3x3_pxn): the single-pass convs of the level-0
flow predictor (flow_conv0@L0 128 -> 32 over 64-channel chunks, flow_conv1@L0 32 -> 32 and flow_conv2+head@L0 32 -> 32
with the fused flow head over 32-channel chunks) run on the folded form, two dy taps of one dx column per M = 64 weight
operand on 32x8 tiles.  They must meet the same bars as the 16x8 form they replace, and must actually run.

The sizes put the level-0 grid at a multiple of 32 rows (256x320), at 32x8 tiles whose last tile row is clipped inside
one consumer warpgroup's 16 rows (100x150, 65x129) and at a last tile row that leaves the second warpgroup with no row
in the frame (176x240).  The flow pyramid at level 0 is read back as well as the frame: the fused flow head writes it."""
import os
import subprocess

import numpy as np
import pytest

from frame_interpolation_b200 import build, synthetic

PLAN = 4e-4         # default precision plan, against the oracle (as test_conv_pixels_on_n.py)
DT = np.full((1,), 0.5, np.float32)
LAYERS = ("flow_conv0@L0", "flow_conv1@L0", "flow_conv2+head@L0")
SIZES = [(256, 320, 64), (100, 150, None), (65, 129, None), (176, 240, 16)]

_HARNESS = r"""
#include <cstdio>
#include "film_pack.h"
int main() {
  const int chunk = CHUNK, ktot = 2 * 9 * chunk;
  std::vector<uint16_t> w((size_t)32 * ktot);
  for (size_t i = 0; i < w.size(); ++i) w[i] = (uint16_t)(i % 65521 + 1);
  for (uint16_t v : film::pack_dy_pairs(w, ktot, chunk)) std::printf("%u\n", (unsigned)v);
}
"""


@pytest.mark.parametrize("chunk", [64, 32])
def test_dy_pair_packing_reproduces_the_per_tap_k_values(tmp_path, chunk):
    """Two chunks of nine dx-major taps: block 2 dx of a chunk holds tap (-1, dx) in rows 0-31 and (0, dx) in rows
    32-63, block 2 dx + 1 zeros in rows 0-31 and tap (+1, dx) below."""
    src = tmp_path / "pack.cpp"
    src.write_text(_HARNESS.replace("CHUNK", str(chunk)))
    exe = tmp_path / "pack"
    subprocess.run([build._nvcc(), "-std=c++17", "-I", build.CSRC, str(src), "-o", str(exe)], check=True,
                   capture_output=True)
    vals = np.array(subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split(), np.int64)
    ktot = 2 * 9 * chunk
    per_tap = (np.arange(32 * ktot) % 65521 + 1).reshape(32, 2, 3, 3, chunk)   # [n][chunk][dx][dy][c]
    got = vals.reshape(64, 2, 3, 2, chunk)                                      # [row][chunk][dx][pair][c]
    np.testing.assert_array_equal(got[:32, :, :, 0], per_tap[:, :, :, 0])
    np.testing.assert_array_equal(got[32:, :, :, 0], per_tap[:, :, :, 1])
    np.testing.assert_array_equal(got[32:, :, :, 1], per_tap[:, :, :, 2])
    assert not got[:32, :, :, 1].any()


@pytest.fixture(scope="module")
def oracles(synthetic_weights):
    import torch
    from oracle.film_oracle import OracleInterpolator
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    return {a: OracleInterpolator(synthetic_weights[1], align=a) for a in (64, None, 16)}


def _engine(synthetic_weights, align, pxn, onepass_mask=None):
    from frame_interpolation_b200.interpolator import Interpolator
    eng = Interpolator(synthetic_weights[0], align=align)
    eng.set_option("any_size", 1)
    eng.set_option("keep_debug", 1)   # the flow pyramid stays readable; the same kernels run
    eng.set_option("conv3x3_pxn", pxn)
    if onepass_mask is not None:
        eng.set_option("onepass_mask", onepass_mask)
    return eng


def _forms(eng):
    return {r["name"]: r["form"] for r in eng.op_table() if r["category"] == 0}


def _flows(eng, h, w):
    return np.stack([eng.debug_read(f"flow_{d}/0").reshape(-1, 2) for d in ("fwd", "bwd")])


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,align", SIZES)
def test_cout32_pixels_on_n_agrees_and_runs(synthetic_weights, oracles, h, w, align):
    x0, x1 = synthetic.frame_pair(h, w, seed=37, n_waves=8)
    aux = {}
    ref = oracles[align].interpolate(x0, x1, DT, aux)
    ref_flow = np.stack([t[0].permute(1, 2, 0).contiguous().numpy().reshape(-1, 2)
                         for t in (aux["forward_flow_pyramid"][0], aux["backward_flow_pyramid"][0])])
    on, off = _engine(synthetic_weights, align, 2), _engine(synthetic_weights, align, 0)
    try:
        got, base = on(x0, x1, DT), off(x0, x1, DT)
        f_on, f_off = _forms(on), _forms(off)
        for name in LAYERS:
            assert f_on[name] == "3x3_pxn", f_on
            assert f_off[name] == "3x3", f_off
        assert "3x3_pxn" not in f_off.values(), f_off
        fl_on, fl_off = _flows(on, h, w), _flows(off, h, w)
        assert fl_on.shape == ref_flow.shape
        err = np.abs(got.astype(np.float64) - ref).max()
        err_off = np.abs(base.astype(np.float64) - ref).max()
        diff = np.abs(got - base).max()
        ferr = np.abs(fl_on.astype(np.float64) - ref_flow).max()
        ferr_off = np.abs(fl_off.astype(np.float64) - ref_flow).max()
        fdiff = np.abs(fl_on - fl_off).max()
        scale = max(1.0, float(np.abs(ref_flow).max()))
        print(f"{h}x{w}: frame err {err:.3e} (16x8 {err_off:.3e}) diff {diff:.3e}; "
              f"flow err {ferr:.3e} (16x8 {ferr_off:.3e}) diff {fdiff:.3e} scale {scale:.2f}")
        assert err < PLAN, err
        assert diff < 2.5e-4, diff
        # the folded sums reorder the single-pass products: the flow moves no further from the oracle than the 16x8
        # form's own distance allows
        assert ferr < 2.0 * ferr_off + 1e-4 * scale, (ferr, ferr_off)
        assert fdiff < 1e-3 * scale, fdiff
    finally:
        on.close()
        off.close()


@pytest.mark.gpu
def test_cout32_three_pass_keeps_the_16x8_form(synthetic_weights):
    """Every conv three-pass: the Cout = 32 layers stay on the 16x8 form even under option 2."""
    x0, x1 = synthetic.frame_pair(256, 320, seed=5, n_waves=4)
    eng = _engine(synthetic_weights, 64, 2, onepass_mask=0)
    try:
        eng(x0, x1, DT)
        forms = _forms(eng)
        for name in LAYERS:
            assert forms[name] == "3x3", forms
        assert forms["fe_conv1@L0"] == "3x3_pxn", forms   # the Cout = 64 layers still move
    finally:
        eng.close()


@pytest.mark.gpu
def test_cout32_default_rule_moves_the_full_size_layers(synthetic_weights):
    """Option 1 (default) moves the folded layers where 32x8 tiles give two waves: 256x320 has 640 tiles per layer."""
    x0, x1 = synthetic.frame_pair(256, 320, seed=6, n_waves=4)
    from frame_interpolation_b200.interpolator import Interpolator
    eng = Interpolator(synthetic_weights[0], align=64)
    try:
        assert eng.get_option("conv3x3_pxn") == 1
        eng(x0, x1, DT)
        forms = _forms(eng)
        for name in LAYERS:
            assert forms[name] == "3x3_pxn", forms
    finally:
        eng.close()
