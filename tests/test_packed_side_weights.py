"""Packed side-source weights of fusion_conv1 (csrc/film_pack.h).

The side tensor holds 10 real channels in a 64-channel chunk, so the persistent 3x3 kernel issues k-step 0 alone of
each of its nine taps.  On the pixels-on-N form its weights are packed one K block per dx column (the three dy taps'
16-channel slices at K offsets 0 / 16 / 32); the 16x8 form and the generic kernel keep one block per tap.  The CPU
test checks the packing itself; the GPU tests run fusion_conv1 on both forms (pixels on N always with three dx boxes,
16x8 tiles with dx boxes and with the wide halo box) against the oracle and against the generic kernel."""
import os
import subprocess

import numpy as np
import pytest

from frame_interpolation_b200 import build, synthetic

PLAN = 4e-4         # default precision plan, against the oracle (as test_kernel_variants_agree)
TIGHT = 1e-4        # every conv three-pass (onepass_mask = 0)
DT = np.full((1,), 0.5, np.float32)

_HARNESS = r"""
#include <cstdio>
#include "film_pack.h"
int main() {
  const int cout = 3, chunk = 64;
  const std::vector<int> src_chunks = {1, 2, 1}, packed = {0, 1, 0};
  const int ktot = 4 * 9 * chunk;
  std::vector<uint16_t> w((size_t)cout * ktot);
  for (size_t i = 0; i < w.size(); ++i) w[i] = (uint16_t)(i % 65521 + 1);
  int ktot_out = 0;
  const std::vector<uint16_t> p = film::pack_dx_blocks(w, cout, ktot, chunk, src_chunks, packed, ktot_out);
  std::printf("%d\n", ktot_out);
  for (uint16_t v : p) std::printf("%u\n", (unsigned)v);
}
"""


def test_dx_block_packing_reproduces_the_per_tap_k_values(tmp_path):
    """Sources (1 chunk per tap, 2 chunks packed, 1 chunk per tap): the packed chunks keep k-step 0 of tap (dy, dx)
    at K offset 16 dy of block dx and zeros in the fourth k-step; the other sources are copied unchanged."""
    src = tmp_path / "pack.cpp"
    src.write_text(_HARNESS)
    exe = tmp_path / "pack"
    subprocess.run([build._nvcc(), "-std=c++17", "-I", build.CSRC, str(src), "-o", str(exe)], check=True,
                   capture_output=True)
    vals = np.array(subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split(), np.int64)
    cout, chunk, ktot = 3, 64, 4 * 9 * 64
    per_tap = (np.arange(cout * ktot) % 65521 + 1).reshape(cout, ktot // chunk, chunk)   # [n][(chunk, tap)][c]
    assert vals[0] == ktot - 2 * 6 * chunk
    got = vals[1:].reshape(cout, vals[0] // chunk, chunk)
    np.testing.assert_array_equal(got[:, :9], per_tap[:, :9])            # source 0: nine per-tap blocks
    np.testing.assert_array_equal(got[:, 15:], per_tap[:, 27:])          # source 2 after 2 x 3 packed blocks
    for ch in range(2):
        for dx in range(3):
            blk = got[:, 9 + 3 * ch + dx]
            for dy in range(3):
                np.testing.assert_array_equal(blk[:, 16 * dy:16 * dy + 16], per_tap[:, 9 + 9 * ch + 3 * dx + dy, :16])
            assert not blk[:, 48:].any()


@pytest.fixture(scope="module")
def oracle(synthetic_weights):
    import torch
    from oracle.film_oracle import OracleInterpolator
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    return OracleInterpolator(synthetic_weights[1], align=None)


def _engine(synthetic_weights, **opts):
    from frame_interpolation_b200.interpolator import Interpolator
    eng = Interpolator(synthetic_weights[0], align=None)
    eng.set_option("any_size", 1)
    for k, v in opts.items():
        eng.set_option(k, v)
    return eng


def _form(eng, name="fusion_conv1@L0"):
    return {r["name"]: r["form"] for r in eng.op_table() if r["category"] == 0}[name]


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(256, 320), (100, 150), (65, 129)])
@pytest.mark.parametrize("pxn", [0, 2])
@pytest.mark.parametrize("halo", [0, 3])
def test_packed_side_layers_match_the_oracle(synthetic_weights, oracle, h, w, pxn, halo):
    x0, x1 = synthetic.frame_pair(h, w, seed=37, n_waves=8)
    ref = oracle(x0, x1, DT)
    eng = _engine(synthetic_weights, conv3x3_pxn=pxn, conv3x3_halo=halo)
    try:
        for mask, tol in ((None, PLAN), (0, TIGHT)):
            if mask is not None:
                eng.set_option("onepass_mask", mask)
            got = eng(x0, x1, DT)
            assert _form(eng) == ("3x3_pxn" if pxn else "3x3")
            err = np.abs(got.astype(np.float64) - ref).max()
            assert err < tol, (mask, err)
    finally:
        eng.close()


@pytest.mark.gpu
def test_default_rule_moves_fusion_conv1_to_pixels_on_n_at_1080p(synthetic_weights):
    """At 1088x1920 the 32x8 tiles of fusion_conv1@L0 take half the waves of 16x8 tiles (62 against 124 on 132 SMs),
    so the default moves it; at 256x320 (3 against 5) test_pixels_on_n_default_rule keeps it on 16x8."""
    from frame_interpolation_b200.interpolator import Interpolator
    x0, x1 = synthetic.frame_pair(1080, 1920, seed=5, n_waves=4)
    eng = Interpolator(synthetic_weights[0], align=64)
    try:
        eng(x0, x1, DT)
        assert _form(eng) == "3x3_pxn"
        assert _form(eng, "fusion_conv1@L1") == "3x3"
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pxn", [0, 2])
@pytest.mark.parametrize("halo", [0, 3])
def test_packed_side_layers_match_the_per_tap_generic_kernel(synthetic_weights, pxn, halo):
    """Every conv three-pass: the persistent kernel with packed side weights against the generic kernel, which reads
    one weight block per tap and issues every k-step."""
    x0, x1 = synthetic.frame_pair(256, 320, seed=41, n_waves=8)
    eng = _engine(synthetic_weights, conv3x3_pxn=pxn, conv3x3_halo=halo, onepass_mask=0)
    gen = _engine(synthetic_weights, conv3x3_v2=0, onepass_mask=0)
    try:
        got, base = eng(x0, x1, DT), gen(x0, x1, DT)
        assert _form(gen) == "tc"
        diff = np.abs(got - base).max()
        assert diff < 2e-5, diff
    finally:
        eng.close()
        gen.close()
