"""Pixels on the wgmma N dimension (option conv3x3_pxn): the Cout = 64 persistent 3x3 layers computed as
D^T = W_tap x A^T on 32x8 tiles must meet the same bars as every other kernel variant, and must actually run.

Option value 2 puts every eligible layer on the new form, so the small pyramid levels of these sizes, whose heights are
not multiples of 32, exercise the bottom-edge clipping of the split stores and of the fused 2x2 pool; 100x150 pads to
128x192 and also leaves partial tiles in x on its coarse levels."""
import numpy as np
import pytest

from frame_interpolation_b200 import synthetic

pytestmark = pytest.mark.gpu

PLAN = 4e-4         # default precision plan, against the oracle (as test_kernel_variants_agree)
TIGHT = 1e-4        # every conv three-pass (onepass_mask = 0)
DT = np.full((1,), 0.5, np.float32)


@pytest.fixture(scope="module")
def oracle(synthetic_weights):
    import os

    import torch
    from oracle.film_oracle import OracleInterpolator
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    return OracleInterpolator(synthetic_weights[1], align=64)


def _forms(eng):
    return {r["name"]: r["form"] for r in eng.op_table() if r["category"] == 0}


@pytest.mark.parametrize("h,w", [(256, 320), (100, 150), (192, 320)])
def test_pixels_on_n_agrees_and_runs(synthetic_weights, oracle, h, w):
    from frame_interpolation_b200.interpolator import Interpolator
    x0, x1 = synthetic.frame_pair(h, w, seed=29, n_waves=8)
    ref = oracle(x0, x1, DT)
    on = Interpolator(synthetic_weights[0], align=64)
    off = Interpolator(synthetic_weights[0], align=64)
    on.set_option("conv3x3_pxn", 2)
    off.set_option("conv3x3_pxn", 0)
    assert on.get_option("conv3x3_pxn") == 2
    try:
        for mask in (None, 0):   # default precision plan, then every conv three-pass
            if mask is not None:
                for e in (on, off):
                    e.set_option("onepass_mask", mask)
            got, base = on(x0, x1, DT), off(x0, x1, DT)
            f_on, f_off = _forms(on), _forms(off)
            # the new form ran on the 64 -> 64 layers with a plain store (fusion_conv1) and with the fused pool (fe_conv1)
            assert f_on["fusion_conv1@L0"] == "3x3_pxn" and f_on["fe_conv1@L0"] == "3x3_pxn", f_on
            assert "3x3_pxn" not in f_off.values(), f_off
            # ... and nowhere else: Cout != 64 layers and the RGB-head epilogue keep the persistent kernel
            assert f_on["fusion_conv2+rgb@L0"] == "3x3"
            assert all(f == "3x3_pxn" or f_off[n] == f for n, f in f_on.items())
            err = np.abs(got.astype(np.float64) - ref).max()
            diff = np.abs(got - base).max()
            if mask is None:
                assert err < PLAN, err
                assert diff < 2.5e-4, diff
            else:
                assert err < TIGHT, err
                assert diff < 5e-5, diff
    finally:
        on.close()
        off.close()


def test_pixels_on_n_default_rule(synthetic_weights):
    """The default (1) moves a layer only where 32x8 tiles still give two waves over the SMs and no source skips
    k-steps: at 256x320 the level-0 feature convs (2 x 8 x 40 tiles for the image pair) move, the 128x160 level-1
    feature convs do not, and neither does fusion_conv1@L0 (its 10-of-64-channel side source)."""
    from frame_interpolation_b200.interpolator import Interpolator
    x0, x1 = synthetic.frame_pair(256, 320, seed=3, n_waves=4)
    eng = Interpolator(synthetic_weights[0], align=64)
    try:
        assert eng.get_option("conv3x3_pxn") == 1
        eng(x0, x1, DT)
        forms = _forms(eng)
        assert forms["fe_conv1@L0"] == "3x3_pxn" and forms["fe_conv1@L1"] == "3x3", forms
        assert forms["fusion_conv1@L0"] == "3x3", forms
    finally:
        eng.close()
