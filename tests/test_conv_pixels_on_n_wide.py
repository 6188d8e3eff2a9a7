"""Pixels on the wgmma N dimension for the wide layers (option conv3x3_pxn): the single-pass Cout = 128 / 256 / 512
persistent 3x3 layers computed as D^T = W_tap x A^T on 32x8 tiles, each 128-cout N tile as two M = 64 weight halves, must
meet the same bars as the 16x8 form they replace, and must actually run.  Three-pass wide layers keep the 16x8 form.

The feature sub-trees carry every width: fe_conv2 / fe_conv3 have Cout = 128, fe_conv4 / fe_conv5 256 and fe_conv6 /
fe_conv7 512, and fe_conv3 and fe_conv5 store the fused 2x2 pool as well.  Option value 2 moves every eligible layer,
so the coarse levels of these sizes, whose heights are not multiples of 32, exercise the bottom-edge clipping of the
split stores and of the pool, and their few tiles the narrower N tiles (BN = 64) of the small levels."""
import numpy as np
import pytest

from frame_interpolation_b200 import synthetic

pytestmark = pytest.mark.gpu

PLAN = 4e-4         # default precision plan, against the oracle (as test_conv_pixels_on_n.py)
TIGHT = 1e-4        # every conv three-pass (onepass_mask = 0)
DT = np.full((1,), 0.5, np.float32)
COUT = {"fe_conv2": 128, "fe_conv3": 128, "fe_conv4": 256, "fe_conv5": 256, "fe_conv6": 512, "fe_conv7": 512}
POOLED = ("fe_conv3", "fe_conv5")


@pytest.fixture(scope="module")
def oracle(synthetic_weights):
    import os

    import torch
    from oracle.film_oracle import OracleInterpolator
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    return OracleInterpolator(synthetic_weights[1], align=64)


def _forms(eng):
    return {r["name"]: r["form"] for r in eng.op_table() if r["category"] == 0}


def _moved(forms, layer):
    return [n for n, f in forms.items() if n.split("@")[0] == layer and f == "3x3_pxn"]


@pytest.mark.parametrize("h,w", [(256, 320), (100, 150), (192, 320)])
def test_wide_pixels_on_n_agrees_and_runs(synthetic_weights, oracle, h, w):
    from frame_interpolation_b200.interpolator import Interpolator
    x0, x1 = synthetic.frame_pair(h, w, seed=31, n_waves=8)
    ref = oracle(x0, x1, DT)
    on = Interpolator(synthetic_weights[0], align=64)
    off = Interpolator(synthetic_weights[0], align=64)
    on.set_option("conv3x3_pxn", 2)
    off.set_option("conv3x3_pxn", 0)
    try:
        for mask in (None, 0):   # default precision plan, then every conv three-pass
            if mask is not None:
                for e in (on, off):
                    e.set_option("onepass_mask", mask)
            got, base = on(x0, x1, DT), off(x0, x1, DT)
            f_on, f_off = _forms(on), _forms(off)
            if mask is None:   # the default plan runs fe_conv2..7 of the level-0 sub-tree single-pass
                for cout in (128, 256, 512):
                    assert any(_moved(f_on, n) for n, c in COUT.items() if c == cout), (cout, f_on)
                assert any(_moved(f_on, n) for n in POOLED), f_on
            else:              # every conv three-pass: only the Cout = 64 layers move
                assert not any(_moved(f_on, n) for n in COUT), f_on
                assert f_on["fe_conv1@L0"] == "3x3_pxn", f_on
            assert "3x3_pxn" not in f_off.values(), f_off
            # the RGB-head epilogue keeps the 16x8 form, and nothing moves to another form than pixels on N
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


def test_wide_pixels_on_n_keeps_the_side_source_layers(synthetic_weights):
    """fusion_conv1 above level 0 reads the 10-of-64-channel side source, whose k-steps the kernel skips: even under
    option 2 it keeps the 16x8 form, where its weights stay one block per tap."""
    from frame_interpolation_b200.interpolator import Interpolator
    x0, x1 = synthetic.frame_pair(192, 320, seed=5, n_waves=4)
    eng = Interpolator(synthetic_weights[0], align=64)
    try:
        eng.set_option("conv3x3_pxn", 2)
        eng(x0, x1, DT)
        forms = _forms(eng)
        for lv in (1, 2, 3):
            assert forms[f"fusion_conv1@L{lv}"] == "3x3", forms
    finally:
        eng.close()
