"""Generates tests/golden/*.npz from the CPU oracle (the reference itself cannot run here:
no TensorFlow, no SavedModel -- so these vectors pin the ORACLE, i.e.
they guard the restatement against accidental change and give the GPU tests fixed targets).

    python tests/golden/make_golden.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from frame_interpolation_b200 import synthetic, weights  # noqa: E402
from oracle.film_oracle import OracleInterpolator  # noqa: E402

CASES = {
    "g64": dict(h=64, w=64, seed=5, align=64, block=None),
    "g100x60_align": dict(h=100, w=60, seed=6, align=64, block=None),
    "g128_tiled2x2": dict(h=128, w=128, seed=7, align=64, block=[2, 2]),
}


def main():
    torch.set_num_threads(4)
    w = weights.synthetic_weights(1234)
    here = os.path.dirname(os.path.abspath(__file__))
    for name, c in CASES.items():
        x0, x1 = synthetic.frame_pair(c["h"], c["w"], seed=c["seed"], n_waves=6)
        dt = np.full((1,), 0.5, np.float32)
        orc = OracleInterpolator(w, align=c["align"], block_shape=c["block"])
        out32 = orc(x0, x1, dt)
        out64 = OracleInterpolator(w, align=c["align"], block_shape=c["block"], dtype=torch.float64)(x0, x1, dt)
        aux = {}
        if c["block"] is None:
            orc.interpolate(x0, x1, dt, aux)
            fwd = aux["forward_flow_pyramid"][0][0].permute(1, 2, 0).numpy()
            bwd = aux["backward_flow_pyramid"][0][0].permute(1, 2, 0).numpy()
        else:
            fwd = bwd = np.zeros((0,), np.float32)
        # image = fp64-oracle result rounded to fp32 (the "truth"); the fp32 oracle is within ~1e-6 of it
        np.savez_compressed(os.path.join(here, name + ".npz"), image=out64.astype(np.float32),
                            flow_fwd_l0=fwd.astype(np.float32),
                            weights_sha256=np.array(weights.digest(w)), x0_sum=np.float64(x0.sum()),
                            x1_sum=np.float64(x1.sum()), **{k: np.array(str(v)) for k, v in c.items()})
        print(name, out32.shape, float(np.abs(out32 - out64).max()))


if __name__ == "__main__":
    main()
