#!/usr/bin/env python
"""Golden vectors for d mse / d theta through the unrolled momentum-GD loop, from torch float64
autograd on the restated training graph (oracle/gd_grad_torch.py; the reference's TF graph,
multi-label-cls/icnn-back.py:116-139, cannot run here).  TEST INFRASTRUCTURE ONLY.
Usage:  python -m oracle.gen_golden_gd_grad   -> tests/golden/gd_grad.npz"""
import numpy as np

from oracle import regen, synth
from oracle.gd_grad_torch import torch_unrolled_grads

GOLDEN = "gd_grad.npz"

CASES = {
    # tag: (config, B, nIter, lr, momentum)   -- icnn-back.py defaults are lr .01, momentum .3, 30 its
    "c1": ("C1", 32, 8, 0.05, 0.3),
    "c1_m9": ("C1", 16, 30, 0.01, 0.9),
}


def true_labels(B, n, seed=11):
    return (np.random.RandomState(seed).uniform(size=(B, n)) < 0.3).astype(np.float64)


def generate():
    out = {}
    for tag, (name, B, nIter, lr, mom) in CASES.items():
        p, x, y0 = synth.make_inputs(name, B=B)
        tY = true_labels(B, p.n)
        yN, loss, G = torch_unrolled_grads(p, x, y0, tY, nIter, lr, mom)
        out[tag + "_meta"] = np.array([B, nIter, lr, mom])
        out[tag + "_yN"] = yN
        out[tag + "_loss"] = np.array(loss)
        for k in ("Wy", "Wz", "Wu", "bu", "Wzu", "bzu", "Wyu", "byu"):
            for i, g in enumerate(G[k]):
                if g is not None:
                    out["%s_%s%d" % (tag, k, i)] = g
    return out


if __name__ == "__main__":
    regen.main(("gen_golden_gd_grad",))
