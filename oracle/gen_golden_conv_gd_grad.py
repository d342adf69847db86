#!/usr/bin/env python
"""Golden vectors for the conv-PICNN GD training gradient, produced by EXECUTING THE REFERENCE'S OWN code.

Executed reference code (paths relative to a locuslab/icnn checkout), unmodified, cut out with ``ast``:
  completion/icnn.back.py    Model.__init__ (:121-156) and Model.f (:276-396) on oracle/tf_shim.py: building it unrolls
                             nGdIter momentum-GD steps (lr = 0.01, momentum = 0.9), evaluates yn_ and
                             mse_ = reduce_mean(square(255 (yn_ - trueY))) and gv_ = compute_gradients(mse_, theta_)
The nets and x are those of oracle/gen_golden_conv.py (non-zero biases, non-identity batch-norm); y0 is one fixed row
for every sample (as the script's meanY is) and trueY is seeded.  The Model is built once per sample, so mse_ is the
mean over that sample and every output is stored per sample ([B, ...]); the batch gradient of the mean over B samples
is the mean of the per-sample ones.  Arrays of at most 4096 entries per sample are stored whole, every larger one as
its projections on four fixed random vectors (gen_golden_conv_grad.probe, [B, 4]).  '<tag>_gv_names' lists every
variable gv_ holds.

TEST INFRASTRUCTURE ONLY; needs a checkout of the reference at $ICNN_REFERENCE_DIR.
Usage:  python oracle/gen_golden_conv_gd_grad.py   -> tests/golden/conv/conv_gd_grad.npz
"""
import contextlib
import io
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = ("conv_bn_odd", "conv_bn_olivetti")     # tags of oracle/gen_golden_conv.py
N_GD_ITER = 30                                  # completion/icnn.back.py --nGdIter default
MAX_WHOLE = 4096


def case_inputs(tag):
    """-> (variables, x [B, H*W], y0 [B, H*W], trueY [B, H*W], H, W), seeded."""
    from oracle.gen_golden_conv import case
    v, x, _y, H, W = case(tag)
    rs = np.random.RandomState(311 + len(tag))
    B = x.shape[0]
    y0 = np.tile(rs.uniform(0.2, 0.8, size=(1, H * W)), (B, 1))
    trueY = rs.uniform(size=(B, H * W))
    return v, x, y0, trueY, H, W


def model_outputs(v, path, H, W, x, y0, trueY, nGdIter):
    """(yn_, mse_, {name: gradient}) of the reference's back-optimisation Model built on the shim with these feeds."""
    from oracle.gen_golden_tfshim import extract
    from oracle.tf_shim import Shim, tensor_get_shape
    B = len(x)
    sh = Shim(v)
    for k, a, rg in (("x", x.reshape(B, H, W, 1), False), ("y", y0.reshape(B, H, W, 1), True),
                     ("trueY", trueY.reshape(B, H, W, 1), False)):
        sh.feed(k, a, requires_grad=rg)
    ns = extract(path, ["Model"], {"tf": sh.tf, "tflearn": sh.tflearn, "np": np,
                                   "variable_summaries": lambda *a, **k: None})
    with contextlib.redirect_stdout(io.StringIO()), tensor_get_shape():
        model = ns["Model"]([H, W, 1], [H, W, 1], None, nGdIter)
    assert not sh.unused_variables(), sh.unused_variables()
    grads = {var.name[:-2]: g.detach().numpy().copy() for g, var in model.gv_}
    return model.yn_.detach().numpy().reshape(B, -1), float(model.mse_.detach()), grads


def generate():
    import torch
    from oracle.gen_golden import REF
    from oracle.gen_golden_conv_grad import probe
    torch.set_num_threads(1)          # the same float64 sums on every regeneration
    path = os.path.join(REF, "completion/icnn.back.py")
    out = {}
    for tag in CASES:
        v, x, y0, trueY, H, W = case_inputs(tag)
        B = len(x)
        per, names, yn, mse = {}, None, np.zeros((B, H * W)), np.zeros(B)
        for u in range(B):
            s = slice(u, u + 1)
            yn[u], mse[u], gv = model_outputs(v, path, H, W, x[s], y0[s], trueY[s], N_GD_ITER)
            names = sorted(gv) if names is None else names
            assert sorted(gv) == names
            for name, ga in gv.items():
                per.setdefault(name, np.zeros((B,) + ga.shape))[u] = ga
        for name, arr in per.items():
            if arr[0].size <= MAX_WHOLE:
                out["%s_grad_%s" % (tag, name)] = arr
            else:
                out["%s_probe_%s" % (tag, name)] = probe(arr.reshape(B, -1))
        out[tag + "_gv_names"] = np.array(names)
        out[tag + "_yn"], out[tag + "_mse"] = yn, mse
        out[tag + "_nGdIter"] = np.array(N_GD_ITER)
        print(tag, "B", B, "gv_", len(names), "whole", sum(k.startswith(tag + "_grad_") for k in out), flush=True)
    return out


def main():
    out = generate()
    path = os.path.join(ROOT, "tests", "golden", "conv", "conv_gd_grad.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays,", os.path.getsize(path) // 1024, "KB")


if __name__ == "__main__":
    main()
