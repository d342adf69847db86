#!/usr/bin/env python
"""Golden vectors for the convolutional PICNN of the image-completion experiment (E_ and dE_dy_), produced by
EXECUTING THE REFERENCE'S OWN completion ``Model`` (completion/icnn_ebundle.py:105-161,337-452, cut out with ``ast``,
unmodified) on oracle/tf_shim.py, like ``run_completion_model`` of oracle/gen_golden_tfshim.py.

Unlike the ``conv_small`` / ``conv_olivetti`` goldens of picnn_tfshim.npz (zero u biases, identity batch-norm), these
cases have non-zero biases in every layer that has one and non-identity batch-norm statistics, so that the literal
(unfolded) batch-norm, the bias placement and TensorFlow's 'SAME' padding at an odd image size are pinned too.
Weights and inputs are regenerated from seeds by ``case`` (shared with the tests); only outputs are stored.

TEST INFRASTRUCTURE ONLY; needs a checkout of the reference at $ICNN_REFERENCE_DIR.
Usage:  python oracle/gen_golden_conv.py   -> tests/golden/conv/conv_picnn.npz
"""
import contextlib
import io
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = {"conv_bn_olivetti": (3, 64, 32, 11), "conv_bn_odd": (4, 17, 9, 12)}     # tag -> (B, H, W, seed)


def _f32(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def case(tag):
    """-> (variables {name: float64 array, float32-representable}, x [B, H*W], y [B, H*W], H, W)."""
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from conv_picnn import ConvPICNN
    from oracle.gen_golden_tfshim import conv_variables
    B, H, W, seed = CASES[tag]
    v = conv_variables(ConvPICNN(H, W, seed=seed, dtype=torch.float64))
    rs = np.random.RandomState(1000 + seed)
    for name in sorted(v):
        a = v[name]
        if name.endswith("/moving_mean"):
            a = 0.3 * rs.randn(*a.shape)
        elif name.endswith("/moving_variance"):
            a = rs.uniform(0.5, 2.0, size=a.shape)
        elif name.endswith("/gamma"):
            a = rs.uniform(0.5, 1.5, size=a.shape)
        elif name.endswith("/beta"):
            a = 0.2 * rs.randn(*a.shape)
        elif name.endswith("_yu_u/b"):
            a = 0.5 + 0.3 * rs.randn(*a.shape)
        elif name.endswith("/b"):
            a = a + 0.1 * rs.randn(*a.shape)
        v[name] = _f32(a)
    x = _f32(rs.uniform(size=(B, H * W)))
    y = _f32(rs.uniform(0.05, 0.95, size=(B, H * W)))
    return v, x, y, H, W


def run(tag, ref):
    from oracle.gen_golden_tfshim import extract
    from oracle.tf_shim import Shim, tensor_get_shape
    v, x, y, H, W = case(tag)
    B = x.shape[0]
    sh = Shim(v)
    rs = np.random.RandomState(5)
    for k, a, rg in (("x", x.reshape(B, H, W, 1), False), ("y", y.reshape(B, H, W, 1), True),
                     ("trueY", np.zeros((B, H, W, 1)), False), ("v", rs.randn(B, H * W), False), ("c", rs.randn(B), False),
                     ("l_yN", np.zeros(()), False), ("nBundleIter", np.zeros(B), False), ("nActive", np.zeros(B), False)):
        sh.feed(k, a, requires_grad=rg)
    ns = extract(os.path.join(ref, "completion/icnn_ebundle.py"), ["Model"],
                 {"tf": sh.tf, "tflearn": sh.tflearn, "np": np, "variable_summaries": lambda *a, **k: None})
    with contextlib.redirect_stdout(io.StringIO()), tensor_get_shape():
        model = ns["Model"]([H, W, 1], [H, W, 1], None)
    assert not sh.unused_variables(), sh.unused_variables()
    return model.E_.detach().numpy(), model.dE_dyFlat_.detach().numpy()


def main():
    ref = os.environ.get("ICNN_REFERENCE_DIR", "")
    out = {}
    for tag in CASES:
        out[tag + "_f"], out[tag + "_g"] = run(tag, ref)
        print(tag, "f", out[tag + "_f"], "max|g|", np.abs(out[tag + "_g"]).max())
    path = os.path.join(ROOT, "tests", "golden", "conv", "conv_picnn.npz")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path) // 1024, "KB")


if __name__ == "__main__":
    main()
