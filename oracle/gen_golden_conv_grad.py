#!/usr/bin/env python
"""Golden vectors for the conv-PICNN training gradient, produced by EXECUTING THE REFERENCE'S OWN code.

Executed reference code (paths relative to a locuslab/icnn checkout), unmodified, cut out with ``ast``:
  lib/bundle_entropy.py         solveBatch (imported unchanged) -> yN, G, h, lam, ys
  completion/icnn_ebundle.py    mseGrad (:493-522) and Model.train_step_fd (:315-335) -> the feed rows (y, v, c)
  completion/icnn_ebundle.py    Model.__init__ (:105-161) and Model.f (:337-452) on oracle/tf_shim.py: building it
                                evaluates F_ (:129-130) and gv_ = compute_gradients(F_, theta_) (:138-139)
The solve's fg is oracle/conv_energy.fg in float64 (pinned to the reference's own E_ / dE_dy_ by
tests/golden/conv/conv_picnn.npz); the nets and x are those of oracle/gen_golden_conv.py (non-zero biases,
non-identity batch-norm).  The feed rows are rounded to float32, as the reference's placeholders hold them.  The
Model is built once per sample on that sample's rows, so every gradient is stored per sample ([B, ...]).  The
reference's Model has one architecture (three conv layers of 32 / 64 / 64 channels, a 512-wide dense layer), so its
dense weights alone are ~1M entries per sample: arrays of at most 4096 entries are stored whole, every larger one as
its projections on four fixed random vectors (``probe``, [B, 4]), which pins each of its entries.  '<tag>_gv_names'
lists every variable gv_ holds.

TEST INFRASTRUCTURE ONLY; needs a checkout of the reference at $ICNN_REFERENCE_DIR.
Usage:  python -m oracle.gen_golden_conv_grad   -> tests/golden/conv/conv_train_grad.npz
"""
import types

import numpy as np

from oracle import conv_energy, refcode, regen
from oracle.conv_picnn import CONVS, FCS
from oracle.tf_shim import Shim, tensor_get_shape

GOLDEN = "conv/conv_train_grad.npz"
CASES = {"conv_bn_odd": 10, "conv_bn_olivetti": 8}     # tag of oracle/gen_golden_conv.py -> solver iterations
MAX_WHOLE = 4096


def probe(a):
    """a [..., N] (flattened per sample) -> [..., 4]: projections on four fixed standard-normal vectors."""
    a = np.asarray(a, dtype=np.float64)
    N = a.shape[-1]
    return a @ np.random.RandomState(N % 100003).randn(N, 4)


def case_rows_inputs(tag):
    """-> (variables, x [B, H*W], y0 [B, H*W], trueY [B, H*W], H, W, nIter), seeded."""
    from oracle.gen_golden_conv import case
    v, x, _y, H, W = case(tag)
    rs = np.random.RandomState(77 + len(tag))
    B = x.shape[0]
    y0 = np.tile(rs.uniform(0.2, 0.8, size=(1, H * W)), (B, 1))
    trueY = rs.uniform(size=(B, H * W))
    return v, x, y0, trueY, H, W, CASES[tag]


def model_grads(v, H, W, xr, Y, V, c):
    """gv_ of the reference's completion Model built on the shim with feeds (x, y, v, c) = the given rows."""
    R = len(Y)
    sh = Shim(v)
    for k, a, rg in (("x", xr.reshape(R, H, W, 1), False), ("y", Y.reshape(R, H, W, 1), True),
                     ("trueY", np.zeros((R, H, W, 1)), False), ("v", V, False), ("c", c, False),
                     ("l_yN", np.zeros(()), False), ("nBundleIter", np.zeros(R), False), ("nActive", np.zeros(R), False)):
        sh.feed(k, a, requires_grad=rg)
    ns = refcode.extract("completion/icnn_ebundle.py", ["Model"],
                         {"tf": sh.tf, "tflearn": sh.tflearn, "np": np, "variable_summaries": lambda *a, **k: None})
    with refcode.quiet(), tensor_get_shape():
        model = ns["Model"]([H, W, 1], [H, W, 1], None)
    assert not sh.unused_variables(), sh.unused_variables()
    return {var.name[:-2]: g.detach().numpy().copy() for g, var in model.gv_}


def generate():
    import torch
    threads = torch.get_num_threads()
    torch.set_num_threads(1)          # the float64 fg bit for bit on every regeneration
    ref_pc = refcode.load("ref_pc", "lib/bundle_entropy.py")
    train_step_fd = refcode.extract("completion/icnn_ebundle.py", ["mseGrad", "Model.train_step_fd"],
                                    {"np": np})["train_step_fd"]
    f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)  # noqa: E731
    out = {}
    for tag in CASES:
        v, x, y0, trueY, H, W, nIter = case_rows_inputs(tag)
        # what conv_energy reads, as icnn_b200.conv_picnn.parse_variables would return it for these variables
        spec = types.SimpleNamespace(H=H, W=W, convs=list(CONVS), fcs=list(FCS),
                                     vars={k: np.ascontiguousarray(a, dtype=np.float32) for k, a in v.items()})
        B = len(x)
        fg = lambda y: conv_energy.fg(spec, x, y)          # noqa: E731
        with refcode.quiet():
            yN, G, h, lam, ys, nIters = ref_pc.solveBatch(fg, y0.copy(), nIter=nIter)
        counts = np.array([len(g) for g in G])
        stub = types.SimpleNamespace(x_="x", y_="y", v_="v", c_="c", outputSz=(H * W,))
        with np.errstate(all="ignore"):
            fd = train_step_fd(stub, B, x, trueY, G, yN, ys, lam)
        assert np.array_equal(fd["x"], np.repeat(x, counts, axis=0))
        Y, V, c = f32(fd["y"]), f32(fd["v"]), f32(fd["c"])
        off = np.concatenate([[0], np.cumsum(counts)])
        per, names = {}, None
        for u in range(B):
            if not counts[u]:
                continue
            s = slice(off[u], off[u + 1])
            gv = model_grads(v, H, W, np.repeat(x[u:u + 1], counts[u], axis=0), Y[s], V[s], c[s])
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
        out[tag + "_Y"], out[tag + "_V"], out[tag + "_c"] = (a.astype(np.float32) for a in (Y, V, c))   # exact
        out[tag + "_counts"] = counts
        print(tag, "rows", len(Y), "gv_", len(names), "whole", sum(k.startswith(tag + "_grad_") for k in out))
    torch.set_num_threads(threads)    # the generators run after this one compute as they do alone
    return out


if __name__ == "__main__":
    regen.main(("gen_golden_conv_grad",))
