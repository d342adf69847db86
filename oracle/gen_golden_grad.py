#!/usr/bin/env python
"""Golden vectors for argmin differentiation from the UNMODIFIED reference function bodies.

multi-label-cls/icnn_ebundle.py and completion/icnn_ebundle.py import TensorFlow at module level,
so the modules cannot be imported; `crossEntrGrad` (:390-417) and `mseGrad` (:493-522) are pure
numpy, so their source is cut out with `ast` and exec'd as-is, and so is `Model.train_step_fd`
(:296-314 / :315-335), which assembles the training step's feed rows from them.  Inputs: bundle states
produced by the reference lib/bundle_entropy.solveBatch on seeded synthetic problems (C1 and C3 dims).
TEST INFRASTRUCTURE ONLY; needs a checkout of the reference at $ICNN_REFERENCE_DIR.
Usage:  python -m oracle.gen_golden_grad   -> tests/golden/argmin_grad.npz
"""
import types

import numpy as np

from oracle import picnn_np, refcode, regen, synth

GOLDEN = "argmin_grad.npz"


def generate():
    ns = {"xent": refcode.extract("multi-label-cls/icnn_ebundle.py", ["crossEntrGrad", "Model.train_step_fd"],
                                  {"np": np}),
          "mse": refcode.extract("completion/icnn_ebundle.py", ["mseGrad", "Model.train_step_fd"], {"np": np})}
    grad = {"xent": ns["xent"]["crossEntrGrad"], "mse": ns["mse"]["mseGrad"]}
    ref_pc = refcode.load("ref_pc", "lib/bundle_entropy.py")
    out = {}
    for tag, cfgname, B, nIter in [("c1", "C1", 32, 5), ("c3", "C3", 12, 10)]:
        p, x, y0 = synth.make_inputs(cfgname, B=B)
        fg = picnn_np.make_fg(p, x)
        with refcode.quiet():
            yN, G, h, lam, ys, nIters = ref_pc.solveBatch(fg, y0.copy(), nIter=nIter)
        rs = np.random.RandomState(17)
        trueY = (rs.uniform(size=yN.shape) < 0.3).astype(np.float64)
        kmax = max(len(g) for g in G)
        n = yN.shape[1]
        for name in ("xent", "mse"):
            cy = np.zeros((B, n)); clam = np.zeros((B, kmax)); ct = np.zeros(B)
            for j in range(B):
                with np.errstate(all="ignore"):
                    a, b_, c = grad[name](yN[j], trueY[j], np.array(G[j]))
                cy[j] = a; clam[j, :len(b_)] = b_; ct[j] = np.asarray(c).ravel()[0]
            out["%s_%s_cy" % (tag, name)] = cy
            out["%s_%s_clam" % (tag, name)] = clam
            out["%s_%s_ct" % (tag, name)] = ct
        # the (v, c) assembly of the training step, by the reference's own method on a stub ``self``
        # (placeholders = dictionary keys)
        for name, oshape in (("xent", None), ("mse", (yN.shape[1],))):
            stub = types.SimpleNamespace(x_="x", y_="y", v_="v", c_="c", outputSz=oshape)
            with np.errstate(all="ignore"):
                fd = ns[name]["train_step_fd"](stub, B, x, trueY, G, yN, ys, lam)
            assert np.array_equal(fd["x"], np.repeat(x, [len(g) for g in G], axis=0))
            out["%s_%s_fd_ys" % (tag, name)] = fd["y"]
            out["%s_%s_fd_vs" % (tag, name)] = fd["v"]
            out["%s_%s_fd_cs" % (tag, name)] = fd["c"]
        out[tag + "_trueY"] = trueY
        out[tag + "_yN"] = yN
        out[tag + "_counts"] = np.array([len(g) for g in G])
    return out


if __name__ == "__main__":
    regen.main(("gen_golden_grad",))
