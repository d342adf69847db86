#!/usr/bin/env python
"""Golden vectors for the bundle-entropy training gradient, produced by EXECUTING THE REFERENCE'S OWN code.

Executed reference code (paths relative to a locuslab/icnn checkout), unmodified, cut out with ``ast``:
  lib/bundle_entropy.py             solveBatch (imported unchanged) -> yN, G, h, lam, ys
  multi-label-cls/icnn_ebundle.py   crossEntrGrad (:390-417) and Model.train_step_fd (:296-314)
  completion/icnn_ebundle.py        mseGrad (:493-522) and Model.train_step_fd (:315-335)
  multi-label-cls/icnn_ebundle.py   Model.__init__ (:120-171) and Model.f (:316-388) on oracle/tf_shim.py: building
                                    it evaluates F_ (:148) and gv_ = opt.compute_gradients(F_, theta_) (:154)
The solve's fg is oracle/picnn_np.py in float64 (the reference's f is a TensorFlow graph).  The feed rows are
rounded to float32, as the reference's placeholders hold them (:128-131).  The Model is built once per sample on
that sample's rows, so every gradient is stored per sample ([B, ...]): every array of the small net, the arrays of
at most 4096 entries at C3.  Weights and x are regenerated from seeds by ``case_inputs`` (shared with the tests).

TEST INFRASTRUCTURE ONLY; needs a checkout of the reference at $ICNN_REFERENCE_DIR.
Usage:  python -m oracle.gen_golden_bundle_grad   -> tests/golden/training/bundle_grad.npz
"""
import types

import numpy as np

from icnn_b200 import workloads  # (pure-numpy input generator)
from oracle import picnn_np, refcode, regen
from oracle.tf_shim import Shim, variables_from_params

# a subdirectory: tests/test_oracle_golden.py runs every tests/golden/*.npz as a solveBatch case
GOLDEN = "training/bundle_grad.npz"

# tag -> (B, nIter, layerSizes passed to Model; the Model appends nLabels)
CASES = {"small": (12, 8, [14, 11]), "c3": (6, 10, [600])}
LOSSES = ("xent", "mse")
BN_EPS = 1e-5


def case_inputs(tag):
    """-> (p, x [B, m], y0 [B, n], trueY [B, n], nIter, layerSizes), seeded."""
    B, nIter, sizes = CASES[tag]
    rs = np.random.RandomState(4242 + len(tag))
    if tag == "small":     # three hidden layers, last hidden width = n, non-zero biases everywhere
        p = workloads.synth_params(33, 12, 9, [14, 11, 9])
        f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)  # noqa: E731
        for i in range(len(p.Wy)):
            p.Wy[i] = f32(3.0 * p.Wy[i])
        for i in range(p.L):
            p.bu[i] = f32(0.3 * rs.randn(p.hidden[i]))
        for i in range(p.L + 1):
            if i > 0:
                p.bzu[i] = f32(0.3 * rs.randn(p.sizes[i - 1]))
            p.byu[i] = f32(0.5 + 0.3 * rs.randn(p.n))
            p.bzx[i] = f32(0.3 * rs.randn(p.sizes[i]))
        x = f32(rs.randn(B, p.m))
        y0 = np.full((B, p.n), 0.5)
    else:
        p, x, y0 = workloads.make_inputs("C3", B=B)
    trueY = (rs.uniform(size=y0.shape) < 0.3).astype(np.float64)
    return p, x, y0, trueY, nIter, list(sizes)


def tf_name_to_param(name):
    """'z1_yu/W' -> ('Wy', 1) etc. (oracle/tf_shim.variables_from_params naming); None for batch-norm."""
    scope, var = name.rsplit("/", 1)
    if "/bn" in name:
        return None
    if scope.startswith("u"):
        return ("Wu" if var == "W" else "bu"), int(scope[1:])
    i = int(scope[1:].split("_")[0])
    kind = scope.split("_", 1)[1]
    table = {"zu_u": ("Wzu", "bzu"), "zu_proj": ("Wz", None), "yu_u": ("Wyu", "byu"), "yu": ("Wy", None),
             "u": ("Wzx", "bzx")}
    return table[kind][0 if var == "W" else 1], i


def model_grads(p, sizes, xr, Y, V, c):
    """gv_ of the reference's Model built on the shim with feeds (x, y, v, c) = the given rows: {tf name: grad}."""
    n = p.n
    bnvars = [(np.ones(s), np.zeros(s), np.zeros(s), np.full(s, 1.0 - BN_EPS)) for s in p.hidden[:-1]]
    sh = Shim(variables_from_params(p, bnvars))
    for k, a, rg in (("x", xr, False), ("y", Y, True), ("trueY", np.zeros((len(Y), n)), False), ("v", V, False),
                     ("c", c, False)):
        sh.feed(k, a, requires_grad=rg)
    ns = refcode.extract("multi-label-cls/icnn_ebundle.py", ["Model"],
                         {"tf": sh.tf, "tflearn": sh.tflearn, "np": np, "variable_summaries": lambda *a, **k: None})
    with refcode.quiet():
        model = ns["Model"](p.m, n, list(sizes), None)
    assert not sh.unused_variables(), sh.unused_variables()
    assert model.szs == p.hidden
    return {v.name[:-2]: g.detach().numpy().copy() for g, v in model.gv_}


def generate():
    ref_pc = refcode.load("ref_pc", "lib/bundle_entropy.py")
    grad_fns = {"xent": ("multi-label-cls/icnn_ebundle.py", "crossEntrGrad", None),
                "mse": ("completion/icnn_ebundle.py", "mseGrad", "n")}
    out = {}
    for tag in CASES:
        p, x, y0, trueY, nIter, sizes = case_inputs(tag)
        B = len(x)
        with refcode.quiet():
            yN, G, h, lam, ys, nIters = ref_pc.solveBatch(picnn_np.make_fg(p, x), y0.copy(), nIter=nIter)
        counts = np.array([len(g) for g in G])
        for loss in LOSSES:
            rel, fname, oshape = grad_fns[loss]
            train_step_fd = refcode.extract(rel, [fname, "Model.train_step_fd"], {"np": np})["train_step_fd"]
            stub = types.SimpleNamespace(x_="x", y_="y", v_="v", c_="c", outputSz=(p.n,) if oshape else None)
            with np.errstate(all="ignore"):
                fd = train_step_fd(stub, B, x, trueY, G, yN, ys, lam)
            assert np.array_equal(fd["x"], np.repeat(x, counts, axis=0))
            f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)  # noqa: E731
            Y, V, c = f32(fd["y"]), f32(fd["v"]), f32(fd["c"])
            key = "%s_%s_" % (tag, loss)
            out[key + "Y"], out[key + "V"], out[key + "c"] = Y, V, c
            off = np.concatenate([[0], np.cumsum(counts)])
            per = {}
            for u in range(B):
                s = slice(off[u], off[u + 1])
                gv = model_grads(p, sizes, np.repeat(x[u:u + 1], counts[u], axis=0), Y[s], V[s], c[s]) \
                    if counts[u] else {}
                for name, ga in gv.items():
                    per.setdefault(name, np.zeros((B,) + ga.shape))[u] = ga
            for name, arr in per.items():
                pn = tf_name_to_param(name)
                if pn is None or (tag == "c3" and arr[0].size > 4096):
                    continue
                out[key + "grad_%s%d" % pn] = arr
            print(tag, loss, "rows", len(Y), "stored", sum(k.startswith(key + "grad_") for k in out))
        out[tag + "_counts"] = counts
        out[tag + "_trueY"] = trueY
    return out


if __name__ == "__main__":
    regen.main(("gen_golden_bundle_grad",))
