#!/usr/bin/env python
"""Golden vectors for the PICNN energy f, df/dy, the unrolled momentum-GD loop and its training gradient,
produced by EXECUTING THE REFERENCE'S OWN graph code (cut out of its files with ``ast``, unmodified) on
oracle/tf_shim.py -- TensorFlow / tflearn are not installed, the shim restates only their primitives.

Executed reference code (paths relative to a locuslab/icnn checkout):
  multi-label-cls/icnn_ebundle.py  class Model: __init__ (:120-166) and f (:316-388)  -> E_, dE_dy_
  multi-label-cls/icnn-back.py     class Model: __init__ (:104-147) and f (:233-305)  -> yn_, energies_, mse_,
                                   opt.compute_gradients(mse_, theta_)
  RL/src/icnn.py                   class Agent: negQ (:325-404), bundle_entropy (:148-158); entropy (:455-458)
  RL/src/bundle_entropy.py         solveBatch (imported unchanged, called BY Agent.bundle_entropy)
  completion/icnn_ebundle.py       class Model: __init__ (:105-161) and f (:337-452): the CONVOLUTIONAL PICNN of the
                                   Olivetti experiment -> E_, dE_dy_; pins oracle/conv_picnn.py, the user-side ``fg`` the
                                   GPU callback-mode test drives K2 with

The goldens pin oracle/picnn_np.py (f, df/dy, gates incl. batch-norm, momentum GD, the RL affine wrapper) and
oracle/gd_grad_np.py (training gradient through the unrolled loop) -- tests/test_oracle_tfshim.py -- and are
compared with the device kernels in tests/test_gpu_picnn.py.  Weights and inputs are regenerated from seeds by
``case_inputs`` (shared with the tests); only outputs are stored.

TEST INFRASTRUCTURE ONLY; needs a checkout of the reference at $ICNN_REFERENCE_DIR.
Usage:  python -m oracle.gen_golden_tfshim   -> tests/golden/picnn_tfshim.npz
"""
import types

import numpy as np

from icnn_b200 import workloads  # (pure-numpy input generator)
from oracle import refcode, regen
from oracle.tf_shim import Shim, tensor_get_shape, variables_from_params

GOLDEN = "picnn_tfshim.npz"
BN_EPS = 1e-5


# --------------------------------------------------------------------------------------------------------
# seeded inputs (shared with the tests)
# --------------------------------------------------------------------------------------------------------

def _f32(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def _random_biases(p, rs):
    """Non-zero biases everywhere the reference has one, so that bias placement is pinned too."""
    for i in range(p.L):
        p.bu[i] = _f32(0.3 * rs.randn(p.hidden[i]))
    for i in range(p.L + 1):
        if i > 0:
            p.bzu[i] = _f32(0.3 * rs.randn(p.sizes[i - 1]))
        p.byu[i] = _f32(0.5 + 0.3 * rs.randn(p.n))
        p.bzx[i] = _f32(0.3 * rs.randn(p.sizes[i]))


def case_inputs(tag):
    """-> dict(p, x, y, bnvars, and the case's scalars).  ``bnvars[i]`` = (gamma, beta, moving_mean, moving_variance)
    of the batch-norm after u_i (multi-label f applies one for every i < L-1), ``p.bn`` the matching affine map or
    None when the variables are the identity (variance 1 - eps, so that variance + eps = 1)."""
    rs = np.random.RandomState(abs(hash_tag(tag)) % (2 ** 31))
    c = dict(tag=tag)
    if tag == "ml_fg_c3":            # the shape / inputs of tests/test_gpu_picnn.py::test_fg_matches_oracle[C3-77]
        p, x, y0 = workloads.make_inputs("C3", B=77)
        y = _f32(np.random.RandomState(11).uniform(0.02, 0.98, size=y0.shape))
        c.update(p=p, x=x, y=y, layerSizes=[600])
    elif tag == "ml_fg_bn":          # three z-layers, odd widths, biases, real batch-norm statistics
        p = workloads.synth_params(31, 10, 7, [12, 9, 7])
        _random_biases(p, rs)
        x = _f32(rs.randn(16, 10))
        y = _f32(rs.uniform(0.02, 0.98, size=(16, 7)))
        c.update(p=p, x=x, y=y, layerSizes=[12, 9])
        c["bnvars"] = [(_f32(rs.uniform(0.5, 1.5, s)), _f32(0.2 * rs.randn(s)), _f32(0.3 * rs.randn(s)),
                        _f32(rs.uniform(0.5, 2.0, s))) for s in p.hidden[:-1]]
    elif tag == "rl_fg_c4":          # the shape / inputs of test_fg_matches_oracle[C4-300]
        p, x, y0 = workloads.make_inputs("C4", B=300)
        y = _f32(np.random.RandomState(11).uniform(0.02, 0.98, size=y0.shape))
        c.update(p=p, x=x, y=y)
    elif tag == "rl_fg_entr_c4":     # func = _fg_entr of Agent.adam: actions in [-1, 1] incl. the clipped ends of entropy()
        p, x, y0 = workloads.make_inputs("C4", B=40)
        a = _f32(rs.uniform(-1.0, 1.0, size=y0.shape))
        a[::7, 0], a[3::9, 2] = 1.0 - 1e-8, -1.0 + 1e-8      # where Agent.adam clips to (:211)
        c.update(p=p, x=x, y=a)
    elif tag == "rl_act_c4":         # Agent.bundle_entropy end to end (reference solveBatch on the reference negQ)
        p, x, y0 = workloads.make_inputs("C4", B=48)
        c.update(p=p, x=x, y=y0)
    elif tag == "trace_c3":          # ebundle-vs-gd.py:84-107: nSamples = 10 rows, 10 bundle iterations, callback trace of mean(f - H)
        p, x, y0 = workloads.make_inputs("C3", B=10)
        c.update(p=p, x=x, y=y0, layerSizes=[600], nIter=10)
    elif tag == "gd_c3":             # the case of test_momentum_gd_matches_oracle[C3-50-0.01-0.3] (script defaults)
        p, x, y0 = workloads.make_inputs("C3", B=50)
        c.update(p=p, x=x, y=y0, layerSizes=[600], lr=0.01, momentum=0.3, nIter=30,
                 trueY=(rs.uniform(size=y0.shape) < 0.1).astype(np.float64))
    elif tag == "gdgrad_small":      # every parameter gradient of the unrolled loop on a net small enough to store
        p = workloads.synth_params(32, 12, 9, [14, 11, 9])
        for i in range(len(p.Wy)):
            p.Wy[i] = _f32(3.0 * p.Wy[i])
        _random_biases(p, rs)
        x = _f32(rs.randn(20, 12))
        c.update(p=p, x=x, y=np.full((20, 9), 0.5), layerSizes=[14, 11], lr=0.02, momentum=0.5, nIter=7,
                 trueY=(rs.uniform(size=(20, 9)) < 0.3).astype(np.float64))
    else:
        raise KeyError(tag)
    p = c["p"]
    if "bnvars" in c:
        p.bn = [workloads.bn_affine(*v, eps=BN_EPS) for v in c["bnvars"]] + [None]
    elif p.alpha == 0.0:             # multi-label f always applies bn: identity statistics
        c["bnvars"] = [(np.ones(s), np.zeros(s), np.zeros(s), np.full(s, 1.0 - BN_EPS)) for s in p.hidden[:-1]]
    return c


def hash_tag(tag):
    return sum((i + 1) * ord(ch) for i, ch in enumerate(tag)) * 7919


CASES = ["ml_fg_c3", "ml_fg_bn", "rl_fg_c4", "rl_fg_entr_c4", "rl_act_c4", "trace_c3", "gd_c3", "gdgrad_small"]


# --------------------------------------------------------------------------------------------------------
# reference code on the shim
# --------------------------------------------------------------------------------------------------------

def _shim(c, feeds, prefix=""):
    sh = Shim(variables_from_params(c["p"], c.get("bnvars"), prefix))
    for k, (a, rg) in feeds.items():
        sh.feed(k, a, requires_grad=rg)
    return sh


def run_multilabel_model(c, rel, ctor_args):
    """Model(...) of a multi-label script: building it evaluates the whole graph on the fed tensors."""
    B, n = c["y"].shape
    rs = np.random.RandomState(5)
    feeds = {"x": (c["x"], False), "y": (c["y"], True), "trueY": (c.get("trueY", np.zeros((B, n))), False),
             "v": (rs.randn(B, n), False), "c": (rs.randn(B), False)}
    sh = _shim(c, feeds)
    ns = refcode.extract(rel, ["Model"], {"tf": sh.tf, "tflearn": sh.tflearn, "np": np,
                                          "variable_summaries": lambda *a, **k: None})
    with refcode.quiet():
        model = ns["Model"](c["p"].m, c["p"].n, *ctor_args, None)
    assert not sh.unused_variables(), sh.unused_variables()
    assert model.szs == c["p"].hidden
    return sh, model


def run_negq(c, agent_ns, obs, act, entr=False):
    """One evaluation of Agent.negQ and tf.gradients(negQ, act) (RL/src/icnn.py:59-63), under scope 'q'."""
    sh = _shim(c, {"obs": (obs, False), "act": (act, True)}, prefix="q/")
    agent_ns["tf"], agent_ns["tflearn"] = sh.tf, sh.tflearn
    agent = agent_ns["Agent"].__new__(agent_ns["Agent"])
    agent.dimA, agent.dimO = c["p"].n, c["p"].m
    agent.sess = types.SimpleNamespace(close=lambda: None)
    with sh.tf.variable_scope("q"):
        negQ = agent.negQ(sh.feeds["obs"], sh.feeds["act"])
    (grad,) = sh.tf.gradients(negQ, sh.feeds["act"])
    assert not sh.unused_variables(), sh.unused_variables()
    if entr:        # negQ_entr = negQ - entropy(act), act_grad_entr (RL/src/icnn.py:60-63, entropy :455-458)
        negQ_entr = negQ - agent_ns["entropy"](sh.feeds["act"])
        (grad_entr,) = sh.tf.gradients(negQ_entr, sh.feeds["act"])
        return agent, negQ_entr.detach().numpy().copy(), grad_entr.detach().numpy().copy()
    return agent, negQ.detach().numpy().copy(), grad.detach().numpy().copy()


# ---- the convolutional PICNN of completion/ (callback-mode fg of the GPU tests) ---------------------------------

CONV_CASES = {"conv_small": (4, 16, 8, 3), "conv_olivetti": (2, 64, 32, 1)}     # tag -> (B, H, W, seed)


def conv_case(tag):
    """-> (ConvPICNN float64, x [B, H*W], y [B, H*W]) of oracle/conv_picnn.py, seeded."""
    import torch
    from oracle.conv_picnn import ConvPICNN
    B, H, W, seed = CONV_CASES[tag]
    net = ConvPICNN(H, W, seed=seed, dtype=torch.float64)
    rs = np.random.RandomState(100 + seed)
    return net, rs.uniform(size=(B, H * W)), rs.uniform(0.05, 0.95, size=(B, H * W))


def conv_variables(net):
    """oracle/conv_picnn.py parameters -> the reference's variable names and TensorFlow layouts: conv kernels
    [k, k, c_in, c_out]; the dense layers behind the last conv see its feature map flattened in NHWC order.  The
    architecture is read off the parameters, not off a module's CONVS / FCS, so any net of that class converts: each
    conv layer's stride is the reference's for its kernel size (8 -> 4, 4 -> 2, 3 -> 1), checked against the width
    of the first dense layer."""
    P = net.P
    v = {}
    nc = sum(k.startswith("y_red") for k in P)
    cw = lambda w: w.permute(2, 3, 1, 0).numpy()                                    # noqa: E731
    h, w = net.H, net.W
    for i in range(nc):
        k = P["u%d" % i][0].shape[-1]
        s_ = k // 2 if k % 2 == 0 else 1
        h, w = -(-h // s_), -(-w // s_)
    C = P["u%d" % (nc - 1)][0].shape[0]
    assert P["u%d" % nc][0].shape[0] == C * h * w, "the conv strides do not follow the kernel-size rule"
    perm = np.arange(C * h * w).reshape(C, h, w).transpose(1, 2, 0).reshape(-1)     # NHWC position -> NCHW index
    for i in range(sum(k.startswith("z_u") for k in P)):
        conv = i < nc
        Wu, bu = P["u%d" % i]
        v["u%d/W" % i] = cw(Wu) if conv else (Wu.numpy()[perm] if i == nc else Wu.numpy())
        v["u%d/b" % i] = bu.numpy()
        width = Wu.shape[0] if conv else Wu.shape[1]
        if conv or width != 1:          # bn(...) on every u layer but the width-1 one (:352-366); identity statistics
            for nm, a in (("gamma", np.ones(width)), ("beta", np.zeros(width)), ("moving_mean", np.zeros(width)),
                          ("moving_variance", np.full(width, 1.0 - BN_EPS))):
                v["u%d/BatchNormalization/%s" % (i, nm)] = a
        if i > 0:
            Wq, bq = P["zu_u%d" % i]
            if conv:
                v["z%d_zu_u/W" % i], v["z%d_zu_proj/W" % i] = cw(Wq), cw(P["zu_proj%d" % i])
                v["z%d_zu_u/b" % i] = bq.numpy()
            elif i == nc:
                v["z%d_zu_u/W" % i], v["z%d_zu_u/b" % i] = Wq.numpy()[perm][:, perm], bq.numpy()[perm]
                v["z%d_zu_proj/W" % i] = P["zu_proj%d" % i].numpy()[perm]
            else:
                v["z%d_zu_u/W" % i], v["z%d_zu_u/b" % i] = Wq.numpy(), bq.numpy()
                v["z%d_zu_proj/W" % i] = P["zu_proj%d" % i].numpy()
        if conv:
            v["z%d_yu_u/W" % i], v["z%d_yu_u/b" % i] = cw(P["yu_u%d" % i][0]), P["yu_u%d" % i][1].numpy()
            v["z%d_yu/W" % i] = cw(P["yu%d" % i])
            v["z%d_y_red/W" % i], v["z%d_y_red/b" % i] = cw(P["y_red%d" % i][0]), P["y_red%d" % i][1].numpy()
        Wz, bz = P["z_u%d" % i]
        v["z%d_u/W" % i] = cw(Wz) if conv else (Wz.numpy()[perm] if i == nc else Wz.numpy())
        v["z%d_u/b" % i] = bz.numpy()
    return v


def run_completion_model(tag):
    net, x, y = conv_case(tag)
    B, H, W, _ = CONV_CASES[tag]
    sh = Shim(conv_variables(net))
    rs = np.random.RandomState(5)
    for k, a, rg in (("x", x.reshape(B, H, W, 1), False), ("y", y.reshape(B, H, W, 1), True),
                     ("trueY", np.zeros((B, H, W, 1)), False), ("v", rs.randn(B, H * W), False), ("c", rs.randn(B), False),
                     ("l_yN", np.zeros(()), False), ("nBundleIter", np.zeros(B), False), ("nActive", np.zeros(B), False)):
        sh.feed(k, a, requires_grad=rg)
    ns = refcode.extract("completion/icnn_ebundle.py", ["Model"],
                         {"tf": sh.tf, "tflearn": sh.tflearn, "np": np, "variable_summaries": lambda *a, **k: None})
    with refcode.quiet(), tensor_get_shape():
        model = ns["Model"]([H, W, 1], [H, W, 1], None)
    assert not sh.unused_variables(), sh.unused_variables()
    return model.E_.detach().numpy(), model.dE_dyFlat_.detach().numpy(), len(sh.created)


def generate():
    """-> {name: array}: every golden of tests/golden/picnn_tfshim.npz, recomputed from the reference checkout."""
    out = {}

    # ---- multi-label Model (bundle-entropy script): E_ and dE_dy_ ------------------------------------------------
    for tag in ("ml_fg_c3", "ml_fg_bn"):
        c = case_inputs(tag)
        sh, model = run_multilabel_model(c, "multi-label-cls/icnn_ebundle.py", (list(c["layerSizes"]),))
        out[tag + "_f"] = model.E_.detach().numpy()
        out[tag + "_g"] = model.dE_dy_.detach().numpy()
        out[tag + "_g_entr"] = model.dE_entr_dy_.detach().numpy()
        print(tag, "variables in creation order:", len(sh.created), "f[:3]", out[tag + "_f"][:3])

    # ---- RL Agent.negQ and Agent.bundle_entropy ---------------------------------------------------------------
    flags = types.SimpleNamespace(l1size=200, l2size=200, icnn_bn=False, lrelu=0.01)
    ref_rl = refcode.load("bundle_entropy", "RL/src/bundle_entropy.py")
    agent_ns = {"np": np, "FLAGS": flags, "bundle_entropy": ref_rl, "variable_summaries": lambda *a, **k: None}
    refcode.extract("RL/src/icnn.py", ["Agent", "entropy"], agent_ns)
    c = case_inputs("rl_fg_c4")
    # the wrapper of Agent.bundle_entropy (:150-153), applied by hand for the fg golden: a = 2x - 1, grad *= 2
    _agent, f, g = run_negq(c, agent_ns, c["x"], 2.0 * c["y"] - 1.0)
    out["rl_fg_c4_f"], out["rl_fg_c4_g"] = f, 2.0 * g
    c = case_inputs("rl_fg_entr_c4")
    _agent, out["rl_fg_entr_c4_f"], out["rl_fg_entr_c4_g"] = run_negq(c, agent_ns, c["x"], c["y"], entr=True)
    c = case_inputs("rl_act_c4")
    agent, _f, _g = run_negq(c, agent_ns, c["x"], 2.0 * c["y"] - 1.0)

    def func(obs, act):                      # what Fun([obs, act], [negQ, act_grad]) returns (:107)
        _a, f_, g_ = run_negq(c, agent_ns, obs, act)
        return f_, g_
    with refcode.quiet():
        out["rl_act_c4_act"] = agent.bundle_entropy(func, c["x"])
    print("rl_act_c4 act[0]", out["rl_act_c4_act"][0])

    # ---- the reference's own benchmark of the inner loop (multi-label-cls/ebundle-vs-gd.py:84-107): its Model graph as fg,
    # its lib/bundle_entropy.solveBatch, its entr(), and the callback (t, es, x) -> mean(es - entr(x)) it plots
    c = case_inputs("trace_c3")
    ref_pc = refcode.load("ref_pc_trace", "lib/bundle_entropy.py")
    entr = refcode.extract("multi-label-cls/ebundle-vs-gd.py", ["entr"], {"np": np})["entr"]
    trace, iters = [], []

    def fg_ref(yhats):                       # sess.run([model.E_, model.dE_dy_]) (:88-91)
        cc = dict(c, y=np.asarray(yhats, dtype=np.float64))
        _sh, model = run_multilabel_model(cc, "multi-label-cls/icnn_ebundle.py", (list(c["layerSizes"]),))
        return model.E_.detach().numpy().copy(), model.dE_dy_.detach().numpy().copy()

    def cb(iterNum, es, x):                  # :93-98
        iters.append(iterNum)
        trace.append(np.mean(es - entr(x)))
    with refcode.quiet():
        r = ref_pc.solveBatch(fg_ref, c["y"].copy(), nIter=c["nIter"], callback=cb)
    out["trace_c3_iters"], out["trace_c3_f_minus_H"], out["trace_c3_yN"] = np.array(iters), np.array(trace), r[0]
    print("trace_c3 mean(f - H) per iteration:", np.round(trace, 3))

    # ---- multi-label Model (back-optimisation script): unrolled momentum GD and its training gradient ----------
    for tag in ("gd_c3", "gdgrad_small"):
        c = case_inputs(tag)
        args = types.SimpleNamespace(layerSizes=list(c["layerSizes"]), inference_lr=c["lr"],
                                     inference_momentum=c["momentum"], inference_nIter=c["nIter"])
        sh, model = run_multilabel_model(c, "multi-label-cls/icnn-back.py", (args,))
        out[tag + "_yN"] = model.yn_.detach().numpy()
        out[tag + "_energies"] = model.energies_.detach().numpy()
        out[tag + "_mse"] = np.array(float(model.mse_.detach()))
        names = []
        for g_, v_ in sh.tf.train.AdamOptimizer().compute_gradients(model.mse_, model.theta_):
            nm = v_.name[:-2].replace("/", "__")
            names.append(nm)
            ga = np.zeros(tuple(v_.value.shape)) if g_ is None else g_.detach().numpy()
            if tag == "gdgrad_small" or ga.size <= 1024:      # gd_c3: biases and the width-1 output layer only
                out["%s_grad_%s" % (tag, nm)] = ga
        out[tag + "_theta"] = np.array(names)
        print(tag, "mse", out[tag + "_mse"], "theta", len(names), "stored grads",
              sum(k.startswith(tag + "_grad_") for k in out))

    # ---- completion Model: the convolutional PICNN ------------------------------------------------------------------
    for tag in CONV_CASES:
        out[tag + "_f"], out[tag + "_g"], nv = run_completion_model(tag)
        print(tag, "variables", nv, "f", out[tag + "_f"])

    return out


if __name__ == "__main__":
    regen.main(("gen_golden_tfshim",))
