#!/usr/bin/env python
"""Golden vectors of the RL agent's TD training step, produced by EXECUTING THE REFERENCE'S OWN code.

Executed reference code (paths relative to a locuslab/icnn checkout), unmodified, cut out with ``ast``:
  RL/src/icnn.py   the statements of Agent.__init__ from ``obs = tf.placeholder`` (:55) through
                   ``grads_and_vars_q = optim_q.compute_gradients(loss_q)`` (:108) -- both scopes' negQ, the TD
                   target with its clamp, ms_td_error, the L2 losses, theta_, makeCvx / proj, update_target --
                   plus Agent.negQ (:325-404) and entropy (:455-458)
on oracle/tf_shim.py with the RL primitives of oracle/tf_shim_rl.py.  FLAGS are the RL/src/agent.py defaults with
icnn_opt = 'adam' and icnn_bn = False (l1size / l2size: the case's hidden widths); the scalars Agent.__init__ reads from FLAGS before :55 (tau, discount,
l2norm, learning_rate) are bound from the same FLAGS.  The feeds are float32 values, as the reference's placeholders
hold them.  Stored per case: loss_q, td and gv_ (d loss_q / d v under the reference's variable names, '/' -> '__'):
every array of the small net, the arrays of at most 4096 entries at C4 dims.  Weights and rows are regenerated from
seeds by oracle/td_grad_np.case.  Deterministic: a second run writes identical bytes.

TEST INFRASTRUCTURE ONLY; needs a checkout of the reference at $ICNN_REFERENCE_DIR.
Usage:  python -m oracle.gen_golden_td_grad   -> tests/golden/rl/td_grad.npz
"""
import types

import numpy as np
import torch

from oracle import refcode, regen
from oracle import td_grad_np as tg
from oracle.tf_shim import variables_from_params
from oracle.tf_shim_rl import RLShim

GOLDEN = "rl/td_grad.npz"
FIRST = 'obs = tf.placeholder(tf.float32, [None, dimO], "obs")'             # RL/src/icnn.py:55
LAST = "grads_and_vars_q = optim_q.compute_gradients(loss_q)"               # RL/src/icnn.py:108
FLAGS = types.SimpleNamespace(l1size=200, l2size=200, icnn_bn=False, lrelu=0.01, icnn_opt="adam", tau=0.01,
                              discount=0.99, l2norm=0.0001, rate=0.001, outheta=0.15, ousigma=0.1)


def run_case(c):
    p, pt = c["p"], c["pt"]
    v = variables_from_params(p, prefix="q/")
    v.update(variables_from_params(pt, prefix="q_target/"))
    sh = RLShim(v)
    for k, a, rg in (("obs", c["obs"], False), ("act", c["act"], True), ("rew", c["rew"], False),
                     ("obs_target", c["ob2"], False), ("act_target", c["act2"], True)):
        sh.feed(k, a, requires_grad=rg)
    sh.feeds["term_target"] = torch.as_tensor(np.asarray(c["term"], dtype=bool))
    flags = types.SimpleNamespace(**vars(FLAGS))
    flags.l1size, flags.l2size = p.hidden          # negQ's two layer sizes (:326)
    ns = {"np": np, "FLAGS": flags, "bundle_entropy": None, "variable_summaries": lambda *a, **k: None,
          "tf": sh.tf, "tflearn": sh.tflearn}
    refcode.extract("RL/src/icnn.py", ["Agent", "entropy"], ns)
    agent = ns["Agent"].__new__(ns["Agent"])
    agent.dimA, agent.dimO = p.n, p.m
    agent.sess = types.SimpleNamespace(close=lambda: None)
    ns.update(self=agent, dimA=p.n, dimO=p.m, tau=FLAGS.tau, discount=FLAGS.discount, l2norm=FLAGS.l2norm,
              learning_rate=FLAGS.rate)
    with refcode.quiet():
        refcode.run_statements("RL/src/icnn.py", "Agent.__init__", FIRST, LAST, ns)
    assert not sh.unused_variables(), sh.unused_variables()
    out = dict(loss_q=np.array(float(ns["loss_q"].detach())), td=ns["td_error"].detach().numpy().copy())
    names = []
    for g, var in ns["grads_and_vars_q"]:
        name = var.name[:-2]
        if name.startswith("q_target/"):
            assert g is None, name            # y is under stop_gradient: the target network gets no gradient
            continue
        assert name.startswith("q/") and g is not None, name
        names.append(name)
        out["gv_" + name.replace("/", "__")] = g.detach().numpy().copy()
    assert len(agent.theta_) == len(names) == len(agent.theta_target_)
    return out, names


def generate():
    res = {}
    for tag in tg.CASES:
        out, names = run_case(tg.case(tag))
        res["%s_loss_q" % tag], res["%s_td" % tag] = out["loss_q"], out["td"]
        res["%s_theta" % tag] = np.array(names)
        for k, a in out.items():
            if k.startswith("gv_") and (tag == "small" or a.size <= 4096):
                res["%s_%s" % (tag, k)] = a
        print(tag, "loss_q", float(out["loss_q"]), "variables", len(names))
    return res


if __name__ == "__main__":
    regen.main(("gen_golden_td_grad",))
