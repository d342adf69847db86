"""numpy float64 restatement of the RL agent's TD training step (test infrastructure).

What the reference computes (RL/src/icnn.py:55-109, ``--icnn_opt adam``):

    q_entr        = -(negQ(obs, act) - H(act))                       H = entropy (:455-458)
    q_target_entr = -(negQ_target(ob2, act2) - H(act2))
    y  = select(term2, rew, rew + discount q_target_entr);  y = min(q_entr + 1, max(q_entr - 1, y));  stop_gradient
    td = q_entr - y;  loss_q = mean(td^2) + l2norm * sum_W weight_decay * sum(W^2) / 2
    grads_and_vars_q = compute_gradients(loss_q)

y is constant for the gradient, so d mean(td^2) / d negQ_u = c_u = -2 td_u / B and the TD part of the gradient is
that of sum_u c_u negQ(obs_u, act_u): oracle/bundle_grad_np.bundle_grad at Y = act, V = 0, one row per sample
(its forward is oracle/picnn_np's recurrence, its x-path backprop ``xpath_backward``).  The L2 term adds
l2norm * weight_decay * W to every weight matrix and nothing to the biases.  Pinned by tests/test_td_grad_golden_cpu.py
against the reference's own code on the TF shim (tests/golden/rl/td_grad.npz, oracle/gen_golden_td_grad.py).
"""
from __future__ import annotations

import numpy as np

from oracle import bundle_grad_np as bg
from icnn_b200 import workloads

DISCOUNT, L2NORM, WEIGHT_DECAY = 0.99, 1e-4, 1e-3
WEIGHTS = ("Wy", "Wz", "Wu", "Wzu", "Wyu", "Wzx")
PARAMS = bg.PARAMS
CLAMP_GAP = 1e-5          # golden rows keep the unclamped target at least this far from q_entr -/+ 1


def entropy(a):
    p = np.clip((np.asarray(a, dtype=np.float64) + 1.0) / 2.0, 1e-4, 1.0 - 1e-4)
    return -(p * np.log(p) + (1.0 - p) * np.log(1.0 - p)).sum(axis=1)


def negq(p, obs, act):
    """negQ(obs_u, act_u) per sample (the energy, layer L's pre-activation)."""
    B = len(act)
    _, zs, _, _, _ = bg.row_pass(p, obs, act, np.zeros_like(np.asarray(act, dtype=np.float64)), np.zeros(B),
                                 np.ones(B, dtype=np.int64))
    return zs[p.L][:, 0]


def td_parts(p, pt, obs, act, rew, ob2, act2, term, discount=DISCOUNT):
    """-> (td, q_entr, y before the clamp)."""
    q = -(negq(p, obs, act) - entropy(act))
    qt = -(negq(pt, ob2, act2) - entropy(act2))
    rew = np.asarray(rew, dtype=np.float64)
    y0 = np.where(np.asarray(term, dtype=bool), rew, rew + discount * qt)
    y = np.minimum(q + 1.0, np.maximum(q - 1.0, y0))
    return q - y, q, y0


def clamp_gap(q, y0):
    """Per row: how far the unclamped target sits from the clamp boundaries q -/+ 1."""
    return np.minimum(np.abs(y0 - (q - 1.0)), np.abs(y0 - (q + 1.0)))


def l2_loss(p, weight_decay=WEIGHT_DECAY):
    return sum(weight_decay * 0.5 * float(np.sum(np.asarray(w, dtype=np.float64) ** 2))
               for k in WEIGHTS for w in getattr(p, k) if w is not None)


def td_grad(p, pt, obs, act, rew, ob2, act2, term, discount=DISCOUNT, l2norm=L2NORM, weight_decay=WEIGHT_DECAY):
    """-> (loss_q, td, grads): grads maps PARAMS to per-layer lists summed over the minibatch (with the L2 term) and
    'dcy', 'dcz', 'dd' to the per-sample gate adjoints of mean(td^2)."""
    td, _, _ = td_parts(p, pt, obs, act, rew, ob2, act2, term, discount)
    B = len(td)
    c = -2.0 * td / B
    act = np.asarray(act, dtype=np.float64)
    g = bg.bundle_grad(p, obs, act, np.zeros_like(act), c, np.ones(B, dtype=np.int64), per_sample=False)
    lam = l2norm * weight_decay
    for k in WEIGHTS:
        g[k] = [None if w is None else gk + lam * np.asarray(w, dtype=np.float64) for gk, w in zip(g[k], getattr(p, k))]
    return float(np.mean(td ** 2) + l2norm * l2_loss(p, weight_decay)), td, g


# ---- seeded cases (shared by the golden generator and the tests) -------------------------------------------------

def _f32(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def make_net(tag, seed):
    if tag == "c4":           # the RL configuration: m 17, n 6, hidden [200, 200], alpha 0.01, gate biases 1
        p, _, _ = workloads.make_inputs("C4", B=1, seed=seed)
        return p
    rs = np.random.RandomState(seed)   # a small odd-width net with non-zero biases everywhere
    p = workloads.synth_params(seed, 5, 3, [7, 5], alpha=0.01, gate_bias=1.0)
    for i in range(p.L):
        p.bu[i] = _f32(0.3 * rs.randn(p.hidden[i]))
    for i in range(p.L + 1):
        if i > 0:
            p.bzu[i] = _f32(0.5 + 0.3 * rs.randn(p.sizes[i - 1]))
        p.byu[i] = _f32(0.5 + 0.3 * rs.randn(p.n))
        p.bzx[i] = _f32(0.3 * rs.randn(p.sizes[i]))
    return p


def make_rows(p, pt, B, seed, discount=DISCOUNT):
    """Minibatch (obs, act, rew, ob2, act2, term) in float32 values: terminal and non-terminal rows, the clamp active
    from above and from below and inactive, actions at -1 / +1 (the entropy clip), and no row within CLAMP_GAP of a
    clamp boundary."""
    rs = np.random.RandomState(seed)
    obs, ob2 = _f32(rs.randn(B, p.m)), _f32(rs.randn(B, p.m))
    act, act2 = _f32(rs.uniform(-1, 1, (B, p.n))), _f32(rs.uniform(-1, 1, (B, p.n)))
    act[::3, 0], act[1::4, -1], act2[::5, 0], act2[2::3, -1] = 1.0, -1.0, -1.0, 1.0
    term = (np.arange(B) % 4) == 1
    q = -(negq(p, obs, act) - entropy(act))
    qt = -(negq(pt, ob2, act2) - entropy(act2))
    # wanted y0 - q: inside the clamp, above q + 1, below q - 1 (cycled over the rows)
    off = np.array([0.37, 1.6, -1.45, -0.62, 2.3, -2.8])[np.arange(B) % 6] + 0.05 * rs.uniform(-1, 1, B)
    rew = _f32(np.where(term, q + off, q + off - discount * qt))
    _, q, y0 = td_parts(p, pt, obs, act, rew, ob2, act2, term, discount)
    assert clamp_gap(q, y0).min() > 10 * CLAMP_GAP
    return obs, act, rew, ob2, act2, term


CASES = {"c4": (24, 7, 8), "small": (16, 3, 4)}     # tag -> (B, net seed, target-net seed)


def case(tag):
    """-> dict(p, pt, obs, act, rew, ob2, act2, term) of a golden case."""
    B, s1, s2 = CASES[tag]
    p, pt = make_net(tag, s1), make_net(tag, s2)
    obs, act, rew, ob2, act2, term = make_rows(p, pt, B, 100 + s1)
    return dict(p=p, pt=pt, obs=obs, act=act, rew=rew, ob2=ob2, act2=act2, term=term)
