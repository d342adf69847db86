"""The RL agent's TD training gradient on the GPU (icnn_td_grad, icnn_b200.td_grad) against the reference's own code
on the TF shim (tests/golden/rl/td_grad.npz) and the float64 oracle (oracle/td_grad_np.py).

Tolerance (test_gpu_bundle_grad's rule): every array must agree to RTOL = 2e-4 of its largest entry.  A float32
evaluation of a row whose pre-activation sits within 1e-5 (relative) of zero can land on the other side of the leaky
ReLU kink, and a row whose unclamped TD target sits within 1e-5 of a clamp boundary q -/+ 1 can land on the other
side of the clamp: either changes that sample's gradient by O(1).  Such a sample may be set aside only when it
disagrees AND the float64 oracle shows it that close, at most max(1, 2 %) of the samples; the rest is compared again
without it."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import bundle_grad_np as bg
from oracle import td_grad_np as tg
from oracle.gen_golden_bundle_grad import tf_name_to_param

pytestmark = pytest.mark.gpu
np.seterr(all="ignore")

RTOL = 2e-4
KINK = 1e-5
GATES = ("dcy", "dcz", "dd")


def relerr(a, b):
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(np.asarray(a, dtype=np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def _nets(p, pt):
    import icnn_b200
    return icnn_b200.PICNN.from_params(p, device="cuda"), icnn_b200.PICNN.from_params(pt, device="cuda")


def _device(net, tnet, rows, **kw):
    from icnn_b200.td_grad import td_grad
    obs, act, rew, ob2, act2, term = rows
    return td_grad(net.bind(obs), tnet.bind(ob2), obs, act, rew, act2, term, **kw)


def _subset(rows, keep):
    return tuple(np.asarray(a)[keep] for a in rows)


def _compare(p, pt, net, tnet, rows, tag):
    """Device vs oracle on ``rows`` after setting aside what the kink / clamp rule allows."""
    obs, act, rew, ob2, act2, term = rows
    B = len(act)
    loss, td, dev = _device(net, tnet, rows)
    oloss, otd, orc = tg.td_grad(p, pt, obs, act, rew, ob2, act2, term)
    bad = np.abs(td - otd) >= RTOL * max(np.abs(otd).max(), 1e-30)
    for k in GATES:
        for a, b in zip(dev[k], orc[k]):
            if b is not None:
                bad |= np.abs(a - b).max(axis=1) / max(np.abs(b).max(), 1e-30) >= RTOL
    _, q, y0 = tg.td_parts(p, pt, obs, act, rew, ob2, act2, term)
    near = (bg.min_rel_preact(p, obs, act, np.ones(B, dtype=np.int64)) < KINK) | \
           (tg.clamp_gap(q, y0) < KINK * np.maximum(1.0, np.abs(q)))
    assert not (bad & ~near).any(), np.nonzero(bad & ~near)[0][:10]
    drop = bad & near
    assert drop.sum() <= max(1, int(0.02 * B)), (int(drop.sum()), B)
    if drop.any():
        rows = _subset(rows, ~drop)
        loss, td, dev = _device(net, tnet, rows)
        oloss, otd, orc = tg.td_grad(p, pt, *rows)
    errs = {"loss": abs(loss - oloss) / abs(oloss), "td": relerr(td, otd)}
    for k in tg.PARAMS + GATES:
        for i, b in enumerate(orc[k]):
            if b is not None:
                errs["%s%d" % (k, i)] = relerr(dev[k][i], b)
    worst = max(errs, key=errs.get)
    print(tag, "B", B, "set aside", int(drop.sum()), "max rel err %.2e (%s)" % (errs[worst], worst))
    assert errs[worst] < RTOL, errs


def _last_mode():
    from icnn_b200 import _capi
    out = (C.c_int32 * 5)()
    assert _capi.lib.icnn_tc_last_launch(out) == 0
    return out[4]


@pytest.mark.parametrize("tag", ["small", "c4"])
def test_reference_golden(tag, golden_dir):
    """loss_q, td and every stored gv_ of the reference's own Agent graph on the shim."""
    gold = np.load(os.path.join(golden_dir, "rl", "td_grad.npz"))
    c = tg.case(tag)
    net, tnet = _nets(c["p"], c["pt"])
    rows = (c["obs"], c["act"], c["rew"], c["ob2"], c["act2"], c["term"])
    loss, td, dev = _device(net, tnet, rows)
    assert abs(loss - float(gold[tag + "_loss_q"])) <= RTOL * abs(float(gold[tag + "_loss_q"]))
    assert relerr(td, gold[tag + "_td"]) < RTOL
    n = 0
    for name in gold[tag + "_theta"]:
        key = "%s_gv_%s" % (tag, str(name).replace("/", "__"))
        if key not in gold.files:
            continue
        k, i = tf_name_to_param(str(name)[2:])
        g = dev[k][i].reshape(gold[key].shape)
        assert relerr(g, gold[key]) < RTOL, (name, relerr(g, gold[key]))
        n += 1
    assert n >= 15, n


@pytest.mark.parametrize("B", [1, 63, 64, 256, 4096, 65536])
def test_c4_against_oracle(B):
    """C4 dims on both GEMM paths (3xTF32 wgmma for B >= 64, FP32 FFMA below), every array against float64."""
    p, pt = tg.make_net("c4", 7), tg.make_net("c4", 8)
    rows = tg.make_rows(p, pt, B, 1000 + B)
    net, tnet = _nets(p, pt)
    from icnn_b200.td_grad import _launch
    from icnn_b200.gd_grad import _f32
    obs, act, rew, ob2, act2, term = rows
    fg, fgt = net.bind(obs), tnet.bind(ob2)
    negq_t, _ = fgt.fg_device(_f32(act2, net.device))
    net.gates(_f32(obs, net.device))               # a mode-3 (x-path) tensor-core GEMM last
    assert _last_mode() == 3
    dv = lambda a, dt=torch.float32: torch.as_tensor(np.asarray(a), device=net.device).to(dt).contiguous()  # noqa: E731
    _launch(fg, dv(act), negq_t, dv(act2), dv(rew), dv(term, torch.uint8), 0.99)
    torch.cuda.synchronize()
    assert _last_mode() == (1 if B >= 64 else 3)   # backward on the wgmma GEMM, or no tensor-core GEMM at all
    _compare(p, pt, net, tnet, rows, "c4")


@pytest.mark.parametrize("B", [63, 4096])
def test_equals_train_grad_with_zero_direction(B):
    """icnn_td_grad's y-path gradients and gate adjoints are icnn_train_grad's at Y = act, V = 0, c = -2 td / B,
    one row per sample."""
    from icnn_b200.bundle_grad import train_grad
    p, pt = tg.make_net("c4", 7), tg.make_net("c4", 8)
    rows = tg.make_rows(p, pt, B, 2000 + B)
    net, tnet = _nets(p, pt)
    obs, act, rew, ob2, act2, term = rows
    _loss, td, dev = _device(net, tnet, rows, l2norm=0.0)
    c = -2.0 * td.astype(np.float64) / B
    ref = train_grad(net.bind(obs), act, np.zeros_like(act), c.astype(np.float32), np.ones(B, dtype=np.int64))
    for k in ("Wy", "Wz") + GATES:
        for i, b in enumerate(ref[k]):
            if b is not None:
                assert relerr(dev[k][i], b) < RTOL, (k, i, relerr(dev[k][i], b))


def test_deterministic():
    p, pt = tg.make_net("c4", 7), tg.make_net("c4", 8)
    for B in (63, 4096):
        rows = tg.make_rows(p, pt, B, 3000 + B)
        net, tnet = _nets(p, pt)
        l1, t1, g1 = _device(net, tnet, rows)
        l2, t2, g2 = _device(net, tnet, rows)
        assert l1 == l2 and np.array_equal(t1, t2)
        for k in g1:
            for a, b in zip(g1[k], g2[k]):
                assert (a is None and b is None) or np.array_equal(a, b), k


def test_affine_binding_refused():
    from icnn_b200 import _capi
    from icnn_b200.td_grad import _launch, td_grad
    c = tg.case("small")
    net, tnet = _nets(c["p"], c["pt"])
    rows = (c["obs"], c["act"], c["rew"], c["act2"], c["term"])
    with pytest.raises(ValueError, match="affine"):
        td_grad(net.bind(c["obs"], affine=True), tnet.bind(c["ob2"]), *rows)
    with pytest.raises(ValueError, match="affine"):
        td_grad(net.bind(c["obs"]), tnet.bind(c["ob2"], affine=True), *rows)
    fg = net.bind(c["obs"], affine=True)
    B, n = fg.B, net.n
    z = lambda *s: torch.zeros(*s, device=net.device)  # noqa: E731
    with pytest.raises(_capi.IcnnError, match="affine"):
        _launch(fg, z(B, n), z(B), z(B, n), z(B), torch.zeros(B, dtype=torch.uint8, device=net.device), 0.99)


def test_training_step_matches_oracle_step():
    """adam.solve on the target -> td_grad -> torch Adam -> proj -> Polyak update -> update_weights, against the
    same step driven by the oracle's gradients."""
    from icnn_b200 import adam
    from icnn_b200.gd_grad import proj
    from icnn_b200.td_grad import td_grad
    B, lr, tau = 256, 1e-3, 0.01
    p, pt = tg.make_net("c4", 7), tg.make_net("c4", 8)
    obs, act, rew, ob2, _act2, term = tg.make_rows(p, pt, B, 4000)
    net, tnet = _nets(p, pt)
    act2 = tg._f32(adam.solve(tnet.bind(ob2)))
    keys = tg.PARAMS
    params = lambda nt: [(k, i, t) for k in keys for i, t in enumerate(getattr(nt, k)) if t is not None]  # noqa: E731
    pre = {(k, i): t.clone() for k, i, t in params(net)}
    _loss, _td, dev = td_grad(net.bind(obs), tnet.bind(ob2), obs, act, rew, act2, term, return_device=True)
    _oloss, _otd, orc = tg.td_grad(p, pt, obs, act, rew, ob2, act2, term)

    # the oracle arm: the same pre-step tensors, the oracle's gradients, the same optimiser
    ref = {key: t.clone() for key, t in pre.items()}
    for k, i, t in params(net):
        t.grad = dev[k][i].reshape(t.shape)
        ref[(k, i)].grad = torch.as_tensor(orc[k][i], dtype=torch.float32, device=t.device).reshape(t.shape)
    for ts in ([t for _, _, t in params(net)], list(ref.values())):
        opt = torch.optim.Adam(ts, lr=lr)
        opt.step()
    proj(net.Wz)
    proj([ref[("Wz", i)] for i in range(1, net.L + 1)])
    for k, i, tt in params(tnet):        # Polyak update with the pre-step theta (the values loss_q was evaluated at)
        tt.sub_(tau * (tt - pre[(k, i)]))
    net.update_weights()
    tnet.update_weights()
    net.bind(obs), tnet.bind(ob2)        # both handles accept the re-packed weights
    for k, i, t in params(net):
        g = np.abs(np.asarray(orc[k][i], dtype=np.float64)).reshape(tuple(t.shape))
        d = np.abs(t.cpu().numpy().astype(np.float64) - ref[(k, i)].detach().cpu().numpy())
        firm = g > RTOL * g.max()       # where Adam's first step lr * g / |g| cannot change sign on float32 noise
        assert d[firm].max(initial=0.0) <= 1e-5 * max(1.0, float(np.abs(t.cpu().numpy()).max())), (k, i)
        assert d.max() <= 2 * lr * (1 + 1e-3), (k, i)
    for k, i, tt in params(tnet):
        exp = (1 - tau) * np.asarray(getattr(pt, k)[i], dtype=np.float64) + tau * pre[(k, i)].cpu().numpy()
        assert np.abs(tt.cpu().numpy() - exp).max() <= 1e-6 * max(1.0, np.abs(exp).max()), (k, i)
