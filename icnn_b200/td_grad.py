"""The RL agent's TD training gradient on the device (the training step after ``adam.solve``).

The reference's default agent (``--icnn_opt adam``, RL/src/agent.py:25) trains its Q network once per environment
step: ``Agent.train`` (RL/src/icnn.py:304-323) draws a minibatch (obs, act, rew, ob2, term2), solves
``act2 = Agent.adam(_fg_entr_target, ob2)`` on the target network (``icnn_b200.adam.solve``), and runs Adam on

    q_entr        = -(negQ(obs, act) - entropy(act))                                   (:59-62)
    q_target_entr = -(negQ_target(ob2, act2) - entropy(act2))                          (:69-75)
    y  = select(term2, rew, rew + discount q_target_entr), clamped to [q_entr - 1, q_entr + 1], stop_gradient
    td = q_entr - y,   loss_q = mean(td^2) + l2norm * sum of the L2 regularisation losses under 'q/'   (:78-93)

``td_grad`` returns loss_q, td and d loss_q / d theta of the online network.  The TD error and the y-path gradients
(Wy, Wz) with the per-sample gate adjoints (dcy, dcz, dd) come from ``icnn_td_grad`` (hand-written CUDA in
icnn_b200/csrc/td_grad.cu: one K1 forward at act, the TD kernel, the backward seeded with c = -2 td / B); the x-path
parameters follow from the gate adjoints by dense-layer backprop (``gd_grad._xpath_backward``, in float64: its sums run
over the whole minibatch).  The additive gates
``z{i}_u`` enter negQ, so Wzx / bzx get a gradient.  Every ``fully_connected`` of negQ carries tflearn's
``regularizer='L2'``, i.e. weight_decay * sum(W^2) / 2 on its weight matrix and not on its bias, so each weight
matrix gets l2norm * weight_decay * W on top.  The target network's variables get no gradient.

The optimiser step, ``proj`` (``gd_grad.proj``) and the Polyak update of the target network are left to torch; see
INTEGRATION.md, "Training step (the RL agent)".  Gradients are with respect to the handle's parameters: a PICNN built
by ``PICNN.from_params`` from parameters with an inference-mode batch-norm holds the folded x-path weights.
``--icnn_bn`` trains with batch statistics (RL/src/icnn.py:318), which is out of scope (DESIGN.md section 8).
"""
from __future__ import annotations

import ctypes as C
import types

import numpy as np
import torch

from . import _capi
from .bundle_grad import _grad_buffers
from .gd_grad import _f32, _xpath_backward
from .picnn import BoundPICNN

# agent.py:13-15 (discount, l2norm) and tflearn's fully_connected default weight_decay
DISCOUNT, L2NORM, WEIGHT_DECAY = 0.99, 1e-4, 1e-3
# the weight matrices of negQ (each one a fully_connected W); the biases carry no L2 loss
WEIGHTS = ("Wy", "Wz", "Wu", "Wzu", "Wyu", "Wzx")


def _check(fg, who):
    if not isinstance(fg, BoundPICNN):
        raise TypeError("td_grad: %s must be a BoundPICNN (PICNN.bind(obs))" % who)
    if fg.affine:
        raise ValueError("td_grad: bind %s without affine=True: the TD step sees the action in [-1, 1]" % who)


def _launch(fg, act, negq_t, act2, rew, term, discount):
    """icnn_td_grad on the current stream (asynchronous): (td, loss [1] float64, grads, what must outlive the work)."""
    net, dev, B = fg.net, fg.net.device, fg.B
    grads, arrs, gr = _grad_buffers(fg)
    td = torch.empty(B, dtype=torch.float32, device=dev)
    loss = torch.empty(1, dtype=torch.float64, device=dev)
    nbytes = _capi.lib.icnn_td_grad_workspace_bytes(net._h, B)
    if nbytes == 0:
        raise ValueError("td_grad: no workspace for B = %d (the library takes up to 65536 samples per call)" % B)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _capi.check(_capi.lib.icnn_td_grad(net._h, C.byref(fg.c_gates), act.data_ptr(), negq_t.data_ptr(), act2.data_ptr(),
                                       rew.data_ptr(), term.data_ptr(), float(discount), td.data_ptr(),
                                       loss.data_ptr(), C.byref(gr), ws.data_ptr(), stream))
    return td, loss, grads, (arrs, gr, ws)


def td_grad(fg: BoundPICNN, fg_target: BoundPICNN, obs, act, rew, act2, term, discount=DISCOUNT, l2norm=L2NORM,
            weight_decay=WEIGHT_DECAY, return_device=False):
    """Returns ``(loss_q, td, grads)`` of one minibatch of the RL agent's training step.

    ``fg = net.bind(obs)`` and ``fg_target = target_net.bind(ob2)`` (both without ``affine``); ``obs`` [B, m] is the
    minibatch ``fg`` was bound to (for the x-path gradients); ``act``, ``act2`` [B, n] (act2 from
    ``adam.solve(fg_target)``), ``rew`` [B], ``term`` [B] (bool).  The actions are used in float32, as the
    reference's placeholders hold them; negQ_target is K1's f of the target network at float32(act2), as TensorFlow
    re-evaluates it at the fed act2 (:320).

    ``grads`` maps 'Wy', 'Wz', 'Wu', 'bu', 'Wzu', 'bzu', 'Wyu', 'byu', 'Wzx', 'bzx' (the PICNN attribute names,
    per-layer lists like ``bundle_grad``) to d loss_q / d theta including the L2 term, and 'dcy', 'dcz', 'dd' to the
    per-sample gate adjoints of mean(td^2).  ``loss_q`` is a float and ``td`` [B] numpy; with ``return_device``
    ``loss_q`` is a 0-d float64 tensor and everything else torch tensors on the net's device."""
    _check(fg, "fg")
    _check(fg_target, "fg_target")
    net, dev, B, n = fg.net, fg.net.device, fg.B, fg.net.n
    if fg_target.B != B or fg_target.net.n != n or fg_target.net.device != dev:
        raise ValueError("td_grad: fg_target is for B=%d, n=%d on %s, fg for B=%d, n=%d on %s"
                         % (fg_target.B, fg_target.net.n, fg_target.net.device, B, n, dev))
    with torch.cuda.device(dev):
        actd, act2d, obsd = _f32(act, dev), _f32(act2, dev), _f32(obs, dev)
        rewd = _f32(rew, dev).reshape(-1)
        if isinstance(term, torch.Tensor):
            termd = term.to(device=dev, dtype=torch.bool).to(torch.uint8).reshape(-1).contiguous()
        else:
            termd = torch.as_tensor(np.asarray(term, dtype=bool).astype(np.uint8).reshape(-1), device=dev)
        if tuple(actd.shape) != (B, n) or tuple(act2d.shape) != (B, n):
            raise ValueError("td_grad: act and act2 must be [%d, %d], got %s and %s"
                             % (B, n, tuple(actd.shape), tuple(act2d.shape)))
        if tuple(obsd.shape) != (B, net.m):
            raise ValueError("td_grad: obs must be the [%d, %d] minibatch fg was bound to, got %s"
                             % (B, net.m, tuple(obsd.shape)))
        if rewd.shape[0] != B or termd.shape[0] != B:
            raise ValueError("td_grad: rew and term must have %d entries" % B)
        negq_t, _ = fg_target.fg_device(act2d)
        td, loss, grads, keep = _launch(fg, actd, negq_t, act2d, rewd, termd, discount)
        grads = dict(grads)
        # the x-path sums run over the whole minibatch (65536 samples at C4) with terms of both signs: float64
        d64 = lambda ts: [None if t is None else t.double() for t in ts]   # noqa: E731
        net64 = types.SimpleNamespace(L=net.L, **{k: d64(getattr(net, k)) for k in ("Wu", "bu", "Wzu", "bzu", "Wyu",
                                                                                    "byu", "Wzx", "bzx")})
        xg = _xpath_backward(net64, obsd.double(), d64(grads["dcy"]), d64(grads["dcz"]), d64(grads["dd"]))
        grads.update({k: [None if t is None else t.float() for t in v] for k, v in xg.items()})
        lam = float(l2norm) * float(weight_decay)
        reg = torch.zeros((), dtype=torch.float64, device=dev)
        for k in WEIGHTS:
            for i, w in enumerate(getattr(net, k)):
                if w is not None:
                    grads[k][i] = grads[k][i] + lam * w
                    reg = reg + 0.5 * w.double().square().sum()
        loss_q = loss[0] + lam * reg
        torch.cuda.current_stream().synchronize()      # ws / arrs / the inputs stay alive until the work is done
        del keep
    if return_device:
        return loss_q, td, grads
    host = lambda v: None if v is None else v.cpu().numpy()   # noqa: E731
    return float(loss_q), td.cpu().numpy(), {k: [host(t) for t in v] for k, v in grads.items()}
