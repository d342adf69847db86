"""d loss / d theta through the unrolled momentum-GD inner loop (the ``icnn.back`` training mode).

Reference: the graph of multi-label-cls/icnn-back.py:116-139 (= completion/icnn.back.py:133-156)
unrolls nIter momentum-GD steps on the energy, puts ``mse_ = reduce_mean(square(yn - trueY))`` on the
output and lets ``opt.compute_gradients(self.mse_, self.theta_)`` double-backprop through it.
``gd_grad`` returns the same gradients: the y-path ones (Wy, Wz) and the per-sample gate adjoints
(dcy, dcz) come from ``icnn_gd_backward`` (hand-written CUDA, icnn_b200/csrc/gd_backward.cu); the
x-path parameters (Wu/bu, Wzu/bzu, Wyu/byu) follow from the gate adjoints by ordinary dense-layer
backprop, a handful of library GEMMs outside the hot loop.  The additive gate d_l does not enter
dE/dy, so Wzx/bzx get no gradient (TF returns None for them, filtered at icnn-back.py:137-138).

``gd_grad`` also takes the convolutional PICNN of the image-completion experiment (``ConvPICNN.bind(x)``), whose
back-optimisation mode (completion/icnn.back.py:121-156) unrolls the same loop on the conv energy.  The y-path
gradients and the gate adjoints come from ``icnn_conv_gd_backward`` (icnn_b200/csrc/conv_train_grad.cu: the loop, then
the conv training gradient on one row per (sample, step)), the x-path ones from torch autograd through a
grad-enabled recompute of the gates of the bound minibatch (TF32 off), as for ``bundle_grad``.

``makeCvx`` / ``proj`` (icnn-back.py:141-144) -- the projection of the 'proj' weights Wz onto the
non-negative orthant applied after every optimiser step -- are ``make_cvx`` / ``proj`` below.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _capi
from .conv_picnn import (BoundConvPICNN, _gate_vjp, _to_host, _train_grad_buffers, _ypath_grads, conv_gd_trainable,
                         conv_trainable)
from .picnn import BoundPICNN


def _f32(a, dev):
    if isinstance(a, torch.Tensor):
        return a.to(device=dev, dtype=torch.float32).contiguous()
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device=dev)


def gd_grad(fg: BoundPICNN, y0, trueY, nIter=30, lr=0.01, momentum=0.3, loss_scale=None, x=None,
            return_device=False):
    """Returns ``(yN, grads)``; ``grads`` maps parameter names (the PICNN attribute names: 'Wy', 'Wz',
    and with ``x`` given also 'Wu', 'bu', 'Wzu', 'bzu', 'Wyu', 'byu') to per-layer lists, plus the
    gate adjoints 'dcy', 'dcz'.  ``loss_scale`` defaults to 2/(B n), i.e. the multi-label script's
    ``reduce_mean(square(yn - trueY))``; completion/icnn.back.py:150 is ``2 * 255**2 / (B n)``.
    ``x`` [B, m] is the minibatch the gates were bound to (needed only for the x-path gradients).

    For a ``BoundConvPICNN`` (completion/icnn.back.py:121-156; its values are lr = 0.01, momentum = 0.9 (:133-134),
    nIter = 30 (--nGdIter) and loss_scale = 2 * 255**2 / (B n) for ``reduce_mean(square(255 (yn - trueY)))``):
    ``grads`` maps the TF variable names of ``conv_gd_trainable(net)`` -- exactly the reference's gv_ -- to gradients
    in the variables' shapes, with the x-path from the minibatch ``fg`` was bound to (``x`` is refused), plus the gate
    adjoints 'dcy' (per conv layer) and 'dcz' (per layer, [B, flat gate]).  The additive gates 'z{l}_u/*' and the
    y_red biases 'z{l}_y_red/b' are in gv_ with a gradient that is exactly zero, and are returned as zeros.  Numpy
    arrays, or with ``return_device=True`` torch tensors on the net's device (for ``net.vars[k].grad = g``)."""
    if isinstance(fg, BoundConvPICNN):
        if x is not None:
            raise ValueError("gd_grad: a BoundConvPICNN uses the minibatch it was bound to; do not pass x")
        return _conv_gd_grad(fg, y0, trueY, nIter, lr, momentum, loss_scale, return_device)
    if not isinstance(fg, BoundPICNN):
        raise TypeError("gd_grad needs a BoundPICNN (PICNN.bind(x)) or a BoundConvPICNN (ConvPICNN.bind(x))")
    if fg.affine:
        raise ValueError("gd_grad: the affine RL wrapper is not part of the icnn.back training graph")
    net, dev, B = fg.net, fg.net.device, fg.B
    n, L, hid = net.n, net.L, net.hidden
    width = lambda l: hid[l] if l < L else 1          # noqa: E731
    prev = lambda l: hid[l - 1]                        # noqa: E731
    with torch.cuda.device(dev):
        y0d, tY = _f32(y0, dev), _f32(trueY, dev)
        assert tuple(y0d.shape) == (B, n) and tuple(tY.shape) == (B, n)
        if loss_scale is None:
            loss_scale = 2.0 / (B * n)
        z = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)  # noqa: E731
        dWy = [z(n, width(l)) for l in range(L + 1)]
        dcy = [z(B, n) for _ in range(L + 1)]
        dWz = [None] + [z(prev(l), width(l)) for l in range(1, L + 1)]
        dcz = [None] + [z(B, prev(l)) for l in range(1, L + 1)]
        yN = z(B, n)
        arrs = [_capi.ptr_array(v) for v in (dWy, dWz, dcy, dcz)]
        gr = _capi.GdGrads(*[C.cast(a, _capi._fpp) for a in arrs])
        ws = torch.empty(max(_capi.lib.icnn_gd_backward_workspace_bytes(net._h, B, int(nIter)), 4), dtype=torch.uint8,
                         device=dev)
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        _capi.check(_capi.lib.icnn_gd_backward(net._h, C.byref(fg.c_gates), y0d.data_ptr(), tY.data_ptr(),
                                               float(loss_scale), int(nIter), float(lr), float(momentum),
                                               yN.data_ptr(), C.byref(gr), ws.data_ptr(), stream))
        grads = dict(Wy=dWy, Wz=dWz, dcy=dcy, dcz=dcz)
        if x is not None:
            grads.update(_xpath_backward(net, _f32(x, dev), dcy, dcz))
        torch.cuda.current_stream().synchronize()      # ws / arrs stay alive until the work is done
    if return_device:
        return yN, grads
    host = lambda v: None if v is None else v.cpu().numpy()   # noqa: E731
    return host(yN), {k: [host(t) for t in v] for k, v in grads.items()}


def _conv_gd_grad(fg, y0, trueY, nIter, lr, momentum, loss_scale, return_device):
    net, dev, B, n = fg.net, fg.net.device, fg.B, fg.net.n
    with torch.cuda.device(dev):
        y0d, tY = _f32(y0, dev), _f32(trueY, dev)
        if tuple(y0d.shape) != (B, n) or tuple(tY.shape) != (B, n):
            raise ValueError("gd_grad: y0 and trueY must be [%d, %d], got %s and %s"
                             % (B, n, tuple(y0d.shape), tuple(tY.shape)))
        if loss_scale is None:
            loss_scale = 2.0 / (B * n)
        o, gr, arrs = _train_grad_buffers(fg)
        yN = torch.empty(B, n, dtype=torch.float32, device=dev)
        ws = torch.empty(max(_capi.lib.icnn_conv_gd_backward_workspace_bytes(net._h, B, int(nIter)), 4),
                         dtype=torch.uint8, device=dev)
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        _capi.check(_capi.lib.icnn_conv_gd_backward(net._h, C.byref(fg.c_gates), y0d.data_ptr(), tY.data_ptr(),
                                                    float(loss_scale), int(nIter), float(lr), float(momentum),
                                                    yN.data_ptr(), C.byref(gr), ws.data_ptr(), stream))
        grads = _ypath_grads(net, o)
        # x-path through the gates of the bound minibatch, over the same variables as the bundle-entropy mode (so
        # that the two give the same bits on the same rows); dd is zero, and the output layer's additive gate,
        # which only dd reaches, is then dropped
        names = [k for k in conv_trainable(net) if k not in grads]
        grads.update(_gate_vjp(fg, names, o["dcy"], o["dcz"], o["dd"]))
        grads = {k: grads[k] for k in conv_gd_trainable(net)}
        grads.update(dcy=o["dcy"], dcz=o["dcz"])
        torch.cuda.current_stream().synchronize()      # ws / arrs stay alive until the work is done
    if return_device:
        return yN, grads
    return yN.cpu().numpy(), _to_host(grads)


def _xpath_backward(net, x, dcy, dcz, dd=None):
    """Dense-layer backprop of the gate adjoints into the x-path parameters
    (multi-label-cls/icnn-back.py:255-262 u path, :269-272 cz gate, :279-281 cy gate).  ``dd`` (the adjoints of
    the additive gates d_l = P_l Wzx_l + bzx_l, multi-label-cls/icnn_ebundle.py:372-373) adds 'Wzx' / 'bzx'; the GD-mode energy gradient has
    none, so by default they are left out."""
    L = net.L
    us, pres, p = [], [], x
    for i in range(L):
        pre = torch.addmm(net.bu[i], p, net.Wu[i])
        u = torch.relu(pre) if i < L - 1 else pre
        pres.append(pre); us.append(u); p = u
    out = dict(Wu=[None] * L, bu=[None] * L, Wzu=[None] * (L + 1), bzu=[None] * (L + 1),
               Wyu=[None] * (L + 1), byu=[None] * (L + 1))
    if dd is not None:
        out.update(Wzx=[None] * (L + 1), bzx=[None] * (L + 1))
    dU = [torch.zeros_like(u) for u in us]
    for i in range(L, -1, -1):
        P = x if i == 0 else us[i - 1]
        out["Wyu"][i] = P.t() @ dcy[i]
        out["byu"][i] = dcy[i].sum(0)
        dP = dcy[i] @ net.Wyu[i].t()
        if dd is not None:
            out["Wzx"][i] = P.t() @ dd[i]
            out["bzx"][i] = dd[i].sum(0)
            dP = dP + dd[i] @ net.Wzx[i].t()
        if i > 0:
            pz = dcz[i] * (torch.addmm(net.bzu[i], P, net.Wzu[i]) > 0)
            out["Wzu"][i] = P.t() @ pz
            out["bzu"][i] = pz.sum(0)
            dU[i - 1] += dP + pz @ net.Wzu[i].t()
    for i in range(L - 1, -1, -1):
        du = dU[i] * (pres[i] > 0) if i < L - 1 else dU[i]
        P = x if i == 0 else us[i - 1]
        out["Wu"][i] = P.t() @ du
        out["bu"][i] = du.sum(0)
        if i > 0:
            dU[i - 1] += du @ net.Wu[i].t()
    return out


def make_cvx(Wz, halve=False, divide=None):
    """``makeCvx``: W <- |W| (multi-label-cls/icnn-back.py:143), |W|/2 with ``halve``
    (completion/icnn.back.py:164, completion/icnn_ebundle.py:145), |W|/``divide`` in general
    (synthetic-cls/icnn.py:145 uses 10), for every 'proj' weight Wz[1..L]; in place on torch tensors.
    When applied to a PICNN's own tensors (``make_cvx(net.Wz)``) follow with ``net.update_weights()``: the
    device library works on packed copies, and ``net.bind`` refuses to run on stale ones."""
    for w in Wz:
        if w is not None:
            w.abs_()
            if halve:
                w.mul_(0.5)
            if divide is not None:
                w.div_(float(divide))
    return Wz


def proj(Wz):
    """``proj``: W <- max(W, 0) (multi-label-cls/icnn-back.py:144).  Same re-packing rule as ``make_cvx``."""
    for w in Wz:
        if w is not None:
            w.clamp_(min=0)
    return Wz
