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
from .conv_picnn import BoundConvPICNN, _gate_vjp, _train_grad_buffers, _ypath_grads, conv_gd_trainable, conv_trainable
from .picnn import BoundPICNN


def _f32(a, dev):
    if isinstance(a, torch.Tensor):
        return a.to(device=dev, dtype=torch.float32).contiguous()
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device=dev)


def _host(v):
    """Tensors, also inside lists and dicts, as numpy arrays (None stays None)."""
    if isinstance(v, dict):
        return {k: _host(t) for k, t in v.items()}
    if isinstance(v, list):
        return [_host(t) for t in v]
    return None if v is None else v.cpu().numpy()


def _check_fg(fg, who, x=None, conv=True):
    """Refuses an ``fg`` the training gradient ``who`` does not take: anything but a ``BoundPICNN`` without the
    affine RL wrapper or, with ``conv``, a ``BoundConvPICNN``.  Returns True for the latter, whose x-path uses the
    minibatch it was bound to (so ``x`` is refused)."""
    if conv and isinstance(fg, BoundConvPICNN):
        if x is not None:
            raise ValueError("%s: a BoundConvPICNN uses the minibatch it was bound to; do not pass x" % who)
        return True
    if not isinstance(fg, BoundPICNN):
        raise TypeError("%s needs a BoundPICNN (PICNN.bind(x))%s"
                        % (who, " or a BoundConvPICNN (ConvPICNN.bind(x))" if conv else ""))
    if fg.affine:
        raise ValueError("%s: the affine RL wrapper is not part of this training graph; bind without affine=True" % who)
    return False


def _check_shape(who, shape, **tensors):
    """ValueError unless every one of the named ``tensors`` has ``shape``."""
    if any(tuple(t.shape) != shape for t in tensors.values()):
        raise ValueError("%s: %s must be %s, got %s" % (who, " and ".join(tensors), list(shape),
                                                       " and ".join(str(tuple(t.shape)) for t in tensors.values())))


def _grad_buffers(fg, dd=False):
    """Output buffers of an FC training gradient for ``fg``'s batch: per-layer lists 'Wy', 'Wz', 'dcy', 'dcz' (and
    'dd' with ``dd``), the host pointer arrays, and the C struct over them (``TrainGrads`` with ``dd``, else
    ``GdGrads``).  The arrays must outlive the work."""
    net, dev, B = fg.net, fg.net.device, fg.B
    n, L, hid = net.n, net.L, net.hidden
    width = lambda l: hid[l] if l < L else 1          # noqa: E731
    prev = lambda l: hid[l - 1]                        # noqa: E731
    z = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)  # noqa: E731
    grads = dict(Wy=[z(n, width(l)) for l in range(L + 1)], Wz=[None] + [z(prev(l), width(l)) for l in range(1, L + 1)],
                 dcy=[z(B, n) for _ in range(L + 1)], dcz=[None] + [z(B, prev(l)) for l in range(1, L + 1)])
    if dd:
        grads["dd"] = [z(B, width(l)) for l in range(L + 1)]
    arrs = [_capi.ptr_array(v) for v in grads.values()]
    gr = (_capi.TrainGrads if dd else _capi.GdGrads)(*[C.cast(a, _capi._fpp) for a in arrs])
    return grads, arrs, gr


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
    conv = _check_fg(fg, "gd_grad", x)
    net, dev, B, n = fg.net, fg.net.device, fg.B, fg.net.n
    with torch.cuda.device(dev):
        y0d, tY = _f32(y0, dev), _f32(trueY, dev)
        _check_shape("gd_grad", (B, n), y0=y0d, trueY=tY)
        if loss_scale is None:
            loss_scale = 2.0 / (B * n)
        if conv:
            o, gr, arrs = _train_grad_buffers(fg)
            entry, ws_bytes = _capi.lib.icnn_conv_gd_backward, _capi.lib.icnn_conv_gd_backward_workspace_bytes
        else:
            grads, arrs, gr = _grad_buffers(fg)
            entry, ws_bytes = _capi.lib.icnn_gd_backward, _capi.lib.icnn_gd_backward_workspace_bytes
        yN = torch.empty(B, n, dtype=torch.float32, device=dev)
        ws = _capi.workspace(ws_bytes(net._h, B, int(nIter)), dev)
        _capi.check(entry(net._h, C.byref(fg.c_gates), y0d.data_ptr(), tY.data_ptr(), float(loss_scale), int(nIter),
                          float(lr), float(momentum), yN.data_ptr(), C.byref(gr), ws.data_ptr(), _capi.stream()))
        if conv:
            grads = _ypath_grads(net, o)
            # x-path through the gates of the bound minibatch, over the same variables as the bundle-entropy mode (so
            # that the two give the same bits on the same rows); dd is zero, and the output layer's additive gate,
            # which only dd reaches, is then dropped
            names = [k for k in conv_trainable(net) if k not in grads]
            grads.update(_gate_vjp(fg, names, o["dcy"], o["dcz"], o["dd"]))
            grads = {k: grads[k] for k in conv_gd_trainable(net)}
            grads.update(dcy=o["dcy"], dcz=o["dcz"])
        elif x is not None:
            grads.update(_xpath_backward(net, _f32(x, dev), grads["dcy"], grads["dcz"]))
        torch.cuda.current_stream().synchronize()      # ws / arrs stay alive until the work is done
    if return_device:
        return yN, grads
    return _host(yN), _host(grads)


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
