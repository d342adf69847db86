"""The training gradient of the bundle-entropy method on the device (SURVEY.md section 8f row 1, the step after K3).

The reference's training step (multi-label-cls/icnn_ebundle.py:225-245) solves y* with ``solveBatch``,
differentiates it through the bundle's KKT system (``crossEntrGrad`` / ``mseGrad``), turns the result into one
``train_step_fd`` row per (sample, bundle point) -- x, y = ys_i, v, c (:296-314) -- and runs Adam on
``opt.compute_gradients(F_, theta_)`` (:153-156) of the surrogate

    F_ = c E(x, y) + sum_j v_j dE/dy_j                                        (:148)

summed over the rows.  ``train_grad`` computes that gradient from the feeds (``icnn_train_grad``, hand-written CUDA
in icnn_b200/csrc/train_grad.cu); ``bundle_grad`` runs the whole chain on the bundle state a
``solveBatch(..., return_state=True)`` left on the device: K3 (``argmin_grad``), the gather of the feed rows, and
the gradient, with no host round trip of the rows.

The y-path gradients (Wy, Wz) and the per-sample gate adjoints (dcy, dcz, dd) come from the library; the x-path
parameters follow from the gate adjoints by dense-layer backprop (``gd_grad._xpath_backward``).  Unlike the GD
training mode, the additive gates d_l enter through c E, so Wzx / bzx get a gradient too.

Parameter gradients are with respect to the handle's parameters, i.e. after an inference-mode batch-norm has been
folded into the x-path weights (``PICNN.from_params``), as in ``gd_grad``.  Training-mode batch-norm is out of scope
(DESIGN.md section 8).

Both functions also take the convolutional PICNN of the image-completion experiment (``ConvPICNN.bind(x)``), whose
training step is compute_gradients(F_, theta_) of completion/icnn_ebundle.py:129-140: the y-path gradients and
gate adjoints come from ``icnn_conv_train_grad`` (icnn_b200/csrc/conv_train_grad.cu), the x-path ones from torch
autograd through a grad-enabled recompute of ``ConvPICNN.gates`` on the bound minibatch (TF32 off).  The result is
keyed by TensorFlow variable name with exactly the variables the reference's ``gv_`` holds, each in its own shape,
so with ``return_device=True`` ``net.vars[k].grad = g`` works directly (then the optimiser step, ``proj``, and
``net.update_weights()``).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _capi
from .argmin_grad import LOSS, argmin_grad
from .gd_grad import _f32, _xpath_backward
from .conv_picnn import BoundConvPICNN, _gate_vjp, _to_host, _train_grad_buffers, _ypath_grads, conv_trainable
from .picnn import BoundPICNN

# parameter names of the returned dictionary with x given (the PICNN attribute names)
PARAMS = ("Wy", "Wz", "Wu", "bu", "Wzu", "bzu", "Wyu", "byu", "Wzx", "bzx")


def _check_fg(fg, who):
    if isinstance(fg, BoundConvPICNN):
        return
    if not isinstance(fg, BoundPICNN):
        raise TypeError("%s needs a BoundPICNN (PICNN.bind(x)) or a BoundConvPICNN (ConvPICNN.bind(x))" % who)
    if fg.affine:
        raise ValueError("%s: the affine RL wrapper has no bundle training step (RL/src/icnn.py:84)" % who)


def _check_conv_x(fg, x, who):
    """True for a conv fg (whose x-path uses the minibatch it was bound to: ``x`` is refused)."""
    if not isinstance(fg, BoundConvPICNN):
        return False
    if x is not None:
        raise ValueError("%s: a BoundConvPICNN uses the minibatch it was bound to; do not pass x" % who)
    return True


def _grad_buffers(fg):
    """Output buffers of the icnn_train_grads layout for ``fg``'s batch, the host pointer arrays and the C struct."""
    net, dev, B = fg.net, fg.net.device, fg.B
    n, L, hid = net.n, net.L, net.hidden
    width = lambda l: hid[l] if l < L else 1          # noqa: E731
    prev = lambda l: hid[l - 1]                        # noqa: E731
    z = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)  # noqa: E731
    grads = dict(Wy=[z(n, width(l)) for l in range(L + 1)], Wz=[None] + [z(prev(l), width(l)) for l in range(1, L + 1)],
                 dcy=[z(B, n) for _ in range(L + 1)], dcz=[None] + [z(B, prev(l)) for l in range(1, L + 1)],
                 dd=[z(B, width(l)) for l in range(L + 1)])
    arrs = [_capi.ptr_array(grads[k]) for k in ("Wy", "Wz", "dcy", "dcz", "dd")]
    gr = _capi.TrainGrads(*[C.cast(a, _capi._fpp) for a in arrs])
    return grads, arrs, gr


def _prepare(fg, offsets):
    """Output buffers, the C structs and the workspace of one icnn_train_grad call for the CSR ``offsets``."""
    net, dev, B = fg.net, fg.net.device, fg.B
    R = int(offsets[-1])
    grads, arrs, gr = _grad_buffers(fg)
    off = (C.c_int64 * (B + 1))(*[int(o) for o in offsets])
    ws = torch.empty(max(_capi.lib.icnn_train_grad_workspace_bytes(net._h, B, R), 4), dtype=torch.uint8, device=dev)
    return dict(grads=grads, arrs=arrs, gr=gr, off=off, ws=ws)


def _launch(fg, prep, Y, V, c):
    """icnn_train_grad on the current stream (asynchronous; ``prep`` and the inputs must outlive the work)."""
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _capi.check(_capi.lib.icnn_train_grad(fg.net._h, C.byref(fg.c_gates), prep["off"], Y.data_ptr(), V.data_ptr(),
                                          c.data_ptr(), C.byref(prep["gr"]), prep["ws"].data_ptr(), stream))


def _run(fg, Y, V, c, offsets, x, return_device):
    prep = _prepare(fg, offsets)
    _launch(fg, prep, Y, V, c)
    grads = dict(prep["grads"])
    if x is not None:
        grads.update(_xpath_backward(fg.net, _f32(x, fg.net.device), grads["dcy"], grads["dcz"], grads["dd"]))
    torch.cuda.current_stream().synchronize()      # ws / arrs / the inputs stay alive until the work is done
    if return_device:
        return grads
    host = lambda v: None if v is None else v.cpu().numpy()   # noqa: E731
    return {k: [host(t) for t in v] for k, v in grads.items()}


def _conv_launch(fg, Y, V, c, offsets):
    """icnn_conv_train_grad on the current stream (asynchronous): the output buffers, and what must outlive the work
    under 'keep'."""
    net, dev, B = fg.net, fg.net.device, fg.B
    R = int(offsets[-1])
    o, gr, arrs = _train_grad_buffers(fg)
    off = (C.c_int64 * (B + 1))(*[int(o_) for o_ in offsets])
    ws = torch.empty(max(_capi.lib.icnn_conv_train_grad_workspace_bytes(net._h, B, R), 4), dtype=torch.uint8,
                     device=dev)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _capi.check(_capi.lib.icnn_conv_train_grad(net._h, C.byref(fg.c_gates), off, Y.data_ptr(), V.data_ptr(),
                                               c.data_ptr(), C.byref(gr), ws.data_ptr(), stream))
    return dict(o, keep=(arrs, gr, off, ws))


def _conv_run(fg, Y, V, c, offsets, return_device):
    net = fg.net
    o = _conv_launch(fg, Y, V, c, offsets)
    grads = _ypath_grads(net, o)
    # x-path: d(sum of gate o gate adjoint)/d theta through the gates of the bound minibatch
    names = [k for k in conv_trainable(net) if k not in grads]
    grads.update(_gate_vjp(fg, names, o["dcy"], o["dcz"], o["dd"]))
    grads = {k: grads[k] for k in conv_trainable(net)}
    grads.update(dcy=o["dcy"], dcz=o["dcz"], dd=o["dd"])
    torch.cuda.current_stream().synchronize()      # ws / arrs / the inputs stay alive until the work is done
    return grads if return_device else _to_host(grads)


def train_grad(fg: BoundPICNN, Y, V, c, counts, x=None, return_device=False):
    """d (sum over the rows of F_) / d theta from the ``train_step_fd`` feeds.

    ``Y`` [R, n] (the bundle points ys_i), ``V`` [R, n], ``c`` [R]: one row per (sample, bundle point), samples in
    order; ``counts`` [B] = rows of each sample (sample u owns the next counts[u] rows and sees row u of the gates
    ``fg`` was bound to).  The rows are used in float32, as the reference's placeholders hold them (:129-131).

    Returns the ``gd_grad`` dictionary layout: 'Wy', 'Wz' (per-layer lists, summed over all rows), the per-sample
    gate adjoints 'dcy', 'dcz', 'dd' ([B, .], summed over each sample's rows), and with ``x`` (the minibatch the
    gates were bound to) also 'Wu', 'bu', 'Wzu', 'bzu', 'Wyu', 'byu', 'Wzx', 'bzx'.  Gradients are with respect to
    the handle's (batch-norm-folded) parameters.  Numpy arrays unless ``return_device``.

    For a ``BoundConvPICNN``: {TF variable name: gradient in the variable's shape} over ``conv_trainable(net)``
    (the x-path from the minibatch ``fg`` was bound to; ``x`` is refused), plus 'dcy' (per conv layer), 'dcz' and
    'dd' (per layer, [B, flat gate]); numpy arrays, or with ``return_device=True`` torch tensors on the net's device
    (for ``net.vars[k].grad = g``)."""
    _check_fg(fg, "train_grad")
    conv = _check_conv_x(fg, x, "train_grad")
    net, dev, B = fg.net, fg.net.device, fg.B
    counts = np.asarray(counts.cpu() if isinstance(counts, torch.Tensor) else counts, dtype=np.int64).reshape(-1)
    if counts.shape != (B,) or (counts < 0).any():
        raise ValueError("train_grad: counts must be %d non-negative row counts" % B)
    offsets = np.concatenate([[0], np.cumsum(counts)])
    R = int(offsets[-1])
    with torch.cuda.device(dev):
        Yd, Vd, cd = _f32(Y, dev).reshape(-1, net.n), _f32(V, dev).reshape(-1, net.n), _f32(c, dev).reshape(-1)
        if Yd.shape[0] != R or Vd.shape[0] != R or cd.shape[0] != R:
            raise ValueError("train_grad: Y, V and c must have sum(counts) = %d rows" % R)
        if conv:
            return _conv_run(fg, Yd, Vd, cd, offsets, return_device)
        return _run(fg, Yd, Vd, cd, offsets, x, return_device)


def bundle_grad(fg: BoundPICNN, state, trueY, loss="xent", x=None, return_device=False):
    """The reference's training gradient from a solve's device state: ``argmin_grad`` (K3, crossEntrGrad /
    mseGrad) -> the ``train_step_fd`` rows y = ys[u, i], v = V[u, i], c = clam[u, i] gathered on the device ->
    ``train_grad``.  ``state`` is the ``BundleState`` of ``solveBatch(fg, ..., return_state=True)`` (solved with
    ``keep_xs=True``, the default); ``trueY`` [B, n] the labels; ``loss`` 'xent' or 'mse'.  Same return layout as
    ``train_grad``."""
    _check_fg(fg, "bundle_grad")
    conv = _check_conv_x(fg, x, "bundle_grad")
    if loss not in LOSS:
        raise ValueError("loss must be 'mse' or 'xent'")
    if state.B != fg.B or state.n != fg.net.n:
        raise ValueError("bundle_grad: state is for B=%d, n=%d, fg for B=%d, n=%d" % (state.B, state.n, fg.B, fg.net.n))
    if state.ys is None:
        raise ValueError("bundle_grad: the state was solved with keep_xs=False (no bundle points to train on)")
    dev = fg.net.device
    with torch.cuda.device(dev):
        _cy, clam, _ct, V = argmin_grad(state, trueY, loss=loss, assemble=True, return_device=True)
        counts = state.count.cpu().numpy().astype(np.int64)
        offsets = np.concatenate([[0], np.cumsum(counts)])
        R = int(offsets[-1])
        cnt = torch.as_tensor(counts, device=dev)
        iu = torch.repeat_interleave(torch.arange(state.B, device=dev), cnt, output_size=R)
        ii = torch.arange(R, device=dev) - torch.as_tensor(offsets[:-1], device=dev)[iu]
        slots = state.perm.long()[iu, ii]
        Y = state.ys[iu, slots].float()
        Vr = V[iu, ii].float()
        c = clam[iu, ii].float()
        if conv:
            return _conv_run(fg, Y.contiguous(), Vr.contiguous(), c.contiguous(), offsets, return_device)
        return _run(fg, Y.contiguous(), Vr.contiguous(), c.contiguous(), offsets, x, return_device)
