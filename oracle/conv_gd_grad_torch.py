"""Float64 torch oracle of the conv-PICNN GD training gradient: d loss / d theta through nIter unrolled momentum-GD
steps on the completion energy (completion/icnn.back.py:133-156)

    v' = m v - lr dE/dy(x, y),  y' = y - m v + (1 + m) v',  v_0 = 0;   loss = loss_scale / 2 sum (y_N - trueY)^2

(loss_scale = 2 255^2 / (B n) is the script's mse_ = reduce_mean(square(255 (yn_ - trueY)))).

``gd_grad`` is the literal double backward: autograd through every step's dE/dy (create_graph=True) over every
trainable variable of the completion Model and the gate tensors.  ``kappa_form`` is the piecewise-linear reduction the
device relies on (icnn_b200/csrc/gd_backward.cu's header, icnn_conv_gd_backward): the conv training gradient
(oracle/conv_train_grad_torch.py) on one row per (sample u, step i) with Y = y_i[u], V = kappa_i a[u], c = 0.
tests/test_conv_gd_grad_cpu.py pins the two to each other, tests/test_conv_gd_grad_golden_cpu.py the literal one to
the reference's own graph (tests/golden/conv/conv_gd_grad.npz)."""
import numpy as np
import torch

from oracle import conv_train_grad_torch as T


def kappa(nIter, lr, momentum):
    """kappa_i, i < nIter: c_N = 1 + m, c_i = m c_{i+1} + 1, kappa_i = -lr c_{i+1}, in float64."""
    lr, m = float(lr), float(momentum)
    k, c = np.zeros(nIter), 1.0 + m
    for i in range(nIter - 1, -1, -1):
        k[i] = -lr * c
        c = m * c + 1.0
    return k


def _step(y, v, g, lr, m):
    vn = m * v - lr * g
    return y - m * v + (1.0 + m) * vn, vn


def gd_grad(spec, x, y0, trueY, nIter, lr=0.01, momentum=0.9, loss_scale=None, device="cpu", bn_eps=1e-5,
            dtype=torch.float64):
    """spec: icnn_b200.conv_picnn.parse_variables(...).  Returns (yN [B, n], loss, {name: gradient in the variable's
    shape} over the trainable variables with a gradient (autograd's None = TensorFlow's None, filtered as gv_ is),
    {'dcy': [Lc], 'dcz': [Lc + Ld]} per-sample gate adjoints, min relative |pre-activation| per sample over the nIter
    iterates the gradient is taken at)."""
    f64 = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64), device=device).to(dtype)   # noqa: E731
    Lc, Ld = len(spec.convs), len(spec.fcs)
    n = spec.H * spec.W
    names = T.trainable(list(spec.vars), Lc, Ld)
    V = {k: f64(v).requires_grad_(k in names) for k, v in spec.vars.items()}
    x = f64(x).reshape(-1, n)
    B = x.shape[0]
    if loss_scale is None:
        loss_scale = 2.0 / (B * n)
    lr, m = float(lr), float(momentum)
    cz, cy, d = T.gates(V, spec, x, bn_eps)
    G = [g for g in cz + cy if g is not None]
    y, v = f64(y0).reshape(B, n).requires_grad_(), 0.0
    rel = torch.full((B,), float("inf"), dtype=torch.float64, device=device)
    for _ in range(nIter):
        E, pres, _b = T.y_energy(V, spec, cz, cy, d, y)
        (g,) = torch.autograd.grad(E.sum(), y, create_graph=True)
        with torch.no_grad():
            for a in pres:
                aa = a.abs()
                rel = torch.minimum(rel, aa.min(1).values / aa.max(1).values.clamp_min(1e-300))
        y, v = _step(y, v, g, lr, m)
    loss = 0.5 * loss_scale * ((y - f64(trueY).reshape(B, n)) ** 2).sum()
    out = torch.autograd.grad(loss, [V[k] for k in names] + G, allow_unused=True) if nIter else [None] * (
        len(names) + len(G))
    grads = {k: g.detach().cpu().numpy() for k, g in zip(names, out[:len(names)]) if g is not None}
    it = iter(out[len(names):])

    def take(lst):
        res = []
        for gt in lst:
            t = None if gt is None else next(it)
            res.append(None if gt is None else (torch.zeros_like(gt) if t is None else t).detach().cpu().numpy())
        return res
    adj = dict(dcz=take(cz), dcy=take(cy)[:Lc])
    return y.detach().cpu().numpy(), float(loss.detach()), grads, adj, rel.cpu().numpy()


def trajectory(spec, x, y0, nIter, lr=0.01, momentum=0.9, device="cpu", bn_eps=1e-5):
    """The iterates y_0 .. y_N [N + 1, B, n] of the loop, float64."""
    n = spec.H * spec.W
    V = {k: torch.as_tensor(np.asarray(a, dtype=np.float64), device=device) for k, a in spec.vars.items()}
    x = torch.as_tensor(np.asarray(x, dtype=np.float64), device=device).reshape(-1, n)
    cz, cy, d = T.gates(V, spec, x, bn_eps)
    y, v, ys = torch.as_tensor(np.asarray(y0, dtype=np.float64), device=device).reshape(-1, n), 0.0, []
    for _ in range(nIter):
        ys.append(y)
        yr = y.detach().requires_grad_()
        E, _p, _b = T.y_energy(V, spec, cz, cy, d, yr)
        (g,) = torch.autograd.grad(E.sum(), yr)
        y, v = _step(y, v, g, float(lr), float(momentum))
    ys.append(y)
    return torch.stack(ys).cpu().numpy()


def kappa_form(spec, x, y0, trueY, nIter, lr=0.01, momentum=0.9, loss_scale=None, device="cpu", bn_eps=1e-5):
    """The same gradient as ``gd_grad`` from the rows Y = y_i[u], V = kappa_i a[u], c = 0 (sample-major) through
    oracle/conv_train_grad_torch.train_grad: ({name: gradient} over its trainable set, {'dcy', 'dcz', 'dd'}
    adjoints)."""
    n = spec.H * spec.W
    ys = trajectory(spec, x, y0, nIter, lr, momentum, device, bn_eps)
    B = ys.shape[1]
    if loss_scale is None:
        loss_scale = 2.0 / (B * n)
    a = loss_scale * (ys[-1] - np.asarray(trueY, dtype=np.float64).reshape(B, n))
    k = kappa(nIter, lr, momentum)
    Y = ys[:-1].transpose(1, 0, 2).reshape(B * nIter, n)
    Vr = (k[None, :, None] * a[:, None, :]).reshape(B * nIter, n)
    grads, adj, _rel, _bs = T.train_grad(spec, x, Y, Vr, np.zeros(B * nIter), np.full(B, nIter), device=device,
                                         bn_eps=bn_eps)
    return grads, adj
