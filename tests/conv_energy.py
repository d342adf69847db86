"""The completion ``Model.f`` (completion/icnn_ebundle.py:337-452) in plain torch, evaluated straight from the
reference's TensorFlow variable dict (kernels [k, k, c_in, c_out], NHWC flattening, inference batch-norm, biases).
TEST HELPER ONLY: the float32 arm that sets the accuracy yardstick of the device kernels, and a float64 oracle that
tests/test_conv_picnn_cpu.py pins to the goldens of the reference's own graph."""
import numpy as np
import torch

from icnn_b200.conv_picnn import _same_conv


def energy(spec, x, y, dtype=torch.float64, device="cpu", bn_eps=1e-5):
    """spec: icnn_b200.conv_picnn.parse_variables(...); x, y [B, H*W] -> E [B] (differentiable in y)."""
    V = {k: torch.as_tensor(np.asarray(v), dtype=dtype, device=device) for k, v in spec.vars.items()}
    H, W, Lc = spec.H, spec.W, len(spec.convs)
    x = torch.as_tensor(x, dtype=dtype, device=device).reshape(-1, 1, H, W)
    y = y.reshape(-1, 1, H, W)
    B = x.shape[0]
    flat = lambda t: t.permute(0, 2, 3, 1).reshape(B, -1) if t.dim() == 4 else t      # noqa: E731

    def bn(u, i):
        sh = (1, -1, 1, 1) if u.dim() == 4 else (1, -1)
        p = lambda nm: V["u%d/BatchNormalization/%s" % (i, nm)].reshape(sh)           # noqa: E731
        return (u - p("moving_mean")) / torch.sqrt(p("moving_variance") + bn_eps) * p("gamma") + p("beta")

    us, prev = [], x
    for i, (_c, _k, s) in enumerate(spec.convs):
        prev = bn(torch.relu(_same_conv(prev, V["u%d/W" % i], V["u%d/b" % i], s)), i)
        us.append(prev)
    for j, sz in enumerate(spec.fcs):
        i = Lc + j
        prev = flat(prev) @ V["u%d/W" % i] + V["u%d/b" % i]
        if sz != 1:
            prev = bn(torch.relu(prev), i)
        us.append(prev)
    prevU, prevZ, r = x, None, y
    for i, (_c, _k, s) in enumerate(spec.convs):
        z = _same_conv(r * _same_conv(prevU, V["z%d_yu_u/W" % i], V["z%d_yu_u/b" % i], 1), V["z%d_yu/W" % i], None, s)
        z = z + _same_conv(prevU, V["z%d_u/W" % i], V["z%d_u/b" % i], s)
        if i > 0:
            cz = torch.relu(_same_conv(prevU, V["z%d_zu_u/W" % i], V["z%d_zu_u/b" % i], 1))
            z = z + _same_conv(prevZ * cz, V["z%d_zu_proj/W" % i], None, s)
        r = _same_conv(r, V["z%d_y_red/W" % i], V["z%d_y_red/b" % i], s)
        prevZ, prevU = torch.relu(z), us[i]
    for j, sz in enumerate(spec.fcs):
        i = Lc + j
        P = flat(prevU)
        cz = torch.relu(P @ V["z%d_zu_u/W" % i] + V["z%d_zu_u/b" % i])
        z = (flat(prevZ) * cz) @ V["z%d_zu_proj/W" % i] + P @ V["z%d_u/W" % i] + V["z%d_u/b" % i]
        if sz != 1:
            z = torch.relu(z)
        prevU, prevZ = us[i], z
    return z.reshape(-1)


def fg(spec, x, y, dtype=torch.float64, device="cpu"):
    """(f [B], g [B, H*W]) as numpy float64."""
    yt = torch.as_tensor(np.asarray(y), dtype=dtype, device=device).requires_grad_()
    E = energy(spec, x, yt, dtype=dtype, device=device)
    (g,) = torch.autograd.grad(E.sum(), yt)
    return E.detach().cpu().double().numpy(), g.reshape(yt.shape[0], -1).cpu().double().numpy()
