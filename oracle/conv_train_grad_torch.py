"""Float64 torch oracle of the conv-PICNN training gradient: d (sum_r F_r) / d theta with
F_r = c_r E(x_u, Y_r) + V_r . dE/dy(x_u, Y_r) (completion/icnn_ebundle.py:129-130, summed over the train_step_fd rows
of :315-335), by autograd through dE/dy (create_graph=True) over every trainable variable of the completion Model,
plus the per-sample adjoints of the gates (cy, cz, d in the layouts of include/icnn_b200.h).

The energy is restated from the reference's Model.f (completion/icnn_ebundle.py:337-452) on a dict of tensors, split
into the x-path (per sample: the gates) and the y-path (per row, given its sample's gates), so that the gate
adjoints are gradients with respect to the gate tensors themselves.  tests/test_conv_train_grad_golden_cpu.py pins
its gradient and variable set to the reference's own training step (tests/golden/conv/conv_train_grad.npz);
tests/test_conv_train_grad_cpu.py pins its energy to tests/conv_energy.energy and its gradient to central finite
differences."""
import numpy as np
import torch

from icnn_b200.conv_picnn import _same_conv

BN_STATS = ("moving_mean", "moving_variance")


def trainable(names, Lc, Ld):
    """The variables the reference's gv_ holds (compute_gradients filtered by ``g is not None``): every trainable
    variable but the last u-layer (nothing consumes it) and the last conv layer's y_red (r_Lc is never used)."""
    last_u, last_red = "u%d/" % (Lc + Ld - 1), "z%d_y_red/" % (Lc - 1)
    return [k for k in names if not k.endswith(BN_STATS) and not k.startswith((last_u, last_red))]


def make_variables(H, W, convs, fcs, seed=0, bn=True):
    """Random variables of the completion Model in TensorFlow names and layouts (conv kernels [k, k, c_in, c_out],
    dense [in, out] on the NHWC-flattened map), scaled like tests/conv_picnn.py; with ``bn`` non-identity
    inference batch-norm statistics and affine parameters."""
    rs = np.random.RandomState(seed)
    rnd = lambda *s, fan: rs.randn(*s) / np.sqrt(fan)          # noqa: E731
    v = {}
    Lc = len(convs)

    def bn_vars(i, wd):
        if bn:
            v["u%d/BatchNormalization/gamma" % i] = rs.uniform(0.5, 1.5, wd)
            v["u%d/BatchNormalization/beta" % i] = rs.uniform(-0.2, 0.2, wd)
            v["u%d/BatchNormalization/moving_mean" % i] = rs.uniform(-0.1, 0.3, wd)
            v["u%d/BatchNormalization/moving_variance" % i] = rs.uniform(0.5, 2.0, wd)
        else:
            for nm, a in (("gamma", 1.0), ("beta", 0.0), ("moving_mean", 0.0), ("moving_variance", 1.0)):
                v["u%d/BatchNormalization/%s" % (i, nm)] = np.full(wd, a)

    h, w, cin = H, W, 1
    for i, (C, k, s) in enumerate(convs):
        pf = convs[i - 1][0] if i else 1
        v["u%d/W" % i], v["u%d/b" % i] = rnd(k, k, cin, C, fan=cin * k * k), rs.uniform(0, 0.1, C)
        bn_vars(i, C)
        if i > 0:
            v["z%d_zu_u/W" % i], v["z%d_zu_u/b" % i] = rnd(3, 3, pf, pf, fan=9 * pf), np.ones(pf)
            v["z%d_zu_proj/W" % i] = np.abs(rnd(k, k, pf, C, fan=k * k * pf))
        v["z%d_yu_u/W" % i], v["z%d_yu_u/b" % i] = rnd(3, 3, pf, 1, fan=9 * pf), np.ones(1)
        v["z%d_yu/W" % i] = 3.0 * rnd(k, k, 1, C, fan=k * k)
        v["z%d_y_red/W" % i], v["z%d_y_red/b" % i] = rnd(k, k, 1, 1, fan=k * k), rs.uniform(-0.1, 0.1, 1)
        v["z%d_u/W" % i], v["z%d_u/b" % i] = rnd(k, k, pf, C, fan=k * k * pf), rs.uniform(-0.1, 0.1, C)
        cin, h, w = C, -(-h // s), -(-w // s)
    prev = h * w * cin
    for j, sz in enumerate(fcs):
        i = Lc + j
        sc = 0.005 if j == len(fcs) - 1 else 1.0
        v["u%d/W" % i], v["u%d/b" % i] = rnd(prev, sz, fan=prev), rs.uniform(0, 0.1, sz)
        if sz != 1:
            bn_vars(i, sz)
        v["z%d_zu_u/W" % i], v["z%d_zu_u/b" % i] = rnd(prev, prev, fan=prev), np.ones(prev)
        v["z%d_zu_proj/W" % i] = sc * np.abs(rnd(prev, sz, fan=prev))
        v["z%d_u/W" % i], v["z%d_u/b" % i] = sc * rnd(prev, sz, fan=prev), np.zeros(sz)
        prev = sz
    return v


def gates(V, spec, x, bn_eps=1e-5):
    """x-path of Model.f for x [B, H*W] -> (cz, cy, d) lists over the Lc + Ld layers, flattened per sample in the
    layouts of include/icnn_b200.h (conv maps NHWC)."""
    H, W, Lc, Ld = spec.H, spec.W, len(spec.convs), len(spec.fcs)
    B = x.shape[0]
    x4 = x.reshape(B, 1, H, W)
    flat = lambda t: t.permute(0, 2, 3, 1).reshape(B, -1) if t.dim() == 4 else t      # noqa: E731

    def bn(u, i):
        sh = (1, -1, 1, 1) if u.dim() == 4 else (1, -1)
        p = lambda nm: V["u%d/BatchNormalization/%s" % (i, nm)].reshape(sh)           # noqa: E731
        return (u - p("moving_mean")) / torch.sqrt(p("moving_variance") + bn_eps) * p("gamma") + p("beta")

    us, prev = [], x4
    for i, (_c, _k, s) in enumerate(spec.convs):
        prev = bn(torch.relu(_same_conv(prev, V["u%d/W" % i], V["u%d/b" % i], s)), i)
        us.append(prev)
    for j, sz in enumerate(spec.fcs[:-1]):
        i = Lc + j
        prev = bn(torch.relu(flat(prev) @ V["u%d/W" % i] + V["u%d/b" % i]), i)
        us.append(prev)
    cz, cy, d = [None] * (Lc + Ld), [None] * (Lc + Ld), [None] * (Lc + Ld)
    for i, (_c, _k, s) in enumerate(spec.convs):
        P = x4 if i == 0 else us[i - 1]
        cy[i] = flat(_same_conv(P, V["z%d_yu_u/W" % i], V["z%d_yu_u/b" % i], 1))
        if i > 0:
            cz[i] = flat(torch.relu(_same_conv(P, V["z%d_zu_u/W" % i], V["z%d_zu_u/b" % i], 1)))
        d[i] = flat(_same_conv(P, V["z%d_u/W" % i], V["z%d_u/b" % i], s))
    for j in range(Ld):
        i = Lc + j
        P = flat(us[i - 1])
        cz[i] = torch.relu(P @ V["z%d_zu_u/W" % i] + V["z%d_zu_u/b" % i])
        d[i] = P @ V["z%d_u/W" % i] + V["z%d_u/b" % i]
    return cz, cy, d


def y_energy(V, spec, cz, cy, d, y):
    """y-path of Model.f for rows y [R, H*W] with per-row gates -> (E [R], hidden pre-activations [R, .] per layer,
    the y_red biases broadcast per row [R, 1, 1, 1] for l < Lc - 1)."""
    H, W, Lc = spec.H, spec.W, len(spec.convs)
    R = y.shape[0]
    nchw = lambda t, h, w: t.reshape(R, h, w, -1).permute(0, 3, 1, 2)                # noqa: E731
    r, z, h, w, pres, brows = y.reshape(R, 1, H, W), None, H, W, [], []
    for i, (C, _k, s) in enumerate(spec.convs):
        ho, wo = -(-h // s), -(-w // s)
        a = _same_conv(r * nchw(cy[i], h, w), V["z%d_yu/W" % i], None, s) + nchw(d[i], ho, wo)
        if i > 0:
            a = a + _same_conv(z * nchw(cz[i], h, w), V["z%d_zu_proj/W" % i], None, s)
        if i + 1 < Lc:     # (the bias per row: the rows' own d E_r / d bred_l)
            brows.append(V["z%d_y_red/b" % i].expand(R).reshape(R, 1, 1, 1))
            r = _same_conv(r, V["z%d_y_red/W" % i], None, s) + brows[-1]
        pres.append(a.reshape(R, -1))
        z, h, w = torch.relu(a), ho, wo
    z = z.permute(0, 2, 3, 1).reshape(R, -1)
    for j, sz in enumerate(spec.fcs):
        i = Lc + j
        a = (z * cz[i]) @ V["z%d_zu_proj/W" % i] + d[i]
        if sz != 1:
            pres.append(a)
            a = torch.relu(a)
        z = a
    return z.reshape(-1), pres, brows


def train_grad(spec, x, Y, Vr, c, counts, device="cpu", bn_eps=1e-5, dtype=torch.float64):
    """spec: icnn_b200.conv_picnn.parse_variables(...).  Returns ({trainable name: gradient in the variable's shape},
    {'dcy': [Lc], 'dcz': [Lc + Ld], 'dd': [Lc + Ld]} per-sample gate adjoints [B, .], min relative
    pre-activation per row, {'z{l}_y_red/b': sum_r |c_r dE_r/dbred_l|}), in ``dtype``.  The y_red bias gradient is a sum
    whose terms cancel (a sample's c sum to zero): the last dict is the scale its rounding error is measured on."""
    f64 = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64), device=device).to(dtype)   # noqa: E731
    Lc, Ld = len(spec.convs), len(spec.fcs)
    names = trainable(list(spec.vars), Lc, Ld)
    V = {k: f64(v).requires_grad_(k in names) for k, v in spec.vars.items()}
    x = f64(x).reshape(-1, spec.H * spec.W)
    B = x.shape[0]
    counts = np.asarray(counts, dtype=np.int64)
    iu = torch.as_tensor(np.repeat(np.arange(B), counts), device=device)
    cz, cy, d = gates(V, spec, x, bn_eps)
    G = [g for g in cz + cy + d if g is not None]
    rowg = lambda lst: [None if g is None else g[iu] for g in lst]                       # noqa: E731
    y = f64(Y).reshape(-1, spec.H * spec.W).requires_grad_()
    E, pres, brows = y_energy(V, spec, rowg(cz), rowg(cy), rowg(d), y)
    (gy,) = torch.autograd.grad(E.sum(), y, create_graph=True)
    # scale of dF/dbred_l = sum_r c_r dE_r/dbred_l: a sample's c sum to zero, so the sum mostly cancels
    sb = torch.autograd.grad(E.sum(), brows, retain_graph=True) if brows else ()
    cr = f64(c).reshape(-1)
    bscale = {"z%d_y_red/b" % l: float((cr * g.reshape(-1)).abs().sum()) for l, g in enumerate(sb)}
    F = (f64(c).reshape(-1) * E).sum() + (f64(Vr).reshape(gy.shape) * gy).sum()
    out = torch.autograd.grad(F, [V[k] for k in names] + G, allow_unused=True)
    grads = {}
    for k, g in zip(names, out[:len(names)]):
        grads[k] = (torch.zeros_like(V[k]) if g is None else g).detach().cpu().numpy()
    it = iter(out[len(names):])

    def take(lst):
        res = []
        for g in lst:
            t = None if g is None else next(it)
            res.append(None if g is None else (torch.zeros_like(g) if t is None else t).detach().cpu().numpy())
        return res
    adj = dict(dcz=take(cz), dcy=take(cy), dd=take(d))
    adj["dcy"] = adj["dcy"][:Lc]
    with torch.no_grad():
        rel = torch.full((y.shape[0],), float("inf"), dtype=torch.float64, device=device)
        for a in pres:
            aa = a.abs()
            rel = torch.minimum(rel, aa.min(1).values / aa.max(1).values.clamp_min(1e-300))
    return grads, adj, rel.cpu().numpy(), bscale
