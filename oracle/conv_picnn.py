"""A convolutional PICNN energy in plain torch, written from completion/icnn_ebundle.py:337-452 (the
architecture the reference actually uses on Olivetti: three conv z-layers 32x8/4, 64x4/2, 64x3/1 with
'same' padding, then FC 512 and 1; batch-norm left out, see SURVEY.md section 8c).  TEST INFRASTRUCTURE ONLY: it
plays the role of the USER's ``fg`` in callback mode -- the library never sees the network, only (f, g).  Its
``same_conv`` is the oracle's one TensorFlow 'SAME' convolution (oracle/conv_energy.py and
oracle/conv_train_grad_torch.py use it too).
Pinned by the reference's own Model.__init__ / Model.f executed on oracle/tf_shim.py (E_ and dE_dy_ agree to 1e-10 at the
Olivetti dims: tests/test_oracle_tfshim.py::test_conv_picnn_helper_matches_the_reference_graph)."""
import numpy as np
import torch
import torch.nn.functional as F

CONVS = ((32, 8, 4), (64, 4, 2), (64, 3, 1))
FCS = (512, 1)


def same_conv(x, w, b, stride):
    """tflearn conv_2d default padding='same': out = ceil(in / stride), extra padding at the end."""
    k = w.shape[-1]
    pads = []
    for size in (x.shape[-1], x.shape[-2]):            # F.pad takes (W_left, W_right, H_top, H_bottom)
        out = -(-size // stride)
        tot = max((out - 1) * stride + k - size, 0)
        pads += [tot // 2, tot - tot // 2]
    return F.conv2d(F.pad(x, pads), w, b, stride=stride)


def same_conv_tf(x, w_tf, b, stride):
    """``same_conv`` with a TensorFlow kernel [k, k, c_in, c_out]."""
    return same_conv(x, w_tf.permute(3, 2, 0, 1), b, stride)


class ConvPICNN:
    def __init__(self, H, W, seed=0, dtype=torch.float32, device="cpu"):
        g = torch.Generator().manual_seed(seed)

        def rnd(*shape, fan):
            return (torch.randn(*shape, generator=g, dtype=torch.float64) / np.sqrt(fan)).to(dtype=dtype, device=device)

        self.H, self.W, self.dtype, self.device = H, W, dtype, device
        P = self.P = {}
        cin, h, w = 1, H, W
        for i, (nf, k, s) in enumerate(CONVS):
            P["u%d" % i] = (rnd(nf, cin, k, k, fan=cin * k * k), torch.zeros(nf, dtype=dtype, device=device))
            pf = CONVS[i - 1][0] if i else 1
            if i > 0:
                P["zu_u%d" % i] = (rnd(pf, pf, 3, 3, fan=pf * 9), torch.ones(pf, dtype=dtype, device=device))
                P["zu_proj%d" % i] = rnd(nf, pf, k, k, fan=pf * k * k).abs()        # 'proj' weights >= 0 (makeCvx)
            P["yu_u%d" % i] = (rnd(1, pf, 3, 3, fan=pf * 9), torch.ones(1, dtype=dtype, device=device))
            P["yu%d" % i] = 3.0 * rnd(nf, 1, k, k, fan=k * k)
            P["y_red%d" % i] = (rnd(1, 1, k, k, fan=k * k), torch.zeros(1, dtype=dtype, device=device))
            P["z_u%d" % i] = (rnd(nf, pf, k, k, fan=pf * k * k), torch.zeros(nf, dtype=dtype, device=device))
            cin, h, w = nf, -(-h // s), -(-w // s)
        flat = cin * h * w
        prev_u, prev_z = flat, flat
        for j, sz in enumerate(FCS):
            i = len(CONVS) + j
            P["u%d" % i] = (rnd(prev_u, sz, fan=prev_u), torch.zeros(sz, dtype=dtype, device=device))
            P["zu_u%d" % i] = (rnd(prev_u, prev_z, fan=prev_u), torch.ones(prev_z, dtype=dtype, device=device))
            P["zu_proj%d" % i] = rnd(prev_z, sz, fan=prev_z).abs()
            P["z_u%d" % i] = (rnd(prev_u, sz, fan=prev_u), torch.zeros(sz, dtype=dtype, device=device))
            prev_u, prev_z = sz, sz
        # scale of the width-1 output layer: gradients of O(1..10) so that y* is not saturated
        i = len(CONVS) + len(FCS) - 1
        P["zu_proj%d" % i] = P["zu_proj%d" % i] * 0.005
        P["z_u%d" % i] = (P["z_u%d" % i][0] * 0.005, P["z_u%d" % i][1])

    def to(self, dtype, device):
        other = ConvPICNN.__new__(ConvPICNN)
        other.H, other.W, other.dtype, other.device = self.H, self.W, dtype, device
        mv = lambda t: t.to(dtype=dtype, device=device)  # noqa: E731
        other.P = {k: (tuple(mv(t) for t in v) if isinstance(v, tuple) else mv(v)) for k, v in self.P.items()}
        return other

    def energy(self, x, y):
        """x, y: [B, 1, H, W] -> energies [B]."""
        P = self.P
        us, prev = [], x
        for i, (nf, k, s) in enumerate(CONVS):
            prev = torch.relu(same_conv(prev, *P["u%d" % i], s))
            us.append(prev)
        prev = prev.flatten(1)
        for j, sz in enumerate(FCS):
            i = len(CONVS) + j
            prev = prev @ P["u%d" % i][0] + P["u%d" % i][1]
            if sz != 1:
                prev = torch.relu(prev)
            us.append(prev)
        prevU, prevZ, y_red = x, None, y
        for i, (nf, k, s) in enumerate(CONVS):
            z = same_conv(y_red * same_conv(prevU, *P["yu_u%d" % i], 1), P["yu%d" % i], None, s)
            z = z + same_conv(prevU, *P["z_u%d" % i], s)
            if i > 0:
                zu_u = torch.relu(same_conv(prevU, *P["zu_u%d" % i], 1))
                z = z + same_conv(prevZ * zu_u, P["zu_proj%d" % i], None, s)
            y_red = same_conv(y_red, *P["y_red%d" % i], s)
            prevZ = torch.relu(z)
            prevU = us[i]
        prevZ, prevU = prevZ.flatten(1), prevU.flatten(1)
        for j, sz in enumerate(FCS):
            i = len(CONVS) + j
            zu_u = torch.relu(prevU @ P["zu_u%d" % i][0] + P["zu_u%d" % i][1])
            z = (prevZ * zu_u) @ P["zu_proj%d" % i] + prevU @ P["z_u%d" % i][0] + P["z_u%d" % i][1]
            if sz != 1:
                z = torch.relu(z)
            prevU, prevZ = us[i], z
        return z.reshape(-1)

    def make_fg(self, x, as_numpy=True):
        """``fg(y [B, n]) -> (f [B], g [B, n])`` with the reference's contract
        (completion/icnn_ebundle.py:218-221: sess.run([E_, dE_dy_]))."""
        B = x.shape[0]
        xt = torch.as_tensor(x, dtype=self.dtype, device=self.device).reshape(B, 1, self.H, self.W)

        def fg(y):
            yt = torch.as_tensor(y, dtype=self.dtype, device=self.device).reshape(B, 1, self.H, self.W).requires_grad_()
            E = self.energy(xt, yt)
            (g,) = torch.autograd.grad(E.sum(), yt)
            f, g = E.detach(), g.reshape(B, -1)
            return (f.cpu().numpy(), g.cpu().numpy()) if as_numpy else (f, g)
        return fg
