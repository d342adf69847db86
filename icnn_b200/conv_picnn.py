"""Host-side handle of the convolutional PICNN of the image-completion experiment and its bound ``fg``.

The energy is the reference's ``Model.f`` (completion/icnn_ebundle.py:337-452, = completion/icnn.back.py:276-396):
conv z-layers with TensorFlow 'SAME' padding, then dense z-layers ending in the width-1 energy.  The y-path (the part
every solver iteration evaluates, f and df/dy) runs in ``libicnn_b200.so`` (``icnn_conv_picnn_*``); the x-path (u
layers with inference-mode batch-norm and the gates, once per minibatch) runs here in torch with TF32 switched off.

    net = ConvPICNN.from_variables({v.name[:-2]: sess.run(v) for v in tf.trainable_variables() + bn stats}, H, W)
    fg = net.bind(x)                           # x [B, H*W]
    y, G, h, lam, ys, nIters = bundle_entropy.solveBatch(fg, y0, nIter=30)
    y, f = gd.solve(fg, y0, 30, lr=.01, momentum=.9)
"""
from __future__ import annotations

import contextlib
import ctypes as C
import re
import types

import numpy as np
import torch
import torch.nn.functional as F

from . import _capi
from .picnn import default_device

__all__ = ["parse_variables", "ConvPICNN", "BoundConvPICNN"]

_BN = ("gamma", "beta", "moving_mean", "moving_variance")


def _default_stride(k):
    """Stride the reference pairs with each kernel size (its DQN stack: 8 -> 4, 4 -> 2, 3 -> 1)."""
    return k // 2 if k % 2 == 0 else 1


def parse_variables(variables, H, W, strides=None):
    """Check the reference's TensorFlow variable dict of the completion ``Model`` and infer its architecture.

    ``variables``: {name: array}, names without the ':0' suffix, e.g. 'u0/W', 'u0/BatchNormalization/gamma',
    'z1_zu_proj/W', 'z0_y_red/b'; conv kernels [k, k, c_in, c_out], dense weights [in, out] with the input being the
    NHWC-flattened feature map.  The strides are not part of the variables: ``strides`` gives them per conv layer,
    by default the reference's choice for each kernel size (8 -> 4, 4 -> 2, 3 -> 1); they are checked against the
    width of the first dense layer.  Returns a namespace with ``convs`` [(C, k, s)], ``fcs``, ``H``, ``W`` and
    ``vars`` (float32 arrays).  A missing, unused or mis-shaped variable raises ValueError naming it."""
    V = {re.sub(r":0$", "", k): np.asarray(v) for k, v in variables.items()}
    Lc = 0
    while "z%d_y_red/W" % Lc in V:
        Lc += 1
    if Lc == 0:
        raise ValueError("conv PICNN variables: missing variable 'z0_y_red/W' (no conv z-layer found)")
    Ltot = Lc
    while "z%d_u/W" % Ltot in V:
        Ltot += 1
    if Ltot == Lc:
        raise ValueError("conv PICNN variables: missing variable 'z%d_u/W' (no dense z-layer found)" % Lc)

    def get(name, ndim):
        if name not in V:
            raise ValueError("conv PICNN variables: missing variable %r" % name)
        a = V[name]
        if a.ndim != ndim:
            raise ValueError("conv PICNN variables: %r has shape %s, expected %d dimensions" % (name, a.shape, ndim))
        return a

    convs = []
    for i in range(Lc):
        w = get("z%d_u/W" % i, 4)
        if w.shape[0] != w.shape[1]:
            raise ValueError("conv PICNN variables: 'z%d_u/W' has shape %s, expected [k, k, c_in, c_out]" % (i, w.shape))
        k, Cout = int(w.shape[0]), int(w.shape[3])
        s = _default_stride(k) if strides is None else int(strides[i])
        convs.append((Cout, k, s))
    fcs = [int(get("z%d_u/W" % i, 2).shape[1]) for i in range(Lc, Ltot)]
    if fcs[-1] != 1:
        raise ValueError("conv PICNN variables: 'z%d_u/W' has shape %s, the last dense layer must have width 1"
                         % (Ltot - 1, V["z%d_u/W" % (Ltot - 1)].shape))

    expect = {}
    h, w_, cin = H, W, 1
    for i, (Cc, k, s) in enumerate(convs):
        cp = convs[i - 1][0] if i else 1        # channels of the x-path input P_i (x, or u_{i-1})
        expect["u%d/W" % i] = (k, k, cin, Cc)
        expect["u%d/b" % i] = (Cc,)
        for nm in _BN:
            expect["u%d/BatchNormalization/%s" % (i, nm)] = (Cc,)
        if i > 0:
            expect["z%d_zu_u/W" % i] = (3, 3, cp, cp)
            expect["z%d_zu_u/b" % i] = (cp,)
            expect["z%d_zu_proj/W" % i] = (k, k, cp, Cc)
        expect["z%d_yu_u/W" % i] = (3, 3, cp, 1)
        expect["z%d_yu_u/b" % i] = (1,)
        expect["z%d_yu/W" % i] = (k, k, 1, Cc)
        expect["z%d_y_red/W" % i] = (k, k, 1, 1)
        expect["z%d_y_red/b" % i] = (1,)
        expect["z%d_u/W" % i] = (k, k, cp, Cc)
        expect["z%d_u/b" % i] = (Cc,)
        cin, h, w_ = Cc, -(-h // s), -(-w_ // s)
    prev = h * w_ * cin
    for j, sz in enumerate(fcs):
        i = Lc + j
        expect["u%d/W" % i] = (prev, sz)
        expect["u%d/b" % i] = (sz,)
        if sz != 1:
            for nm in _BN:
                expect["u%d/BatchNormalization/%s" % (i, nm)] = (sz,)
        expect["z%d_zu_u/W" % i] = (prev, prev)
        expect["z%d_zu_u/b" % i] = (prev,)
        expect["z%d_zu_proj/W" % i] = (prev, sz)
        expect["z%d_u/W" % i] = (prev, sz)
        expect["z%d_u/b" % i] = (sz,)
        prev = sz
    for name, shape in expect.items():
        a = get(name, len(shape))
        if tuple(a.shape) != shape:
            hint = " (the strides %s do not give this width)" % ([s for _, _, s in convs],) \
                if name in ("u%d/W" % Lc, "z%d_zu_u/W" % Lc) and a.shape[0] != shape[0] else ""
            raise ValueError("conv PICNN variables: %r has shape %s, expected %s%s" % (name, a.shape, shape, hint))
        if "_zu_proj/" in name and np.any(a < 0):
            raise ValueError("conv PICNN variables: %r has negative entries (the energy is convex in y only for "
                             "non-negative z weights; the reference keeps them >= 0 by makeCvx / proj)" % name)
    extra = sorted(set(V) - set(expect))
    if extra:
        raise ValueError("conv PICNN variables: unused variable %r" % extra[0])
    return types.SimpleNamespace(H=int(H), W=int(W), convs=convs, fcs=fcs,
                                 vars={k: np.ascontiguousarray(V[k], dtype=np.float32) for k in expect})


def _same_conv(x, w_tf, b, stride):
    """TensorFlow 'SAME' conv on an NCHW tensor with a [k, k, c_in, c_out] kernel (the odd pad at the end)."""
    k = w_tf.shape[0]
    pads = []
    for size in (x.shape[-1], x.shape[-2]):
        out = -(-size // stride)
        tot = max((out - 1) * stride + k - size, 0)
        pads += [tot // 2, tot - tot // 2]
    return F.conv2d(F.pad(x, pads), w_tf.permute(3, 2, 0, 1), b, stride=stride)


@contextlib.contextmanager
def _no_tf32():
    """FP32 convolutions and matmuls inside the block; the caller's global flags are restored afterwards."""
    mm = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.backends.cudnn.flags(enabled=torch.backends.cudnn.enabled, benchmark=torch.backends.cudnn.benchmark,
                                        deterministic=torch.backends.cudnn.deterministic, allow_tf32=False):
            yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = mm


class ConvPICNN:
    """Weights of a convolutional PICNN on one CUDA device (see the module docstring)."""

    def __init__(self, spec, bn_eps=1e-5, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("icnn_b200.ConvPICNN needs a CUDA device (no CPU fallback)")
        self.device = torch.device(device) if device is not None else default_device()
        self.H, self.W, self.convs, self.fcs = spec.H, spec.W, list(spec.convs), list(spec.fcs)
        self.n = self.H * self.W
        self.Lc, self.Ld = len(self.convs), len(self.fcs)
        self.bn_eps = float(bn_eps)
        self.vars = {k: torch.as_tensor(v, device=self.device) for k, v in spec.vars.items()}
        self._h = None
        self._pack()

    @classmethod
    def from_variables(cls, variables, H, W, bn_eps=1e-5, device=None, strides=None):
        """Build from the reference's TensorFlow variable dict (:func:`parse_variables`)."""
        return cls(parse_variables(variables, H, W, strides=strides), bn_eps=bn_eps, device=device)

    def _pack(self):
        """Hand the y-path weights to the C library, which keeps packed TF32-split copies."""
        if self._h is not None and self._h.value:
            _capi.lib.icnn_conv_picnn_destroy(self._h)
            self._h = None
        V, Lc, Ld = self.vars, self.Lc, self.Ld
        i32 = lambda a: (C.c_int32 * len(a))(*a)       # noqa: E731
        self._keep = [i32([c for c, _, _ in self.convs]), i32([k for _, k, _ in self.convs]),
                      i32([s for _, _, s in self.convs]), i32(self.fcs)]
        wz = _capi.ptr_array([None] + [V["z%d_zu_proj/W" % i] for i in range(1, Lc + Ld)])
        wy = _capi.ptr_array([V["z%d_yu/W" % i] for i in range(Lc)])
        wr = _capi.ptr_array([V["z%d_y_red/W" % i] for i in range(Lc)])
        br = _capi.ptr_array([V["z%d_y_red/b" % i] for i in range(Lc)])
        desc = _capi.ConvPicnnDesc(self.H, self.W, Lc, *self._keep[:3], Ld, self._keep[3],
                                   *[C.cast(a, _capi._fpp) for a in (wz, wy, wr, br)])
        handle = C.c_void_p()
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            _capi.check(_capi.lib.icnn_conv_picnn_create(C.byref(desc), C.byref(handle), C.c_void_p(stream)))
        self._h = handle
        self._versions = {k: t._version for k, t in V.items()}

    def update_weights(self):
        """Re-pack after the tensors in ``self.vars`` were modified in place; ``bind`` refuses stale copies."""
        with torch.cuda.device(self.device):
            self._pack()

    def _check_fresh(self):
        if {k: t._version for k, t in self.vars.items()} != self._versions:
            raise RuntimeError("ConvPICNN: a weight tensor was modified in place after it was packed for the device "
                               "library; call net.update_weights() before bind()")

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                _capi.lib.icnn_conv_picnn_destroy(h)
            except Exception:
                pass
            self._h = None

    def workspace(self, B):
        nbytes = _capi.lib.icnn_conv_picnn_workspace_bytes(self._h, int(B))
        return torch.empty(max(nbytes, 4), dtype=torch.uint8, device=self.device)

    def _bn(self, u, i, channel_dim, V):
        shape = [1] * u.dim()
        shape[channel_dim] = -1
        p = lambda nm: V["u%d/BatchNormalization/%s" % (i, nm)].reshape(shape)   # noqa: E731
        return (u - p("moving_mean")) / torch.sqrt(p("moving_variance") + self.bn_eps) * p("gamma") + p("beta")

    def gates(self, x):
        """x-path of Model.f (completion/icnn_ebundle.py:349-366,374-440) for x [B, H*W]: the gate lists of
        include/icnn_b200.h (conv maps NHWC), in float32 with TF32 off.  Batch-norm is applied as is, not folded:
        the next conv's zero padding sees the normalised values."""
        x = torch.as_tensor(x, device=self.device).to(torch.float32)
        with torch.no_grad(), _no_tf32():
            return self._gates(x, self.vars)

    def _gates(self, x, V):
        """``gates`` on the weight dict ``V`` (differentiable in its tensors; the caller sets grad mode and TF32)."""
        Lc, Ld = self.Lc, self.Ld
        B = int(x.shape[0])
        nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()                      # noqa: E731
        flat = lambda t: nhwc(t).reshape(B, -1) if t.dim() == 4 else t          # noqa: E731
        cy, cz, d = [None] * (Lc + Ld), [None] * (Lc + Ld), [None] * (Lc + Ld)
        us, prev = [], x.reshape(B, 1, self.H, self.W)
        for i, (_c, _k, s) in enumerate(self.convs):
            prev = self._bn(torch.relu(_same_conv(prev, V["u%d/W" % i], V["u%d/b" % i], s)), i, 1, V)
            us.append(prev)
        for j, sz in enumerate(self.fcs):
            i = Lc + j
            prev = flat(prev) @ V["u%d/W" % i] + V["u%d/b" % i]
            if sz != 1:
                prev = self._bn(torch.relu(prev), i, 1, V)
            us.append(prev)
        for i, (_c, _k, s) in enumerate(self.convs):
            P = x.reshape(B, 1, self.H, self.W) if i == 0 else us[i - 1]
            cy[i] = _same_conv(P, V["z%d_yu_u/W" % i], V["z%d_yu_u/b" % i], 1).reshape(B, -1).contiguous()
            if i > 0:
                cz[i] = nhwc(torch.relu(_same_conv(P, V["z%d_zu_u/W" % i], V["z%d_zu_u/b" % i], 1)))
            d[i] = nhwc(_same_conv(P, V["z%d_u/W" % i], V["z%d_u/b" % i], s))
        for j in range(Ld):
            i = Lc + j
            P = flat(us[i - 1])
            cz[i] = torch.relu(P @ V["z%d_zu_u/W" % i] + V["z%d_zu_u/b" % i]).contiguous()
            d[i] = (P @ V["z%d_u/W" % i] + V["z%d_u/b" % i]).contiguous()
        return cz, cy, d

    def bind(self, x):
        """fg object for a minibatch x [B, H*W]."""
        self._check_fresh()
        return BoundConvPICNN(self, x)


class BoundConvPICNN:
    """``fg`` for one minibatch: callable with the reference's numpy contract; ``solveBatch`` and ``gd.solve`` run
    their whole loop on the device with it."""

    def __init__(self, net: ConvPICNN, x):
        self.net = net
        with torch.cuda.device(net.device):
            self.cz, self.cy, self.d = net.gates(x)
            self.B = int(self.d[0].shape[0])
            self._cy, self._cz, self._d = (_capi.ptr_array(v) for v in (self.cy, self.cz, self.d))
            self.c_gates = _capi.Gates(self.B, C.cast(self._cy, _capi._fpp), C.cast(self._cz, _capi._fpp),
                                       C.cast(self._d, _capi._fpp), 1.0, 0.0, 1.0)
            self.ws = net.workspace(self.B)
            self.x = torch.as_tensor(x, device=net.device).to(torch.float32)   # the training gradient's x-path

    def fg_device(self, y32, f=None, g=None):
        """f [B], g [B, n] (float32 CUDA tensors) for a float32 CUDA iterate y32 [B, n]."""
        net = self.net
        assert y32.is_cuda and y32.dtype == torch.float32 and y32.is_contiguous()
        assert tuple(y32.shape) == (self.B, net.n)
        if f is None:
            f = torch.empty(self.B, dtype=torch.float32, device=net.device)
        if g is None:
            g = torch.empty(self.B, net.n, dtype=torch.float32, device=net.device)
        with torch.cuda.device(net.device):
            stream = torch.cuda.current_stream().cuda_stream
            _capi.check(_capi.lib.icnn_conv_picnn_fg(
                net._h, C.byref(self.c_gates), y32.data_ptr(), f.data_ptr(), g.data_ptr(),
                net.n, None, None, 0, self.ws.data_ptr(), None, C.c_void_p(stream)))
        return f, g

    def __call__(self, y):
        """numpy in, numpy out: fg(y [B, n]) -> (f [B] float32, g [B, n] float32)."""
        y32 = torch.as_tensor(np.ascontiguousarray(y, dtype=np.float32), device=self.net.device)
        f, g = self.fg_device(y32)
        return f.cpu().numpy(), g.cpu().numpy()


# ---- shared by the training gradients (bundle_grad: the bundle-entropy mode, gd_grad: the back-optimisation mode) ----

def conv_trainable(net):
    """Names of the TF variables the reference's gv_ holds for this conv net: every trainable variable except the
    batch-norm statistics, the last u-layer (nothing consumes it) and the last conv layer's y_red (r_Lc is never
    used), in the net's variable order."""
    last_u = "u%d/" % (net.Lc + net.Ld - 1)
    last_red = "z%d_y_red/" % (net.Lc - 1)
    return [k for k in net.vars
            if not k.endswith(("/moving_mean", "/moving_variance")) and not k.startswith((last_u, last_red))]


def conv_gd_trainable(net):
    """Names of the TF variables the gv_ of the back-optimisation mode holds (completion/icnn.back.py:153-155, the
    gradient of the loss through the unrolled GD steps, which see E only through dE/dy): ``conv_trainable`` without
    the output layer's additive gate 'z{NL-1}_u/*', which dE/dy does not depend on.  The other layers' additive gates
    'z{l}_u/*' pass through a ReLU, so TensorFlow connects them to the loss, with a gradient that is exactly zero."""
    out_d = "z%d_u/" % (net.Lc + net.Ld - 1)
    return [k for k in conv_trainable(net) if not k.startswith(out_d)]


def _train_grad_buffers(fg):
    """Output buffers of one icnn_conv_train_grad / icnn_conv_gd_backward call on ``fg``'s minibatch: a dict of the
    per-layer lists 'dWz', 'dWy', 'dWred', 'dbred' (in the variables' shapes), 'dcy', 'dcz', 'dd' ([B, flat gate]),
    and the ConvTrainGrads struct with the pointer arrays it points into (these must outlive the work)."""
    net, dev, B = fg.net, fg.net.device, fg.B
    Lc, NL = net.Lc, net.Lc + net.Ld
    Vr = net.vars
    z = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)  # noqa: E731
    o = dict(dWz=[None] + [z(*Vr["z%d_zu_proj/W" % i].shape) for i in range(1, NL)],
             dWy=[z(*Vr["z%d_yu/W" % l].shape) for l in range(Lc)],
             dWred=[z(*Vr["z%d_y_red/W" % l].shape) if l + 1 < Lc else None for l in range(Lc)],
             dbred=[z(1) if l + 1 < Lc else None for l in range(Lc)],
             dcy=[z(B, fg.cy[l][0].numel()) for l in range(Lc)],
             dcz=[None] + [z(B, fg.cz[i][0].numel()) for i in range(1, NL)],
             dd=[z(B, fg.d[i][0].numel()) for i in range(NL)])
    arrs = [_capi.ptr_array(o[k]) for k in ("dWz", "dWy", "dWred", "dbred", "dcy", "dcz", "dd")]
    gr = _capi.ConvTrainGrads(*[C.cast(a, _capi._fpp) for a in arrs])
    return o, gr, arrs


def _ypath_grads(net, o):
    """{TF variable name: gradient} of the y-path weights from the buffers of ``_train_grad_buffers``."""
    Lc, NL = net.Lc, net.Lc + net.Ld
    grads = {}
    for i in range(1, NL):
        grads["z%d_zu_proj/W" % i] = o["dWz"][i]
    for l in range(Lc):
        grads["z%d_yu/W" % l] = o["dWy"][l]
        if l + 1 < Lc:
            grads["z%d_y_red/W" % l] = o["dWred"][l]
            grads["z%d_y_red/b" % l] = o["dbred"][l]
    return grads


def _gate_vjp(fg, names, dcy, dcz, dd):
    """{k: d(sum over the gates of gate o adjoint) / d net.vars[k]} for k in ``names``: the x-path gradients, by torch
    autograd through a grad-enabled recompute of ``ConvPICNN._gates`` on the minibatch ``fg`` was bound to, with TF32
    off and cuDNN restricted to deterministic algorithms (two calls give the same bits)."""
    net, B, Lc, NL = fg.net, fg.B, fg.net.Lc, fg.net.Lc + fg.net.Ld
    P = {k: (v.detach().requires_grad_() if k in names else v) for k, v in net.vars.items()}
    with torch.enable_grad(), _no_tf32(), torch.backends.cudnn.flags(
            enabled=torch.backends.cudnn.enabled, benchmark=False, deterministic=True, allow_tf32=False):
        gz, gy, gd = net._gates(fg.x, P)
        s = sum((gy[l].reshape(B, -1) * dcy[l]).sum() for l in range(Lc))
        s = s + sum((gz[i].reshape(B, -1) * dcz[i]).sum() for i in range(1, NL))
        s = s + sum((gd[i].reshape(B, -1) * dd[i]).sum() for i in range(NL))
        xg = torch.autograd.grad(s, [P[k] for k in names])
    return dict(zip(names, (g.detach() for g in xg)))
