"""The conv-PICNN GD training gradient on the GPU (icnn_conv_gd_backward, gd_grad with a BoundConvPICNN) against the
float64 torch oracle's literal double backward through the unrolled loop (oracle/conv_gd_grad_torch.py) and the
reference's own graph (tests/golden/conv/conv_gd_grad.npz), at the completion script's lr = 0.01, momentum = 0.9,
nIter = 30 and loss_scale = 2 255^2 / (B n).

Tolerance and kink rule as tests/test_gpu_conv_train_grad.py: every array within RTOL = 2e-4 of its largest entry; a
sample may be set aside only if it disagrees AND the oracle shows a pre-activation within 1e-5 (relative) of zero on
its trajectory (where float32 and float64 iterates may take different sides of a kink); the kept samples are then
compared again, run as their own batch with the full batch's loss_scale."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import conv_gd_grad_torch as O
from oracle import conv_train_grad_torch as T

pytestmark = pytest.mark.gpu
np.seterr(all="ignore")

RTOL = 2e-4
KINK = 1e-5
LR, MOM, NITER = 0.01, 0.9, 30

OLIVETTI = (64, 32, [(32, 8, 4), (64, 4, 2), (64, 3, 1)], [512, 1])
CASES = {
    "olivetti_b70": (OLIVETTI, 70),                                     # the script's batch, tensor-core path
    "odd17x9": ((17, 9, [(5, 3, 2), (7, 2, 1)], [12, 1]), 20),
    "repitch": ((16, 12, [(4, 4, 2), (6, 3, 1)], [9, 1]), 20),          # last conv C = 6: delta repitched
    "ld1": ((12, 10, [(4, 3, 2), (8, 3, 1)], [1]), 20),                 # no dense hidden layer
    "b1": ((10, 8, [(4, 3, 2), (5, 3, 1)], [6, 1]), 1),                 # 30 gradient rows, under 64
}


def relerr(a, b):
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(np.asarray(a, dtype=np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def _net(arch, seed=3):
    import icnn_b200
    from icnn_b200.conv_picnn import parse_variables
    H, W, convs, fcs = arch
    v = T.make_variables(H, W, convs, fcs, seed=seed)
    strides = [s for _, _, s in convs]
    return icnn_b200.ConvPICNN.from_variables(v, H, W, strides=strides), parse_variables(v, H, W, strides=strides)


def _inputs(n, B, seed):
    rs = np.random.RandomState(seed)
    x = rs.uniform(size=(B, n))
    y0 = np.tile(rs.uniform(0.2, 0.8, size=(1, n)), (B, 1))
    return x, y0, rs.uniform(size=(B, n))


def _compare(dev, og, oadj):
    """{name: relative error} over the oracle's gradients and gate adjoints."""
    errs = {k: relerr(dev[k], b) for k, b in og.items()}
    for k in ("dcy", "dcz"):
        for i, b in enumerate(oadj[k]):
            if b is not None:
                errs["%s%d" % (k, i)] = relerr(dev[k][i], b)
    return errs


def _check(net, spec, x, y0, trueY, nIter, tag, loss_scale=None):
    """gd_grad on the device against the oracle with the kink rule; returns (device result, kept samples)."""
    from icnn_b200.gd_grad import conv_gd_trainable, gd_grad
    B, n = x.shape
    ls = 2 * 255.0 ** 2 / (B * n) if loss_scale is None else loss_scale
    fg = net.bind(x)
    yN, dev = gd_grad(fg, y0, trueY, nIter, LR, MOM, ls)
    assert set(dev) == set(conv_gd_trainable(net)) | {"dcy", "dcz"}
    oyN, _loss, og, oadj, rel = O.gd_grad(spec, x, y0, trueY, nIter, LR, MOM, ls, device="cuda")
    assert set(og) == set(conv_gd_trainable(net))
    for k, b in og.items():
        assert dev[k].shape == b.shape, k
    bad = np.abs(yN - oyN).max(axis=1) / max(np.abs(oyN).max(), 1e-30) >= RTOL
    for k in ("dcy", "dcz"):
        for i, b in enumerate(oadj[k]):
            if b is not None:
                bad |= np.abs(dev[k][i] - b).max(axis=1) / max(np.abs(b).max(), 1e-30) >= RTOL
    kink = rel < KINK
    assert not (bad & ~kink).any(), (tag, np.nonzero(bad & ~kink)[0])
    keep = ~(bad & kink)
    assert keep.sum() >= max(1, B // 2), (tag, int((~keep).sum()), B)
    if not keep.all():
        x, y0, trueY = x[keep], y0[keep], trueY[keep]
        yN, dev = gd_grad(net.bind(x), y0, trueY, nIter, LR, MOM, ls)
        oyN, _loss, og, oadj, rel = O.gd_grad(spec, x, y0, trueY, nIter, LR, MOM, ls, device="cuda")
    errs = _compare(dev, og, oadj)
    errs["yN"] = relerr(yN, oyN)
    worst = max(errs, key=errs.get)
    print(tag, "B", B, "set aside", int((~keep).sum()), "max rel err %.2e (%s)" % (errs[worst], worst))
    assert errs[worst] < RTOL, sorted(errs.items(), key=lambda kv: -kv[1])[:6]
    return dev, keep


@pytest.mark.parametrize("tag", ["conv_bn_odd", "conv_bn_olivetti"])
def test_reference_golden(tag, golden_dir):
    """The reference's graph (per-sample gv_, yn_) at its nGdIter: the batch gradient with loss_scale =
    2 255^2 / (B n) is the mean of the per-sample ones over the samples kept; the key set is gv_'s."""
    import os
    import icnn_b200
    from icnn_b200.conv_picnn import parse_variables
    from oracle.gen_golden_conv_grad import probe
    from oracle.gen_golden_conv_gd_grad import case_inputs
    gold = np.load(os.path.join(golden_dir, "conv", "conv_gd_grad.npz"))
    v, x, y0, trueY, H, W = case_inputs(tag)
    net = icnn_b200.ConvPICNN.from_variables(v, H, W)
    nIter = int(gold[tag + "_nGdIter"])
    dev, keep = _check(net, parse_variables(v, H, W), x, y0, trueY, nIter, tag)
    assert set(dev) - {"dcy", "dcz"} == set(str(s) for s in gold[tag + "_gv_names"])
    errs = {}
    for k in gold.files:
        for kind in ("_grad_", "_probe_"):
            if k.startswith(tag + kind):
                name = k[len(tag + kind):]
                got = dev[name] if kind == "_grad_" else probe(dev[name].reshape(-1))
                errs[name] = relerr(got, gold[k][keep].sum(0) / len(x))
    assert len(errs) == 49
    worst = max(errs, key=errs.get)
    print(tag, "vs the reference's gv_: max rel err %.2e (%s)" % (errs[worst], worst))
    assert errs[worst] < RTOL, sorted(errs.items(), key=lambda kv: -kv[1])[:6]


@pytest.mark.parametrize("case", list(CASES))
def test_matches_oracle(case):
    arch, B = CASES[case]
    net, spec = _net(arch)
    x, y0, trueY = _inputs(net.n, B, seed=5)
    _check(net, spec, x, y0, trueY, NITER, case)


def _kappa32(nIter, lr, m):
    """float32 kappa_i as the library forms them: the recurrence in float64 from the float32 lr and m."""
    lr, m = float(np.float32(lr)), float(np.float32(m))
    k, c = np.zeros(nIter, dtype=np.float32), 1.0 + m
    for i in range(nIter - 1, -1, -1):
        k[i] = np.float32(-lr * c)
        c = m * c + 1.0
    return k


def test_composition_pin_and_y_n():
    """y_N is gd.solve's bit for bit, and the result is bit-identical to bundle_grad.train_grad fed the explicit rows
    (Y_i = gd.solve(nIter=i), V = kappa_i a with a = loss_scale (y_N - trueY), c = 0, nIter rows per sample) after
    dropping the output layer's additive gate; the zero entries of gv_ are exactly zero."""
    from icnn_b200 import gd
    from icnn_b200.bundle_grad import train_grad
    from icnn_b200.gd_grad import gd_grad
    arch, B = CASES["odd17x9"]
    net, _spec = _net(arch)
    n, nIter = net.n, 12
    x, y0, trueY = _inputs(n, B, seed=8)
    fg = net.bind(x)
    ls = 2 * 255.0 ** 2 / (B * n)
    yN, g = gd_grad(fg, y0, trueY, nIter, LR, MOM, ls, return_device=True)
    ys = [gd.solve(fg, y0, i, LR, MOM, return_device=True)[0] for i in range(nIter + 1)]
    assert torch.equal(yN, ys[-1])
    dev = yN.device
    a = torch.tensor(ls, dtype=torch.float32, device=dev) * (ys[-1] - torch.as_tensor(trueY, dtype=torch.float32,
                                                                                      device=dev))
    k = torch.as_tensor(_kappa32(nIter, LR, MOM), device=dev)
    Y = torch.stack(ys[:-1], 1).reshape(B * nIter, n)
    V = (k[None, :, None] * a[:, None, :]).reshape(B * nIter, n)
    t = train_grad(fg, Y, V, torch.zeros(B * nIter, device=dev), np.full(B, nIter), return_device=True)
    NL, Lc = net.Lc + net.Ld, net.Lc
    assert set(t) - {"z%d_u/W" % (NL - 1), "z%d_u/b" % (NL - 1), "dd"} == set(g)
    for key, val in g.items():
        for u, w in (zip(val, t[key]) if isinstance(val, list) else [(val, t[key])]):
            if u is not None:
                assert torch.equal(u, w), key
    for i in range(NL - 1):
        assert not g["z%d_u/W" % i].any() and not g["z%d_u/b" % i].any()
    for l in range(Lc - 1):
        assert not g["z%d_y_red/b" % l].any()


def test_zero_and_one_step():
    from icnn_b200.gd_grad import gd_grad
    arch, B = CASES["odd17x9"]
    net, spec = _net(arch)
    x, y0, trueY = _inputs(net.n, 6, seed=4)
    yN, g = gd_grad(net.bind(x), y0, trueY, 0, LR, MOM, 1.0)
    np.testing.assert_array_equal(yN, y0.astype(np.float32))
    for k, v in g.items():
        for a in (v if isinstance(v, list) else [v]):
            assert a is None or not np.any(a), k
    _check(net, spec, x, y0, trueY, 1, "nIter=1")


def test_determinism_chunking_and_tf32_flags(monkeypatch):
    """Two calls are bit-identical; forced chunks agree with one chunk up to the final rounding; the caller's TF32
    flags come back unchanged."""
    from icnn_b200.gd_grad import gd_grad
    arch, B = CASES["odd17x9"]
    net, _spec = _net(arch)
    x, y0, trueY = _inputs(net.n, 24, seed=9)
    fg = net.bind(x)
    monkeypatch.delenv("ICNN_TRAIN_CHUNK", raising=False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", True)      # restored after the test
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", True)
    _yN, a = gd_grad(fg, y0, trueY, NITER, LR, MOM, 1.0)
    assert torch.backends.cuda.matmul.allow_tf32 and torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    _yN, b = gd_grad(fg, y0, trueY, NITER, LR, MOM, 1.0)
    assert not torch.backends.cuda.matmul.allow_tf32 and torch.backends.cudnn.allow_tf32
    for k in a:
        for u, w in (zip(a[k], b[k]) if isinstance(a[k], list) else [(a[k], b[k])]):
            if u is not None:
                np.testing.assert_array_equal(u, w, err_msg=k)
    monkeypatch.setenv("ICNN_TRAIN_CHUNK", "7")        # several chunks, and samples split over chunks
    _yN, s = gd_grad(fg, y0, trueY, NITER, LR, MOM, 1.0)
    for k in a:
        for u, w in (zip(a[k], s[k]) if isinstance(a[k], list) else [(a[k], s[k])]):
            if u is not None:
                assert relerr(w, u) < 1e-6, (k, relerr(w, u))


def test_bad_inputs_raise():
    from icnn_b200 import _capi
    from icnn_b200.gd_grad import gd_grad
    arch, _B = CASES["b1"]
    net, _spec = _net(arch)
    n, B = net.n, 4
    fg = net.bind(np.zeros((B, n)))
    y = np.full((B, n), 0.5)
    with pytest.raises(ValueError):
        gd_grad(fg, y, y, 3, x=np.zeros((B, n)))            # x is the bound minibatch
    with pytest.raises(ValueError):
        gd_grad(fg, y[:3], y, 3)
    with pytest.raises(ValueError):
        gd_grad(fg, y, np.zeros((B, n + 1)), 3)
    with pytest.raises(TypeError):
        gd_grad(net, y, y, 3)
    with pytest.raises(_capi.IcnnError):
        gd_grad(fg, y, y, -1)
    assert b"nIter < 0" in _capi.lib.icnn_last_error()
    assert _capi.lib.icnn_conv_gd_backward_workspace_bytes(net._h, B, 30) > 2 * B * 30 * n * 4
    gates = fg.c_gates
    grads = _capi.ConvTrainGrads()
    assert _capi.lib.icnn_conv_gd_backward(net._h, C.byref(gates), C.c_void_p(16), C.c_void_p(16), 1.0, 1, LR, MOM,
                                           C.c_void_p(16), C.byref(grads), C.c_void_p(16), None) == -1
