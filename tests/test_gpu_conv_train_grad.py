"""The conv-PICNN training gradient d (sum_r F_r) / d theta on the GPU (icnn_conv_train_grad, bundle_grad with a
BoundConvPICNN) against the float64 torch oracle (oracle/conv_train_grad_torch.py) on the same rows.

Tolerance and kink rule as tests/test_gpu_bundle_grad.py: every array within RTOL = 2e-4 of its largest entry; a
sample may be set aside only if it disagrees AND the oracle shows a pre-activation within 1e-5 (relative) of zero at
one of its rows, at most max(1, 2 %) of the samples; the rest is compared again without it."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import conv_train_grad_torch as O

pytestmark = pytest.mark.gpu
np.seterr(all="ignore")

RTOL = 2e-4
KINK = 1e-5

OLIVETTI = (64, 32, [(32, 8, 4), (64, 4, 2), (64, 3, 1)], [512, 1])
CASES = {
    "olivetti": (OLIVETTI, 12, 10),
    "odd17x9": ((17, 9, [(5, 3, 2), (7, 2, 1)], [12, 1]), 20, 10),
    "repitch": ((16, 12, [(4, 4, 2), (6, 3, 1)], [9, 1]), 20, 10),     # last conv C = 6: delta repitched
    "ld1": ((12, 10, [(4, 3, 2), (8, 3, 1)], [1]), 20, 10),            # no dense hidden layer
    "few_rows": ((10, 8, [(4, 3, 2), (5, 3, 1)], [6, 1]), 3, 6),       # fewer than 64 rows
}


def relerr(a, b, scale=0.0):
    """max |a - b| over the largest |b| (or over ``scale`` when larger: the y_red bias gradients, whose row terms
    cancel, are measured against the sum of their terms' magnitudes)"""
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(np.asarray(a, dtype=np.float64) - b).max() / max(np.abs(b).max(), scale, 1e-30))


def _net(arch, seed=3):
    import icnn_b200
    from icnn_b200.conv_picnn import parse_variables
    H, W, convs, fcs = arch
    v = O.make_variables(H, W, convs, fcs, seed=seed)
    strides = [s for _, _, s in convs]
    return icnn_b200.ConvPICNN.from_variables(v, H, W, strides=strides), parse_variables(v, H, W, strides=strides)


def _rows(fg, B, n, nIter, seed):
    """solveBatch on the device, K3 (mse) on its state; rows in float32 with the samples whose KKT matrix is
    numerically singular (cond > 1e9) given zero rows."""
    from icnn_b200 import argmin_grad, bundle_entropy as be
    rs = np.random.RandomState(seed)
    y0 = np.tile(rs.uniform(0.2, 0.8, size=(1, n)), (B, 1))
    yN, G, _h, _lam, _ys, _it, st = be.solveBatch(fg, y0.copy(), nIter=nIter, return_state=True)
    trueY = rs.uniform(size=yN.shape)
    _cy, _clam, _ct, (fY, fV, fc) = argmin_grad.argmin_grad(st, trueY, loss="mse")
    counts = np.array([len(G[u]) for u in range(B)])
    good = np.ones(B, dtype=bool)
    for u in range(B):
        Gu = np.array(G[u], dtype=np.float64)
        if len(Gu):
            yc = np.clip(yN[u], 1e-8, 1 - 1e-8)
            zinv = 1.0 / (1.0 / yc + 1.0 / (1.0 - yc))
            good[u] = np.linalg.cond((Gu * zinv).dot(Gu.T)) <= 1e9
    assert good.mean() >= 0.5
    rows = np.repeat(good, counts)
    f32 = lambda a: np.asarray(a, dtype=np.float32)   # noqa: E731
    return st, trueY, f32(fY[rows]), f32(fV[rows]), f32(fc[rows]), np.where(good, counts, 0)


def _flat_adj(adj):
    return {"%s%d" % (k, i): a for k in ("dcy", "dcz", "dd") for i, a in enumerate(adj[k]) if a is not None}


def _check(fg, spec, Y, V, c, counts, tag):
    from icnn_b200.bundle_grad import train_grad
    B = len(counts)
    x = fg.x.double().cpu().numpy()
    dev = train_grad(fg, Y, V, c, counts, return_device=False)
    og, oadj, rel, bscale = O.train_grad(spec, x, Y, V, c, counts, device="cuda")
    assert set(dev) - {"dcy", "dcz", "dd"} == set(og)
    bad = np.zeros(B, dtype=bool)
    dadj = _flat_adj(dev)
    for k, b in _flat_adj(oadj).items():
        bad |= np.abs(dadj[k] - b).max(axis=1) / max(np.abs(b).max(), 1e-30) >= RTOL
    kink = np.zeros(B, dtype=bool)
    np.logical_or.at(kink, np.repeat(np.arange(B), counts), rel < KINK)
    assert not (bad & ~kink).any(), (tag, np.nonzero(bad & ~kink)[0])
    drop = bad & kink
    assert drop.sum() <= max(1, int(0.02 * B)), (int(drop.sum()), B)
    if drop.any():
        rows = np.repeat(~drop, counts)
        counts = np.where(drop, 0, counts)
        Y, V, c = Y[rows], V[rows], c[rows]
        dev = train_grad(fg, Y, V, c, counts, return_device=False)
        og, oadj, rel, bscale = O.train_grad(spec, x, Y, V, c, counts, device="cuda")
        dadj = _flat_adj(dev)
    errs = {k: relerr(dev[k], b, bscale.get(k, 0.0)) for k, b in og.items()}
    errs.update({k: relerr(dadj[k], b) for k, b in _flat_adj(oadj).items()})
    for k, b in og.items():
        assert dev[k].shape == b.shape, k
    worst = max(errs, key=errs.get)
    print(tag, "rows", len(Y), "samples set aside", int(drop.sum()), "max rel err %.2e (%s)" % (errs[worst], worst))
    assert errs[worst] < RTOL, sorted(errs.items(), key=lambda kv: -kv[1])[:6]
    return dev, ~drop, bscale


@pytest.mark.parametrize("tag", ["conv_bn_odd", "conv_bn_olivetti"])
def test_reference_golden_rows(tag, golden_dir):
    """The rows of the reference's own training step (tests/golden/conv/conv_train_grad.npz) through train_grad:
    against the oracle, and every stored gv_ gradient (whole or probed), summed over the samples kept."""
    import os
    import icnn_b200
    from icnn_b200.conv_picnn import parse_variables
    from oracle.gen_golden_conv_grad import case_rows_inputs, probe
    gold = np.load(os.path.join(golden_dir, "conv", "conv_train_grad.npz"))
    v, x, _y0, _tY, H, W, _n = case_rows_inputs(tag)
    fg = icnn_b200.ConvPICNN.from_variables(v, H, W).bind(x)
    Y, V, c = (gold[tag + k] for k in ("_Y", "_V", "_c"))
    dev, keep, bscale = _check(fg, parse_variables(v, H, W), Y, V, c, gold[tag + "_counts"], tag)
    errs = {}
    for k in gold.files:
        for kind in ("_grad_", "_probe_"):
            if k.startswith(tag + kind):
                name = k[len(tag + kind):]
                got = dev[name] if kind == "_grad_" else probe(dev[name].reshape(-1))
                errs[name] = relerr(got, gold[k][keep].sum(0), bscale.get(name, 0.0))
    assert len(errs) == 51
    worst = max(errs, key=errs.get)
    print(tag, "vs the reference's gv_: max rel err %.2e (%s)" % (errs[worst], worst))
    assert errs[worst] < RTOL, sorted(errs.items(), key=lambda kv: -kv[1])[:6]


@pytest.mark.parametrize("case", list(CASES))
def test_device_chain_matches_oracle(case):
    """solveBatch(conv fg, return_state=True) -> bundle_grad against the oracle on the same rows."""
    from icnn_b200.bundle_grad import bundle_grad, train_grad
    arch, B, nIter = CASES[case]
    net, spec = _net(arch)
    x = np.random.RandomState(5).uniform(size=(B, arch[0] * arch[1]))
    fg = net.bind(x)
    st, trueY, Y, V, c, counts = _rows(fg, B, net.n, nIter, seed=7)
    if case == "few_rows":
        assert len(Y) < 64
    _check(fg, spec, Y, V, c, counts, case)
    # bundle_grad is train_grad on the rows it gathers on the device
    a = bundle_grad(fg, st, trueY, loss="mse", return_device=False)
    from icnn_b200 import argmin_grad
    _cy, _clam, _ct, (fY, fV, fc) = argmin_grad.argmin_grad(st, trueY, loss="mse")
    b = train_grad(fg, fY, fV, fc, st.count.cpu().numpy(), return_device=False)
    for k in a:
        for u, w in (zip(a[k], b[k]) if isinstance(a[k], list) else [(a[k], b[k])]):
            if u is not None:
                np.testing.assert_array_equal(u, w, err_msg=k)


def test_zero_row_sample_and_empty_rows():
    """A sample with zero rows gets zero gate adjoints; no rows at all gives zeros everywhere."""
    from icnn_b200.bundle_grad import train_grad
    arch = CASES["odd17x9"][0]
    net, spec = _net(arch)
    n, B = net.n, 6
    rs = np.random.RandomState(11)
    x = rs.uniform(size=(B, n))
    fg = net.bind(x)
    counts = np.array([3, 0, 2, 4, 0, 1])
    R = int(counts.sum())
    Y = rs.uniform(0.05, 0.95, size=(R, n)).astype(np.float32)
    V = (0.1 * rs.randn(R, n)).astype(np.float32)
    c = rs.randn(R).astype(np.float32)
    _check(fg, spec, Y, V, c, counts, "zero-row sample")
    g = train_grad(fg, Y, V, c, counts, return_device=False)
    for k in ("dcy", "dcz", "dd"):
        for a in g[k]:
            if a is not None:
                assert not np.any(a[counts == 0]) and np.any(a[counts > 0])
    from icnn_b200.bundle_grad import conv_trainable
    gd = train_grad(fg, Y, V, c, counts, return_device=True)      # device tensors, straight into .grad
    for k in conv_trainable(net):
        net.vars[k].grad = gd[k]
        np.testing.assert_array_equal(gd[k].cpu().numpy(), g[k])
    ge = train_grad(fg, np.zeros((0, n)), np.zeros((0, n)), np.zeros(0), np.zeros(B, dtype=int), return_device=False)
    for k, v in ge.items():
        for a in (v if isinstance(v, list) else [v]):
            assert a is None or not np.any(a), k


def test_chunking_determinism_and_tf32_flags(monkeypatch):
    """Two calls are bit-identical; forced chunks cut at sample boundaries agree with one chunk up to the final
    rounding (the weight gradients are float64 sums over rows and chunks, rounded once: a different cut only reorders
    float64 additions); the caller's TF32 flags come back unchanged."""
    from icnn_b200.bundle_grad import train_grad
    arch = CASES["odd17x9"][0]
    net, spec = _net(arch)
    B = 40
    x = np.random.RandomState(2).uniform(size=(B, net.n))
    fg = net.bind(x)
    _st, _tY, Y, V, c, counts = _rows(fg, B, net.n, 10, seed=9)
    monkeypatch.delenv("ICNN_TRAIN_CHUNK", raising=False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", True)      # restored after the test
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", True)
    try:
        a = train_grad(fg, Y, V, c, counts, return_device=False)
        assert torch.backends.cuda.matmul.allow_tf32 and torch.backends.cudnn.allow_tf32
    finally:
        torch.backends.cuda.matmul.allow_tf32 = False
    b = train_grad(fg, Y, V, c, counts, return_device=False)
    assert not torch.backends.cuda.matmul.allow_tf32 and torch.backends.cudnn.allow_tf32
    for k in a:
        for u, w in (zip(a[k], b[k]) if isinstance(a[k], list) else [(a[k], b[k])]):
            if u is not None:
                np.testing.assert_array_equal(u, w, err_msg=k)
    assert counts.max() <= 7
    monkeypatch.setenv("ICNN_TRAIN_CHUNK", "7")        # several chunks, cut at sample boundaries
    s = train_grad(fg, Y, V, c, counts, return_device=False)
    for k in a:
        for u, w in (zip(a[k], s[k]) if isinstance(a[k], list) else [(a[k], s[k])]):
            if u is not None:
                assert relerr(w, u) < 1e-6, (k, relerr(w, u))


def test_bad_inputs_raise_before_any_launch():
    from icnn_b200 import _capi
    from icnn_b200.bundle_grad import bundle_grad, train_grad
    arch = CASES["few_rows"][0]
    net, _spec = _net(arch)
    n, B = net.n, 4
    fg = net.bind(np.zeros((B, n)))
    Y = np.zeros((3, n))
    with pytest.raises(ValueError):
        train_grad(fg, Y, Y, np.zeros(3), [1, 1, 1], x=np.zeros((B, n)))     # x is the bound minibatch
    with pytest.raises(ValueError):
        train_grad(fg, Y, Y, np.zeros(3), [1, 1, 1])                          # counts of the wrong length
    with pytest.raises(ValueError):
        train_grad(fg, Y, Y, np.zeros(3), [1, 1, 1, 1])                       # sum(counts) != rows
    with pytest.raises(ValueError):
        train_grad(fg, Y, Y, np.zeros(3), [1, -1, 2, 1])
    with pytest.raises(ValueError):
        bundle_grad(fg, None, None, loss="hinge")
    off = (C.c_int64 * (B + 1))(0, 1, 0, 2, 3)                              # decreasing offsets
    ptrs = [(C.c_void_p * 8)(*([16] * 8)) for _ in range(7)]                 # never dereferenced
    gr = _capi.ConvTrainGrads(*[C.cast(a, _capi._fpp) for a in ptrs])
    assert _capi.lib.icnn_conv_train_grad(net._h, C.byref(fg.c_gates), off, None, None, None, C.byref(gr),
                                          C.c_void_p(16), None) == -1
    assert b"row_offsets decreasing" in _capi.lib.icnn_last_error()
