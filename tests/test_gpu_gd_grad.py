"""d mse / d theta through the unrolled momentum-GD loop (multi-label-cls/icnn-back.py:116-139) on the
GPU vs the torch-autograd golden vectors and the float64 numpy restatement.

Tolerance: the device path is float32 (3xTF32 wgmma or FFMA GEMMs, float32 accumulation over the
batch and the nIter iterations); every gradient array must agree with the float64 reference to 2e-4
of that array's largest entry on the samples whose iterates cross no ReLU kink differently."""
import os

import numpy as np
import pytest

from oracle import gd_grad_np, picnn_np, synth
from icnn_b200.workloads import synth_params

pytestmark = pytest.mark.gpu

RTOL = 2e-4


def relerr(a, b):
    return float(np.abs(np.asarray(a, dtype=np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def test_matches_autograd_golden(golden_dir):
    import icnn_b200
    from oracle.gen_golden_gd_grad import CASES, true_labels
    gold = np.load(os.path.join(golden_dir, "gd_grad.npz"))
    for tag, (name, B, nIter, lr, mom) in CASES.items():
        p, x, y0 = synth.make_inputs(name, B=B)
        tY = true_labels(B, p.n)
        net = icnn_b200.PICNN.from_params(p)
        yN, gr = icnn_b200.gd_grad.gd_grad(net.bind(x), y0, tY, nIter=nIter, lr=lr, momentum=mom, x=x)
        assert np.abs(yN - gold[tag + "_yN"]).max() < 2e-5
        worst = {}
        for k in ("Wy", "Wz", "Wu", "bu", "Wzu", "bzu", "Wyu", "byu"):
            for i, g in enumerate(gr[k]):
                key = "%s_%s%d" % (tag, k, i)
                if g is None:
                    assert key not in gold.files
                    continue
                worst[key] = relerr(g, gold[key])
        print(tag, "max rel err", max(worst.values()), max(worst, key=worst.get))
        assert max(worst.values()) < RTOL, worst


def _dims_case(m, n, hidden, B, seed):
    p = synth_params(seed, m, n, hidden)
    for i in range(len(p.Wy)):
        p.Wy[i] = (p.Wy[i].astype(np.float32) * np.float32(3.0)).astype(np.float64)
    rs = np.random.RandomState(seed + 1)
    x = rs.randn(B, m).astype(np.float32).astype(np.float64)
    y0 = np.full((B, n), 0.5)
    tY = (rs.uniform(size=(B, n)) < 0.2).astype(np.float64)
    return p, x, y0, tY


@pytest.mark.parametrize("dims,B,nIter,lr,mom", [
    ((1836, 159, [600, 159]), 512, 30, 0.01, 0.3),     # C3 dims, the multi-label script's defaults
    ((64, 512, [1024, 1024]), 200, 6, 0.01, 0.9),      # wide layers: split-K clusters in every GEMM
    ((12, 37, [50, 21, 33]), 77, 10, 0.02, 0.5),       # odd widths, three hidden layers, ragged tiles
])
def test_matches_oracle(dims, B, nIter, lr, mom):
    """A float32 / 3xTF32 iterate that lands on the other side of a ReLU kink changes that sample's
    gradient by O(1) for a step (the sensitivity DESIGN.md section 4 describes for the bundle path;
    reproduced inside the float64 oracle by a 5e-6 relative perturbation of W^y: 3 of 200 rows move,
    parameter gradients by 1e-2).  Such rows are identified from y_N and the per-sample gate adjoints
    (<= 2 % of the batch), dropped from the minibatch, and both sides are run again: on the remaining
    rows every gradient array must agree to RTOL of its largest entry."""
    import icnn_b200
    m, n, hidden = dims
    p, x, y0, tY = _dims_case(m, n, hidden, B, seed=21)
    net = icnn_b200.PICNN.from_params(p)
    keep = np.arange(B)
    dropped = 0
    for attempt in range(4):
        xs, ys, ts = x[keep], y0[keep], tY[keep]
        scale = 2.0 / tY.size          # the same loss weight per sample on every attempt
        yo, go = gd_grad_np.gd_backward(p, picnn_np.gates(p, xs), ys, nIter, lr, mom, lambda y: scale * (y - ts))
        xo = gd_grad_np.xpath_backward(p, xs, go["dcy"], go["dcz"])
        yN, gr = icnn_b200.gd_grad.gd_grad(net.bind(xs), ys, ts, nIter=nIter, lr=lr, momentum=mom, x=xs,
                                           loss_scale=scale)
        bad = np.abs(yN - yo).max(axis=1) >= 1e-4
        for l in range(p.L + 1):
            for k in ("dcy", "dcz"):
                if go[k][l] is not None:
                    d = np.abs(gr[k][l].astype(np.float64) - go[k][l]).max(axis=1) / max(np.abs(go[k][l]).max(), 1e-30)
                    bad |= d >= RTOL
        if not bad.any():
            break
        dropped += int(bad.sum())
        keep = keep[~bad]
    assert not bad.any() and dropped <= 0.02 * B, (dropped, B)
    # the rows set aside are not a free pass: the float64 oracle itself must lose at least as many rows (minus
    # one) under a float32-sized (1e-7 relative) perturbation of W^y -- the kink flips are a property of the
    # iteration, not of the device arithmetic (VERDICT r01, parity item 3)
    if dropped:
        import copy
        rs = np.random.RandomState(99)
        floor = 0
        for rep in range(3):
            pp = copy.deepcopy(p)
            for i in range(len(pp.Wy)):
                pp.Wy[i] = pp.Wy[i] * (1.0 + 1e-7 * rs.choice([-1.0, 1.0], size=pp.Wy[i].shape))
            scale = 2.0 / tY.size
            y1, g1 = gd_grad_np.gd_backward(p, picnn_np.gates(p, x), y0, nIter, lr, mom, lambda y: scale * (y - tY))
            y2, g2 = gd_grad_np.gd_backward(pp, picnn_np.gates(pp, x), y0, nIter, lr, mom, lambda y: scale * (y - tY))
            moved = np.abs(y1 - y2).max(axis=1) >= 1e-4
            for l in range(p.L + 1):
                for k in ("dcy", "dcz"):
                    if g1[k][l] is not None:
                        moved |= (np.abs(g1[k][l] - g2[k][l]).max(axis=1) / max(np.abs(g1[k][l]).max(), 1e-30)) >= RTOL
            floor = max(floor, int(moved.sum()))
        print("oracle rows moved by a 1e-7 perturbation of W^y: %d (device: %d set aside)" % (floor, dropped))
        assert dropped <= floor + 1, (dropped, floor)
    assert np.median(np.abs(yN - yo).max(axis=1)) < 2e-6
    errs = {}
    for l in range(p.L + 1):
        errs["Wy%d" % l] = relerr(gr["Wy"][l], go["dWy"][l])
        errs["Wyu%d" % l] = relerr(gr["Wyu"][l], xo["dWyu"][l])
        if l > 0:
            errs["Wz%d" % l] = relerr(gr["Wz"][l], go["dWz"][l])
            errs["Wzu%d" % l] = relerr(gr["Wzu"][l], xo["dWzu"][l])
    for l in range(p.L):
        errs["Wu%d" % l] = relerr(gr["Wu"][l], xo["dWu"][l])
    print(dims, "rows dropped (kink flips)", dropped, "of", B, "param max rel err %.2e" % max(errs.values()),
          max(errs, key=errs.get))
    assert max(errs.values()) < RTOL, errs


def test_ffma_and_tensor_core_paths_agree(monkeypatch):
    """ICNN_GDB=simt keeps the three gated products on the FP32 FFMA kernel (the accuracy anchor)."""
    import icnn_b200
    p, x, y0, tY = _dims_case(40, 64, [96, 80], 256, seed=5)
    fg = icnn_b200.PICNN.from_params(p).bind(x)
    y_tc, g_tc = icnn_b200.gd_grad.gd_grad(fg, y0, tY, nIter=5, lr=0.02, momentum=0.5)
    monkeypatch.setenv("ICNN_GDB", "simt")
    y_ff, g_ff = icnn_b200.gd_grad.gd_grad(fg, y0, tY, nIter=5, lr=0.02, momentum=0.5)
    assert np.abs(y_tc - y_ff).max() < 1e-5
    for k in ("Wy", "Wz", "dcy", "dcz"):
        for a, b in zip(g_tc[k], g_ff[k]):
            if a is not None:
                assert relerr(a, b.astype(np.float64)) < 5e-5, k


def test_single_pass_and_two_pass_modes_agree(monkeypatch):
    """Default on the tensor-core path: ONE pass over the GD loop with every iteration's activation
    patterns / deltas kept in HBM and the tangent work batched over the iterations; ICNN_GDB=twopass
    replays the loop instead (the mode used when the stores exceed ICNN_GDB_STORE_GB)."""
    import icnn_b200
    for dims, B, nIter in (((40, 64, [96, 80]), 256, 5), ((20, 37, [50, 21, 33]), 100, 7), ((16, 24, [40]), 64, 3)):
        p, x, y0, tY = _dims_case(*dims, B, seed=5)
        fg = icnn_b200.PICNN.from_params(p).bind(x)
        monkeypatch.delenv("ICNN_GDB", raising=False)
        y_a, g_a = icnn_b200.gd_grad.gd_grad(fg, y0, tY, nIter=nIter, lr=0.02, momentum=0.5)
        monkeypatch.setenv("ICNN_GDB", "twopass")
        y_b, g_b = icnn_b200.gd_grad.gd_grad(fg, y0, tY, nIter=nIter, lr=0.02, momentum=0.5)
        monkeypatch.delenv("ICNN_GDB")
        np.testing.assert_array_equal(y_a, y_b)          # the same primal kernels in both modes
        for k in ("Wy", "Wz", "dcy", "dcz"):
            for a, b in zip(g_a[k], g_b[k]):
                if a is not None:
                    assert relerr(a, b.astype(np.float64)) < 2e-5, (dims, k)


def test_yn_is_the_gd_solve_iterate():
    import icnn_b200
    p, x, y0 = synth.make_inputs("C3", B=128)
    tY = np.zeros_like(y0)
    fg = icnn_b200.PICNN.from_params(p).bind(x)
    yN, _ = icnn_b200.gd_grad.gd_grad(fg, y0, tY, nIter=30)
    ys, _ = icnn_b200.gd.solve(fg, y0, nIter=30)
    assert np.abs(yN - ys).max() < 1e-4


def test_zero_iterations_and_errors():
    import icnn_b200
    p, x, y0 = synth.make_inputs("C1", B=8)
    net = icnn_b200.PICNN.from_params(p)
    yN, gr = icnn_b200.gd_grad.gd_grad(net.bind(x), y0, np.zeros_like(y0), nIter=0)
    np.testing.assert_array_equal(yN, y0.astype(np.float32))
    assert all(not np.any(g) for g in gr["Wy"])
    with pytest.raises(ValueError):
        icnn_b200.gd_grad.gd_grad(net.bind(x, affine=True), y0, y0)
    with pytest.raises(TypeError):
        icnn_b200.gd_grad.gd_grad(lambda y: y, y0, y0)


def test_make_cvx_and_proj():
    import torch
    from icnn_b200.gd_grad import make_cvx, proj
    w = [None, torch.tensor([[-1.0, 2.0], [0.5, -4.0]])]
    np.testing.assert_array_equal(proj([None, w[1].clone()])[1].numpy(), [[0, 2], [0.5, 0]])
    np.testing.assert_array_equal(make_cvx([None, w[1].clone()])[1].numpy(), [[1, 2], [0.5, 4]])
    np.testing.assert_array_equal(make_cvx([None, w[1].clone()], halve=True)[1].numpy(), [[0.5, 1], [0.25, 2]])
    np.testing.assert_allclose(make_cvx([None, w[1].clone()], divide=10)[1].numpy(), [[0.1, 0.2], [0.05, 0.4]], rtol=1e-6)


def test_in_place_weight_updates_must_be_repacked():
    """The device library keeps packed / TF32-split copies of the weights: after an in-place update of the torch
    tensors (optimiser step, make_cvx / proj) bind() refuses to run on the stale copies, and
    update_weights() makes K1, the gate GEMMs and the torch-side x-path agree again (ADVICE r01)."""
    import icnn_b200
    from icnn_b200.gd_grad import proj
    p, x, y0, tY = _dims_case(40, 64, [96, 80], 128, seed=9)
    net = icnn_b200.PICNN.from_params(p)
    y = np.random.RandomState(1).uniform(0.1, 0.9, size=y0.shape)
    f0, _ = net.bind(x)(y)
    net.Wz[1].mul_(-1.0)            # in-place change ...
    proj(net.Wz)                    # ... and projection: Wz[1] is now all zeros
    with pytest.raises(RuntimeError, match="update_weights"):
        net.bind(x)
    net.update_weights()
    f1, _ = net.bind(x)(y)
    p.Wz[1] = np.zeros_like(p.Wz[1])
    fo, _ = picnn_np.make_fg(p, x)(y)
    assert np.abs(f1 - fo).max() <= 1e-5 * max(1.0, np.abs(fo).max()) and np.abs(f1 - f0).max() > 1e-3
