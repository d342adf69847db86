"""The bundle-entropy training gradient d (sum_r F_r) / d theta on the GPU (icnn_train_grad, icnn_b200.bundle_grad)
against the reference's own Model on the TF shim (tests/golden/training/bundle_grad.npz) and the float64 oracle
(oracle/bundle_grad_np.py) on the solver's own device state.

Tolerance: the device path is float32 (3xTF32 wgmma or FFMA GEMMs, float32 sums over rows and samples); every
array must agree to RTOL = 2e-4 of its largest entry (test_gpu_gd_grad's tolerance).  A float32 evaluation of a row
whose pre-activation sits within 1e-5 (relative) of zero can land on the other side of the ReLU kink and change
that sample's gradient by O(1): such a sample may be set aside only when it disagrees AND the float64 oracle shows
such a pre-activation at one of its rows, at most max(1, 2 %) of the samples; the rest is compared again without it."""
import os

import numpy as np
import pytest

from oracle import bundle_grad_np as bg
from icnn_b200.workloads import make_inputs, synth_params

pytestmark = pytest.mark.gpu
np.seterr(all="ignore")

RTOL = 2e-4
KINK = 1e-5
PARAMS = ("Wy", "Wz", "Wu", "bu", "Wzu", "bzu", "Wyu", "byu", "Wzx", "bzx")


def relerr(a, b):
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(np.asarray(a, dtype=np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def _rows_mask(counts, keep):
    return np.repeat(keep, counts)


def _set_aside(fg, p, x, Y, V, c, counts):
    """Runs device and oracle; returns (device grads, oracle grads, kept-sample mask) after setting aside the samples
    the kink rule allows (and asserting nothing else disagrees)."""
    from icnn_b200.bundle_grad import train_grad
    B = len(counts)
    dev = train_grad(fg, Y, V, c, counts, x=x)
    orc = bg.bundle_grad(p, x, Y, V, c, counts, per_sample=False)
    bad = np.zeros(B, dtype=bool)
    for k in ("dcy", "dcz", "dd"):
        for a, b in zip(dev[k], orc[k]):
            if b is not None:
                bad |= np.abs(a - b).max(axis=1) / max(np.abs(b).max(), 1e-30) >= RTOL
    near = bg.min_rel_preact(p, x, Y, counts) < KINK
    kink = np.zeros(B, dtype=bool)
    np.logical_or.at(kink, np.repeat(np.arange(B), counts), near)
    assert not (bad & ~kink).any(), np.nonzero(bad & ~kink)[0]
    drop = bad & kink
    assert drop.sum() <= max(1, int(0.02 * B)), (int(drop.sum()), B)
    keep = ~drop
    if drop.any():
        rows = _rows_mask(counts, keep)
        counts = np.where(keep, counts, 0)
        Y, V, c = Y[rows], V[rows], c[rows]
        dev = train_grad(fg, Y, V, c, counts, x=x)
        orc = bg.bundle_grad(p, x, Y, V, c, counts, per_sample=False)
    return dev, orc, keep


def _assert_close(dev, ref, names, tag):
    errs = {}
    for k in names:
        for i, b in enumerate(ref[k]):
            if b is not None:
                errs["%s%d" % (k, i)] = relerr(dev[k][i], b)
    worst = max(errs, key=errs.get)
    print(tag, "max rel err %.2e (%s)" % (errs[worst], worst))
    assert errs[worst] < RTOL, errs


@pytest.mark.parametrize("tag", ["small", "c3"])
@pytest.mark.parametrize("loss", ["xent", "mse"])
def test_reference_golden_rows(tag, loss, golden_dir):
    """The golden's own train_step_fd rows through train_grad; every stored array, summed over the samples kept."""
    import icnn_b200
    from oracle.gen_golden_bundle_grad import case_inputs
    gold = np.load(os.path.join(golden_dir, "training", "bundle_grad.npz"))
    p, x, _y0, _tY, _n, _s = case_inputs(tag)
    key = "%s_%s_" % (tag, loss)
    counts = gold[tag + "_counts"]
    fg = icnn_b200.PICNN.from_params(p).bind(x)
    dev, _orc, keep = _set_aside(fg, p, x, gold[key + "Y"], gold[key + "V"], gold[key + "c"], counts)
    stored = [k for k in gold.files if k.startswith(key + "grad_")]
    assert stored
    errs = {}
    for k in stored:
        name = k[len(key + "grad_"):]
        pname = name.rstrip("0123456789")
        ref = gold[k][keep].sum(0)
        errs[name] = relerr(dev[pname][int(name[len(pname):])], ref)
    worst = max(errs, key=errs.get)
    print(tag, loss, "samples kept %d/%d, max rel err %.2e (%s)" % (keep.sum(), len(keep), errs[worst], worst))
    assert errs[worst] < RTOL, errs


def _state_case(case, loss, seed=17):
    """Solve on the device, K3 on the device state; returns (fg, p, x, st, rows Y/V/c in float32, counts) with the
    samples whose KKT matrix is numerically singular (cond > 1e9) removed from the rows up front."""
    import icnn_b200
    from icnn_b200 import argmin_grad, bundle_entropy as be
    name, B, nIter = case
    if name in ("C3", "T"):
        p, x, y0 = make_inputs(name, B=B)
    else:
        m, n, hidden, alpha = name
        p = synth_params(seed, m, n, hidden, alpha=alpha)
        for i in range(len(p.Wy)):
            p.Wy[i] = (p.Wy[i].astype(np.float32) * np.float32(3.0)).astype(np.float64)
        x = np.random.RandomState(seed).randn(B, m).astype(np.float32).astype(np.float64)
        y0 = np.full((B, n), 0.5)
    fg = icnn_b200.PICNN.from_params(p).bind(x)
    yN, G, h, lam, ys, nIters, st = be.solveBatch(fg, y0.copy(), nIter=nIter, return_state=True)
    trueY = (np.random.RandomState(seed).uniform(size=yN.shape) < 0.3).astype(np.float64)
    _cy, _clam, _ct, (fY, fV, fc) = argmin_grad.argmin_grad(st, trueY, loss=loss)
    counts = np.array([len(G[u]) for u in range(B)])
    good = np.ones(B, dtype=bool)
    for u in range(B):
        Gu = np.array(G[u], dtype=np.float64)
        if len(Gu) == 0:
            continue
        yc = np.clip(yN[u], 1e-8, 1 - 1e-8)
        zinv = 1.0 / (1.0 / yc + 1.0 / (1.0 - yc))
        good[u] = np.linalg.cond((Gu * zinv).dot(Gu.T)) <= 1e9
    assert good.mean() >= 0.5
    rows = _rows_mask(counts, good)
    f32 = lambda a: np.asarray(a, dtype=np.float32).astype(np.float64)   # noqa: E731
    return fg, p, x, st, trueY, f32(fY[rows]), f32(fV[rows]), f32(fc[rows]), np.where(good, counts, 0)


STATE_CASES = {
    "c3": ("C3", 256, 10),
    "t": ("T", 128, 8),
    "leaky": ((20, 16, [48, 32], 0.01), 100, 10),
    "odd3": ((12, 37, [50, 21, 33], 0.0), 77, 10),
    "ffma": ((8, 6, [12, 10], 0.0), 6, 6),        # fewer than 64 rows: the FFMA path
}


@pytest.mark.parametrize("case", list(STATE_CASES))
@pytest.mark.parametrize("loss", ["xent", "mse"])
def test_device_state_matches_oracle(case, loss):
    fg, p, x, _st, _tY, Y, V, c, counts = _state_case(STATE_CASES[case], loss)
    if case == "ffma":
        assert len(Y) < 64
    dev, orc, keep = _set_aside(fg, p, x, Y, V, c, counts)
    print(case, loss, "rows", len(Y), "samples kept", int(keep.sum()), "of", len(keep))
    _assert_close(dev, orc, PARAMS + ("dcy", "dcz", "dd"), case)


def test_bundle_grad_is_train_grad_on_the_assembled_rows():
    from icnn_b200 import argmin_grad
    from icnn_b200.bundle_grad import bundle_grad, train_grad
    fg, p, x, st, tY, *_ = _state_case(("C3", 64, 10), "xent")
    a = bundle_grad(fg, st, tY, loss="xent", x=x)
    _cy, clam, _ct, (fY, fV, fc) = argmin_grad.argmin_grad(st, tY, loss="xent")
    b = train_grad(fg, fY, fV, fc, [len(v) for v in clam], x=x)
    assert set(a) == set(b)
    for k in a:
        for u, v in zip(a[k], b[k]):
            if u is not None:
                np.testing.assert_array_equal(u, v, err_msg=k)


def test_deterministic_paths_and_chunking(monkeypatch):
    """Two calls are bit-identical; the FFMA kernels (ICNN_GDB=simt) agree with the tensor-core path to 5e-5, and a
    forced small chunk size agrees with the default to 1e-6 (the weight gradients are summed over rows and chunks in
    float64, so where the chunks are cut does not matter beyond the final rounding).  Same sample set as the oracle
    comparisons: KKT cond <= 1e9, and the kink rule (a sample sitting on a ReLU kink, where float32 evaluations of
    its pre-activations are unstable, may be set aside)."""
    from icnn_b200.bundle_grad import bundle_grad, train_grad
    fg, p, x, st, tY, Y, V, c, counts = _state_case(("C3", 128, 10), "mse")
    monkeypatch.delenv("ICNN_GDB", raising=False)
    monkeypatch.delenv("ICNN_TRAIN_CHUNK", raising=False)
    a = bundle_grad(fg, st, tY, loss="mse", x=x)
    b = bundle_grad(fg, st, tY, loss="mse", x=x)
    for k in a:
        for u, v in zip(a[k], b[k]):
            if u is not None:
                np.testing.assert_array_equal(u, v, err_msg=k)
    _dev, _orc, keep = _set_aside(fg, p, x, Y, V, c, counts)
    rows = _rows_mask(counts, keep)
    Y, V, c, counts = Y[rows], V[rows], c[rows], np.where(keep, counts, 0)
    assert len(Y) > 600
    base = train_grad(fg, Y, V, c, counts, x=x)
    monkeypatch.setenv("ICNN_TRAIN_CHUNK", "256")      # several chunks of >= 64 rows: still the tensor-core path
    s = train_grad(fg, Y, V, c, counts, x=x)
    monkeypatch.setenv("ICNN_GDB", "simt")
    monkeypatch.delenv("ICNN_TRAIN_CHUNK")
    f = train_grad(fg, Y, V, c, counts, x=x)
    errs = {}
    for k in base:
        for i, (u, v, w) in enumerate(zip(base[k], s[k], f[k])):
            if u is not None:
                errs["%s%d" % (k, i)] = (relerr(v, u), relerr(w, u))
    print("chunked max %.2e, ffma max %.2e" % (max(e[0] for e in errs.values()), max(e[1] for e in errs.values())))
    for name, (ec, ef) in errs.items():
        assert ec < 1e-6, ("chunked", name, ec)
        assert ef < 5e-5, ("ffma", name, ef)


def test_sample_split_across_chunks(monkeypatch):
    """A sample with more rows than a chunk holds is split over chunks; its per-sample outputs are summed over them."""
    from icnn_b200.bundle_grad import train_grad
    fg, p, x, st, tY, Y, V, c, counts = _state_case(STATE_CASES["ffma"], "xent")
    assert counts.max() >= 2
    monkeypatch.delenv("ICNN_TRAIN_CHUNK", raising=False)
    base = train_grad(fg, Y, V, c, counts, x=x)
    monkeypatch.setenv("ICNN_TRAIN_CHUNK", "1")        # every sample with two or more rows is split
    s = train_grad(fg, Y, V, c, counts, x=x)
    for k in base:
        for i, (u, v) in enumerate(zip(base[k], s[k])):
            if u is not None:
                assert relerr(v, u) < 1e-6, (k, i, relerr(v, u))


def test_zero_inputs_and_empty_samples():
    import icnn_b200
    from icnn_b200.bundle_grad import train_grad
    p, x, _y0 = make_inputs("C1", B=8)
    fg = icnn_b200.PICNN.from_params(p).bind(x)
    rs = np.random.RandomState(3)
    counts = np.array([3, 0, 2, 0, 1, 4, 0, 2])
    R = int(counts.sum())
    Y = rs.uniform(0.05, 0.95, size=(R, p.n))
    g0 = train_grad(fg, Y, np.zeros((R, p.n)), np.zeros(R), counts, x=x)
    assert all(not np.any(a) for v in g0.values() for a in v if a is not None)
    g = train_grad(fg, Y, rs.randn(R, p.n), rs.randn(R), counts, x=x)
    for k in ("dcy", "dcz", "dd"):
        for a in g[k]:
            if a is not None:
                assert not np.any(a[counts == 0]) and np.any(a[counts > 0])
    ge = train_grad(fg, np.zeros((0, p.n)), np.zeros((0, p.n)), np.zeros(0), np.zeros(8, dtype=int), x=x)
    assert all(not np.any(a) for v in ge.values() for a in v if a is not None)


def test_errors():
    import icnn_b200
    from icnn_b200 import bundle_entropy as be
    from icnn_b200.bundle_grad import bundle_grad, train_grad
    p, x, y0 = make_inputs("C1", B=8)
    net = icnn_b200.PICNN.from_params(p)
    fg = net.bind(x)
    tY = np.zeros_like(y0)
    *_, st = be.solveBatch(fg, y0.copy(), nIter=3, return_state=True)
    with pytest.raises(TypeError):
        bundle_grad(lambda y: y, st, tY)
    with pytest.raises(TypeError):
        train_grad(lambda y: y, y0, y0, np.zeros(8), np.ones(8, dtype=int))
    with pytest.raises(ValueError):
        bundle_grad(net.bind(x, affine=True), st, tY)
    with pytest.raises(ValueError):
        train_grad(net.bind(x, affine=True), y0, y0, np.zeros(8), np.ones(8, dtype=int))
    with pytest.raises(ValueError):
        bundle_grad(net.bind(x[:4]), st, tY)                         # B does not match the state
    p2, x2, y2 = make_inputs("C1", B=8)
    p2.n, p2.Wy = 7, [w[:7] for w in p2.Wy]
    p2.Wyu, p2.byu = [w[:, :7] for w in p2.Wyu], [b[:7] for b in p2.byu]
    with pytest.raises(ValueError):
        bundle_grad(icnn_b200.PICNN.from_params(p2).bind(x2), st, tY)   # n does not match the state
    *_, st_noxs = be.solveBatch(fg, y0.copy(), nIter=3, return_state=True, keep_xs=False)
    with pytest.raises(ValueError):
        bundle_grad(fg, st_noxs, tY)
    with pytest.raises(ValueError):
        train_grad(fg, y0, y0, np.zeros(8), np.ones(7, dtype=int))
