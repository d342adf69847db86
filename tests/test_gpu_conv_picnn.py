"""The convolutional PICNN of the image-completion experiment on the device (icnn_b200.ConvPICNN, conv_picnn.cu):
f and df/dy against the reference's own graph and the float64 helper, the bundle-slot writes, the fused bundle loop
against callback mode and the float64 oracle, momentum GD, determinism and the stale-weight check.

Accuracy criterion for f and g: max |device - float64| <= max(4 x the same error of the network evaluated in torch
float32 with TF32 off, 1e-6 x max |float64|)."""
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import bundle_np, conv_energy
from oracle import conv_picnn as helper

pytestmark = pytest.mark.gpu
np.seterr(all="ignore")

HERE = os.path.dirname(os.path.abspath(__file__))

PINS = [(-1, -1), (0, 1), (1, 1), (2, 1), (1, 2), (1, 4), (1, 8)]     # (cfg, splitk) of icnn_tc_set_tuning


@pytest.fixture(autouse=True)
def automatic_tuning():
    yield
    from icnn_b200 import _capi
    assert _capi.lib.icnn_tc_set_tuning(-1, -1, -1) == 0


def _pin(cfg, splitk):
    from icnn_b200 import _capi
    assert _capi.lib.icnn_tc_set_tuning(cfg, splitk, -1) == 0


def _no_tf32():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _check(tag, f, g, f64, g64, f32, g32):
    for name, dev, ref, t32 in (("f", f, f64, f32), ("g", g, g64, g32)):
        err = np.abs(dev.astype(np.float64) - ref).max()
        e32 = np.abs(t32.astype(np.float64) - ref).max()
        tol = max(4 * e32, 1e-6 * np.abs(ref).max())
        print("%s %s: device err %.2e, torch float32 err %.2e, tol %.2e" % (tag, name, err, e32, tol))
        assert err <= tol, (tag, name, err, e32, tol)


def _golden_cases():
    from oracle.gen_golden_conv import case
    from oracle.gen_golden_tfshim import conv_case, conv_variables
    g1 = np.load(os.path.join(HERE, "golden", "picnn_tfshim.npz"))
    g2 = np.load(os.path.join(HERE, "golden", "conv", "conv_picnn.npz"))
    out = []
    for tag in ("conv_small", "conv_olivetti"):
        net, x, y = conv_case(tag)
        out.append((tag, conv_variables(net), x, y, net.H, net.W, g1[tag + "_f"], g1[tag + "_g"]))
    for tag in ("conv_bn_olivetti", "conv_bn_odd"):
        v, x, y, H, W = case(tag)
        out.append((tag, v, x, y, H, W, g2[tag + "_f"], g2[tag + "_g"]))
    return out


@pytest.mark.parametrize("pin", PINS, ids=["auto", "128x3", "64x4", "64x2", "64x4s2", "64x4s4", "64x4s8"])
def test_fg_matches_the_reference_graph(pin):
    """E_ / dE_dy_ of the reference's completion Model run on the TF stand-in, from the exact variable dict it ran
    on, under every tile variant and split-K factor of the GEMM."""
    import icnn_b200
    from icnn_b200.conv_picnn import parse_variables
    _no_tf32()
    _pin(*pin)
    for tag, v, x, y, H, W, fr, gr in _golden_cases():
        net = icnn_b200.ConvPICNN.from_variables(v, H, W)
        f, g = net.bind(x)(y)
        f32, g32 = conv_energy.fg(parse_variables(v, H, W), x, y, dtype=torch.float32, device="cuda")
        _check("%s %s" % (tag, pin), f, g, fr, gr, f32, g32)


def _helper_case(H, W, B, seed=4):
    from oracle.gen_golden_tfshim import conv_variables
    net64 = helper.ConvPICNN(H, W, seed=seed, dtype=torch.float64, device="cuda")
    rs = np.random.RandomState(B + H)
    x, y = rs.uniform(size=(B, H * W)), rs.uniform(0.05, 0.95, size=(B, H * W))
    return net64, conv_variables(net64.to(torch.float64, "cpu")), x, y


def _helper_check(H, W, B):
    import icnn_b200
    _no_tf32()
    net64, v, x, y = _helper_case(H, W, B)
    f64, g64 = net64.make_fg(x)(y)
    f32, g32 = net64.to(torch.float32, "cuda").make_fg(x)(y)
    f, g = icnn_b200.ConvPICNN.from_variables(v, H, W).bind(x)(y)
    _check("%dx%d B=%d" % (H, W, B), f, g, f64, g64, f32, g32)


@pytest.mark.parametrize("B", [1, 3, 64, 65, 400])
@pytest.mark.parametrize("H,W", [(16, 8), (64, 32), (17, 9)])
def test_fg_shapes_match_the_float64_helper(H, W, B):
    _helper_check(H, W, B)


@pytest.mark.parametrize("H,W,B", [(16, 8, 5), (17, 9, 70), (64, 32, 3)])
def test_fg_other_architecture(monkeypatch, H, W, B):
    """A second architecture (two convs, C = 8 and 16, dense 32 -> 1): the handle takes it from the variables."""
    monkeypatch.setattr(helper, "CONVS", ((8, 4, 2), (16, 3, 1)))
    monkeypatch.setattr(helper, "FCS", (32, 1))
    _helper_check(H, W, B)


def test_slot_writes_and_skip():
    """g written through perm / count into a bundle slot equals the dense fg bit for bit; with *skip_if_zero == 0
    neither f nor the slot is touched."""
    import ctypes as C
    import icnn_b200
    from icnn_b200 import _capi
    _net64, v, x, y = _helper_case(64, 32, 65)
    fg = icnn_b200.ConvPICNN.from_variables(v, 64, 32).bind(x)
    y32 = torch.as_tensor(y, dtype=torch.float32, device="cuda")
    f0, g0 = fg.fg_device(y32)
    B, n, KS = 65, 64 * 32, 5
    rs = np.random.RandomState(1)
    perm = torch.as_tensor(np.stack([rs.permutation(KS) for _ in range(B)]), dtype=torch.int32, device="cuda")
    count = torch.as_tensor(rs.randint(0, KS, size=B), dtype=torch.int32, device="cuda")
    G = torch.full((B, KS, n), 7.0, device="cuda")
    f = torch.full((B,), 3.0, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(skip):
        _capi.check(_capi.lib.icnn_conv_picnn_fg(fg.net._h, C.byref(fg.c_gates), y32.data_ptr(), f.data_ptr(),
                                                  G.data_ptr(), 0, perm.data_ptr(), count.data_ptr(), KS,
                                                  fg.ws.data_ptr(), skip, stream))
    zero = torch.zeros(1, dtype=torch.int32, device="cuda")
    call(zero.data_ptr())
    assert bool((f == 3.0).all()) and bool((G == 7.0).all())
    call(None)
    slot = perm[torch.arange(B, device="cuda"), count.long()].long()
    assert torch.equal(G[torch.arange(B, device="cuda"), slot], g0) and torch.equal(f, f0)
    mask = torch.ones(B, KS, dtype=torch.bool, device="cuda")
    mask[torch.arange(B, device="cuda"), slot] = False
    assert bool((G[mask] == 7.0).all())


def test_fused_equals_callback_mode():
    """solveBatch fused (one C call) and callback mode driven by the handle's own numpy fg give the same bits."""
    import icnn_b200
    from icnn_b200 import bundle_entropy as be
    _net64, v, x, _y = _helper_case(64, 32, 64)
    fg = icnn_b200.ConvPICNN.from_variables(v, 64, 32).bind(x)
    y0 = np.tile(np.random.RandomState(2).uniform(0.2, 0.8, size=(1, 64 * 32)), (64, 1))
    tol = 1e-9
    a = be.solveBatch(fg, y0.copy(), nIter=10, rank_tol=tol)
    b = be.solveBatch(lambda y: fg(y), y0.copy(), nIter=10, rank_tol=tol)
    assert np.array_equal(a[0], b[0]) and a[5] == b[5]
    for u in range(64):
        assert np.array_equal(np.array(a[1][u]), np.array(b[1][u])) and a[2][u] == b[2][u]
        assert np.array_equal(a[3][u], b[3][u]) and np.array_equal(np.array(a[4][u]), np.array(b[4][u]))
    with pytest.raises(ValueError, match="graph"):
        be.solveBatch(fg, y0.copy(), nIter=2, graph=True)


def test_full_size_subsample_matches_oracle():
    """C2-conv: B = 400 at 64 x 32, 30 iterations; a random subsample against the float64 oracle (oracle/bundle_np
    driven by the float64 helper), with the floor of test_gpu_bundle.py::test_full_size_subsample_matches_oracle: the
    larger of the oracle's own float32 floor (the same solve driven by the helper in float32 with TF32 off) and the
    float64 oracle under 2e-6 relative noise on (f, g).  Over 30 iterations the iterates settle on ReLU kinks of the
    piecewise-linear f, so a sample either agrees to ~1e-6 or moves by ~1e-3; the test bounds how many move."""
    import icnn_b200
    from icnn_b200 import bundle_entropy as be
    _no_tf32()
    B, H, W, nIter, nsub = 400, 64, 32, 30, 48
    from oracle.gen_golden_tfshim import conv_variables
    net64 = helper.ConvPICNN(H, W, seed=2, dtype=torch.float64, device="cuda")
    rs = np.random.RandomState(0)
    x = rs.uniform(size=(B, H * W))
    y0 = np.tile(rs.uniform(0.2, 0.8, size=(1, H * W)), (B, 1))
    fg = icnn_b200.ConvPICNN.from_variables(conv_variables(net64.to(torch.float64, "cpu")), H, W).bind(x)
    r = be.solveBatch(fg, y0.copy(), nIter=nIter)
    rows = np.sort(np.random.RandomState(7).choice(B, size=nsub, replace=False))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        fg64 = net64.make_fg(x[rows])
        o = bundle_np.solve_batch(fg64, y0[rows].copy(), nIter=nIter)
        fg32 = net64.to(torch.float32, "cuda").make_fg(x[rows])
        o32 = bundle_np.solve_batch(lambda y: tuple(a.astype(np.float64) for a in fg32(y)), y0[rows].copy(), nIter=nIter)
        rsn = np.random.RandomState(123)

        def fg_noisy(y):
            f, g = fg64(y)
            return f * (1.0 + 2e-6 * rsn.randn(*f.shape)), g * (1.0 + 2e-6 * rsn.randn(*g.shape))
        on = bundle_np.solve_batch(fg_noisy, y0[rows].copy(), nIter=nIter)
    d = np.abs(r[0][rows] - o[0]).max(axis=1)
    floor32 = np.abs(o32[0] - o[0]).max(axis=1)
    floorn = np.abs(on[0] - o[0]).max(axis=1)
    floor = floorn if np.mean(floorn > 1e-4) > np.mean(floor32 > 1e-4) else floor32
    print("C2-conv subsample: device-vs-oracle max %.2e median %.2e frac>1e-4 %.3f | float32 floor median %.2e "
          "frac>1e-4 %.3f | 2e-6 noise floor median %.2e frac>1e-4 %.3f"
          % (d.max(), np.median(d), np.mean(d > 1e-4), np.median(floor32), np.mean(floor32 > 1e-4),
             np.median(floorn), np.mean(floorn > 1e-4)))
    assert np.mean(d > 1e-4) <= np.mean(floor > 1e-4) + max(0.02, 2.5 / nsub)
    assert np.median(d) <= max(1e-5, 4 * np.median(floor))
    assert d.max() <= 4 * max(floor32.max(), floorn.max())


def test_momentum_gd_matches_float64():
    """gd.solve(fg, y0, 30, lr=.01, momentum=.9) against a float64 torch momentum GD on the helper, within the
    float32 floor (the same loop on the float32 helper)."""
    import icnn_b200
    from icnn_b200 import gd
    _no_tf32()
    net64, v, x, _y = _helper_case(64, 32, 32)
    y0 = np.random.RandomState(3).uniform(0.2, 0.8, size=(32, 64 * 32))

    def loop(fgf, dtype):
        y = torch.as_tensor(y0, dtype=dtype, device="cuda")
        vv = torch.zeros_like(y)
        for _ in range(30):
            _f, g = fgf(y)
            vn = 0.9 * vv - 0.01 * g
            y = y - 0.9 * vv + 1.9 * vn
            vv = vn
        return y.cpu().numpy().astype(np.float64), fgf(y)[0].cpu().numpy().astype(np.float64)
    y64, f64 = loop(net64.make_fg(x, as_numpy=False), torch.float64)
    y32, f32 = loop(net64.to(torch.float32, "cuda").make_fg(x, as_numpy=False), torch.float32)
    yd, fd = gd.solve(icnn_b200.ConvPICNN.from_variables(v, 64, 32).bind(x), y0, 30, lr=0.01, momentum=0.9)
    ey, e32 = np.abs(yd - y64).max(), np.abs(y32 - y64).max()
    ef, ef32 = np.abs(fd - f64).max(), np.abs(f32 - f64).max()
    print("momentum GD: y err %.2e (float32 floor %.2e), f err %.2e (floor %.2e)" % (ey, e32, ef, ef32))
    assert ey <= max(4 * e32, 1e-6) and ef <= max(4 * ef32, 1e-6 * np.abs(f64).max())


def test_determinism_stale_weights_and_tf32_flags():
    import icnn_b200
    from icnn_b200 import bundle_entropy as be
    _net64, v, x, _y = _helper_case(17, 9, 70)
    flags = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    try:
        torch.backends.cudnn.allow_tf32 = True
        torch.backends.cuda.matmul.allow_tf32 = True
        net = icnn_b200.ConvPICNN.from_variables(v, 17, 9)
        fg = net.bind(x)
        assert torch.backends.cudnn.allow_tf32 and torch.backends.cuda.matmul.allow_tf32
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags
    y0 = np.full((70, 17 * 9), 0.5)
    a, b = be.solveBatch(fg, y0.copy(), nIter=12), be.solveBatch(fg, y0.copy(), nIter=12)
    assert np.array_equal(a[0], b[0]) and a[5] == b[5]
    f1 = fg(y0)[0]
    net.vars["z1_zu_proj/W"].mul_(0.5)
    with pytest.raises(RuntimeError, match="update_weights"):
        net.bind(x)
    net.update_weights()
    f2, _g2 = net.bind(x)(y0)
    assert not np.array_equal(f2, f1)
