"""K1 parity on the GPU: PICNN f / df/dy (and the momentum-GD loop built on it) against the
float64 numpy oracle.  Tolerance: the kernel computes in float32 (FFMA), the oracle in float64;
measured max relative error is ~1e-6, asserted at 1e-5 (the 1e-4 target on y* is on the
iterate, tested in test_gpu_bundle.py)."""
import numpy as np
import pytest
import torch

from oracle import picnn_np, synth

pytestmark = pytest.mark.gpu


def _net(name, B):
    import icnn_b200
    cfg = synth.CONFIGS[name]
    p, x, y0 = synth.make_inputs(name, B=B)
    return cfg, p, x, y0, icnn_b200.PICNN.from_params(p)


@pytest.mark.parametrize("name,B", [("C1", 64), ("C1", 1), ("C3", 77), ("C3", 40), ("C4", 300), ("T", 130), ("C5", 5), ("C5", 70),
                                    ("C2", 400)])
def test_fg_matches_oracle(name, B):
    cfg, p, x, y0, net = _net(name, B)
    fg = net.bind(x, affine=cfg["affine"])
    y = np.random.RandomState(11).uniform(0.02, 0.98, size=y0.shape).astype(np.float32).astype(np.float64)
    f, g = fg(y)
    fo, go = picnn_np.make_fg(p, x, affine=cfg["affine"])(y)
    assert f.dtype == np.float32 and g.dtype == np.float32 and g.shape == y.shape
    # FP32 FFMA path: ~3e-7.  wgmma 3xTF32 path (>= 64 rows): the operand split is exact to 2^-22, but the
    # tensor core does not round its FP32 accumulator to nearest; the chunked accumulation keeps the bias
    # small but it still compounds through the wide layers of C2 and C5, hence the looser bound there
    tol = 5e-5 if (name in ("C5", "C2") and B >= 64) or name == "C5" else 1e-5
    assert np.abs(f - fo).max() <= tol * max(1.0, np.abs(fo).max())
    assert np.abs(g - go).max() <= tol * max(1.0, np.abs(go).max())


@pytest.mark.parametrize("tag,affine", [("ml_fg_c3", False), ("rl_fg_c4", True)])
def test_fg_matches_the_reference_graph_golden(tag, affine, golden_dir):
    """K1 against tests/golden/picnn_tfshim.npz: E_ / dE_dy_ of the reference's OWN Model.f
    (multi-label-cls/icnn_ebundle.py:316-388,146) and Agent.negQ under the bundle_entropy wrapper
    (RL/src/icnn.py:325-404,150-153), executed unmodified on oracle/tf_shim.py (oracle/gen_golden_tfshim.py).
    Same inputs and tolerance as test_fg_matches_oracle[C3-77] / [C4-300]."""
    import os
    import icnn_b200
    from oracle.gen_golden_tfshim import case_inputs
    gold = np.load(os.path.join(golden_dir, "picnn_tfshim.npz"))
    c = case_inputs(tag)
    f, g = icnn_b200.PICNN.from_params(c["p"]).bind(c["x"], affine=affine)(c["y"])
    fo, go = gold[tag + "_f"], gold[tag + "_g"]
    assert np.abs(f - fo).max() <= 1e-5 * max(1.0, np.abs(fo).max())
    assert np.abs(g - go).max() <= 1e-5 * max(1.0, np.abs(go).max())


def test_momentum_gd_matches_the_reference_graph_golden(golden_dir):
    """yn_ / energies_ of the reference's unrolled graph (multi-label-cls/icnn-back.py:116-131, script defaults
    lr .01, momentum .3, 30 steps; C3 dims, 50 rows), golden from the reference code on oracle/tf_shim.py."""
    import os
    import icnn_b200
    from oracle.gen_golden_tfshim import case_inputs
    gold = np.load(os.path.join(golden_dir, "picnn_tfshim.npz"))
    c = case_inputs("gd_c3")
    fg = icnn_b200.PICNN.from_params(c["p"]).bind(c["x"])
    y, f = icnn_b200.gd.solve(fg, c["y"], nIter=c["nIter"], lr=c["lr"], momentum=c["momentum"])
    yo, fo = gold["gd_c3_yN"], gold["gd_c3_energies"]
    assert np.abs(y - yo).max() < 2e-5
    assert np.abs(f - fo).max() <= 2e-5 * max(1.0, np.abs(fo).max())


def test_long_reductions_carry_no_systematic_bias():
    """C5 dims (K up to 5120 per GEMM, four hidden layers): the tensor core truncates its FP32 accumulator at
    every MMA; uncorrected that is a systematic -2e-5 relative scaling of f and g which moves y* by 3e-3 at the
    full C5 size.  With the chunked accumulation (chunk accumulator -> FP32 running sum, RN) the SIGNED mean relative error of f must be ~0 and the
    max error at the FP32-GEMM level.  (Fix: chunked accumulation, icnn_b200/csrc/picnn_tc.cu.)"""
    cfg, p, x, y0, net = _net("C5", 256)
    y = np.random.RandomState(12).uniform(0.02, 0.98, size=y0.shape).astype(np.float32).astype(np.float64)
    f, g = net.bind(x)(y)
    fo, go = picnn_np.make_fg(p, x)(y)
    rel = (f - fo) / np.maximum(np.abs(fo), 1.0)
    print("\nC5 f: signed mean rel err %.2e  max |rel err| %.2e ; g max err / max|g| %.2e"
          % (rel.mean(), np.abs(rel).max(), np.abs(g - go).max() / np.abs(go).max()))
    assert abs(rel.mean()) < 2e-6 and np.abs(rel).max() < 1e-5
    assert np.abs(g - go).max() <= 1e-5 * np.abs(go).max()


def test_fg_is_row_independent():
    """A row's result does not depend on which other rows share its batch, up to float32
    summation order (the split-K factor of the GEMM follows the grid size)."""
    cfg, p, x, y0, net = _net("C3", 96)
    y = np.random.RandomState(5).uniform(0.1, 0.9, size=y0.shape)
    f, g = net.bind(x)(y)
    f2, g2 = net.bind(x[37:70])(y[37:70])
    np.testing.assert_allclose(f[37:70], f2, rtol=2e-6, atol=2e-6)
    np.testing.assert_allclose(g[37:70], g2, rtol=2e-6, atol=2e-6)


@pytest.mark.parametrize("name,B,lr,mom", [("C1", 64, 0.01, 0.3), ("C3", 50, 0.01, 0.3), ("T", 40, 0.01, 0.9)])
def test_momentum_gd_matches_oracle(name, B, lr, mom):
    """multi-label-cls/icnn-back.py:116-131 defaults (.01, .3, 30) and completion's (.01, .9)."""
    import icnn_b200
    cfg, p, x, y0, net = _net(name, B)
    fg = net.bind(x)
    y, f = icnn_b200.gd.solve(fg, y0, nIter=30, lr=lr, momentum=mom)
    yo, fo = picnn_np.momentum_gd(picnn_np.make_fg(p, x), y0, 30, lr, mom)
    assert np.abs(y - yo).max() < 2e-5
    assert np.abs(f - fo).max() <= 2e-5 * max(1.0, np.abs(fo).max())


def test_gd_zero_iterations_returns_energy_of_y0():
    import icnn_b200
    cfg, p, x, y0, net = _net("C1", 8)
    y, f = icnn_b200.gd.solve(net.bind(x), y0, nIter=0)
    np.testing.assert_allclose(y, y0, atol=0)
    fo, _ = picnn_np.make_fg(p, x)(y0)
    np.testing.assert_allclose(f, fo, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("name,B", [("C1", 64), ("T", 300), ("C2", 70), ("C5", 40)])
def test_xpath_gates_kernel_matches_oracle(name, B):
    """Gate precompute (SURVEY.md section 8f row 2) on the library's wgmma GEMM vs the float64 oracle
    x-path (multi-label-cls/icnn_ebundle.py:339-373)."""
    cfg, p, x, y0, net = _net(name, B)
    assert net._xpath, "shape should take the tensor-core x-path"
    cz, cy, d = net.gates(x)
    ocz, ocy, od = picnn_np.gates(p, x)
    for i in range(p.L + 1):
        for got, want in ((cz[i], ocz[i]), (cy[i], ocy[i]), (d[i], od[i])):
            if want is None:
                assert got is None
                continue
            g = got.cpu().numpy().astype(np.float64)
            assert g.shape == want.shape
            assert np.abs(g - want).max() <= 1e-5 * max(1.0, np.abs(want).max())


def test_xpath_batchnorm_is_folded_into_the_gate_gemms():
    """Inference-mode batch-norm on the u-path (multi-label-cls/icnn_ebundle.py:343-345; RL/src/icnn.py:350 with
    --icnn_bn): PICNN.from_params folds the per-feature affine map into the consumer weights; the device gates
    must equal the float64 oracle that applies u = bn(relu(fc(.))) literally."""
    import icnn_b200
    from icnn_b200 import workloads
    p = workloads.synth_params(23, 64, 48, [96, 80, 64])
    rs = np.random.RandomState(4)
    for i in range(p.L - 1):
        w = p.hidden[i]
        p.bn[i] = workloads.bn_affine(rs.uniform(0.5, 1.5, w), 0.1 * rs.randn(w), 0.2 * rs.randn(w), rs.uniform(0.5, 2.0, w))
    x = rs.randn(256, 64).astype(np.float32).astype(np.float64)
    net = icnn_b200.PICNN.from_params(p)
    cz, cy, d = net.gates(x)
    ocz, ocy, od = picnn_np.gates(p, x)
    nobn = picnn_np.gates(workloads.synth_params(23, 64, 48, [96, 80, 64]), x)
    assert np.abs(ocy[2] - nobn[1][2]).max() > 1e-2          # the batch-norm matters in this case
    for i in range(p.L + 1):
        for got, want in ((cz[i], ocz[i]), (cy[i], ocy[i]), (d[i], od[i])):
            if want is not None:
                assert np.abs(got.cpu().numpy().astype(np.float64) - want).max() <= 2e-5 * max(1.0, np.abs(want).max())
    # and through the fused loop: same y* as the oracle that applies BN
    from icnn_b200 import bundle_entropy as be
    from oracle import bundle_np
    y0 = np.full((256, 48), 0.5)
    with np.errstate(all="ignore"):
        o = bundle_np.solve_batch(picnn_np.make_fg(p, x), y0.copy(), nIter=5)
    r = be.solveBatch(net.bind(x), y0.copy(), nIter=5)
    assert np.abs(r[0] - o[0]).max() < 1e-4


def test_xpath_falls_back_without_the_tensor_core_path(monkeypatch):
    monkeypatch.setenv("ICNN_K1", "simt")    # FFMA-only handle -> cuBLAS x-path through torch.addmm
    cfg, p, x, y0, net = _net("C3", 16)
    assert not net._xpath
    cz, cy, d = net.gates(x)
    ocz, ocy, od = picnn_np.gates(p, x)
    assert np.abs(cy[0].cpu().numpy() - ocy[0]).max() <= 1e-4 * max(1.0, np.abs(ocy[0]).max())


@pytest.mark.parametrize("dims,B", [((13, 37, [50, 21, 33]), 200), ((17, 6, [200, 200]), 1000),
                                    ((1836, 159, [600, 159]), 300), ((5, 3, [2]), 64)])
def test_unaligned_widths_take_the_tensor_core_path(dims, B):
    """Widths that are not multiples of 4 floats (C3: n = 159, C4: n = 6): the library pads the leading
    dimension of its own operands to a 16-byte pitch, the tensor maps keep the true extents."""
    import icnn_b200
    from icnn_b200.workloads import synth_params
    m, n, hidden = dims
    p = synth_params(31, m, n, hidden)
    rs = np.random.RandomState(32)
    x = rs.randn(B, m).astype(np.float32).astype(np.float64)
    y = rs.uniform(0.02, 0.98, size=(B, n)).astype(np.float32).astype(np.float64)
    net = icnn_b200.PICNN.from_params(p)
    assert net._xpath
    ocz, ocy, od = picnn_np.gates(p, x)
    cz, cy, d = net.gates(x)
    for i in range(p.L + 1):
        for got, want in ((cz[i], ocz[i]), (cy[i], ocy[i]), (d[i], od[i])):
            if want is not None:
                assert np.abs(got.cpu().numpy() - want).max() <= 1e-5 * max(1.0, np.abs(want).max())
    f, g = net.bind(x)(y)
    fo, go = picnn_np.make_fg(p, x)(y)
    assert np.abs(f - fo).max() <= 1e-5 * max(1.0, np.abs(fo).max())
    assert np.abs(g - go).max() <= 1e-5 * max(1.0, np.abs(go).max())
