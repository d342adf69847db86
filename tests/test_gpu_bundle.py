"""K2 / fused-loop parity on the GPU against the numpy oracle and the reference-generated
golden vectors.

Tolerances (stated per test):
  * K2 in isolation -- the oracle and the GPU are fed bit-identical float32-representable (f, g):
    Mehrotra-PC and dual-Newton modes are restatements of the same float64 algorithm, asserted
    at 1e-9 on y* with identical active-set sizes and nIters;
  * fused (float32 K1) vs the float64 oracle -- the north-star tolerance 1e-4 on y* at the
    reference's short horizons (5 / 10 iterations); at long horizons the oracle itself moves by
    more than 1e-4 under float32 rounding of f, g (SURVEY.md section 7 hard part 1), so the assertion
    is "GPU-vs-oracle no worse than oracle(float32 fg)-vs-oracle(float64 fg)" plus a median bound.
"""
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import bundle_np, picnn_np, synth

pytestmark = pytest.mark.gpu
np.seterr(all="ignore")


def _parity_record(key, d, floor, extra=None):
    """Append the per-config parity statistics to $ICNN_PARITY_DIR/parity_raw.json when that directory is set
    and exists (nothing is written otherwise)."""
    import json
    out = os.environ.get("ICNN_PARITY_DIR")
    if not out or not os.path.isdir(out):
        return
    path = os.path.join(out, "parity_raw.json")
    try:
        with open(path) as f:
            data = json.load(f)
    except Exception:
        data = {}
    rec = {"rows": int(d.size), "device_vs_ref": {"max": float(d.max()), "median": float(np.median(d)),
                                                  "frac_gt_1e-4": float(np.mean(d > 1e-4))},
           "oracle_f32_floor": {"max": float(floor.max()), "median": float(np.median(floor)),
                                "frac_gt_1e-4": float(np.mean(floor > 1e-4))}}
    if extra:
        rec.update(extra)
    data[key] = rec
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


def r32(fg):
    def w(y):
        f, g = fg(y)
        return f.astype(np.float32).astype(np.float64), g.astype(np.float32).astype(np.float64)
    return w


def rowdiff(a, b):
    return np.abs(a - b).max(axis=1)


def lens(rows):
    return np.array([len(r) for r in rows])


K2_CASES = [("C1", 64, 5), ("C1", 13, 20), ("C3", 24, 10), ("T", 12, 10), ("C5", 3, 6)]


def _shape(n, hidden, seed):
    """A small-network workload at n_y = n: what K2 launches depends on (n_y, nIter) only."""
    return dict(synth.CONFIGS["C3"], m=64, n=n, hidden=hidden, seed=seed)


# The builds of the two-sweep PC kernel that no named workload reaches.  With the cases above (C3: one warp, two column
# chunks, scalar row loads; C5: three-vector build) and the C2 golden cases (8 warps) every build bundle_pc.cu selects
# is compared with the oracle.
K2_PC_SHAPES = [
    pytest.param(_shape(100, [96, 64], 11), 24, 10, id="n100-1warp-1chunk"),
    pytest.param(_shape(90, [96, 64], 11), 24, 10, id="n90-1warp-1chunk-scalar"),
    pytest.param(_shape(200, [96, 64], 11), 24, 10, id="n200-1warp-2chunks"),
    # 57 slots at n_y = 4096: two three-vector samples no longer fit an SM -> four-vector build, 16 warps, 2 chunks
    pytest.param(_shape(4096, [96, 64], 11), 24, 56, id="n4096-57slots-16warps-2chunks"),
    pytest.param(_shape(5000, [256, 128], 12), 24, 10, id="n5000-16warps-4chunks"),
]


@pytest.mark.parametrize("name,B,nIter", K2_CASES + K2_PC_SHAPES)
def test_k2_pc_matches_oracle(name, B, nIter):
    from icnn_b200 import bundle_entropy as be
    p, x, y0 = synth.make_inputs(name, B=B)
    fg = r32(picnn_np.make_fg(p, x))
    o = bundle_np.solve_batch(fg, y0.copy(), nIter=nIter, variant="lib", solver="pc")
    r = be.solveBatch(fg, y0.copy(), nIter=nIter, solver="pc", variant="lib")
    same = (lens(r[1]) == lens(o[1])) & (np.array(r[5]) == np.array(o[5]))
    assert same.mean() >= 0.95          # a rank-stop decision may flip on a near-dependent row
    assert rowdiff(r[0], o[0])[same].max() < 1e-9
    assert rowdiff(r[0], o[0]).max() < 1e-4
    for u in np.flatnonzero(same)[:8]:
        k = len(o[1][u])
        if k:
            np.testing.assert_allclose(r[3][u], o[3][u], atol=1e-8)
            np.testing.assert_allclose(np.array(r[2][u]), np.array(o[2][u]), atol=1e-9)
            np.testing.assert_allclose(np.array(r[1][u]), np.array(o[1][u]), atol=0)
            np.testing.assert_allclose(np.array(r[4][u]), np.array(o[4][u]), atol=1e-9)


@pytest.mark.parametrize("name,B,nIter", K2_CASES[:4])
def test_k2_dual_matches_oracle(name, B, nIter):
    from icnn_b200 import bundle_entropy as be
    p, x, y0 = synth.make_inputs(name, B=B)
    fg = r32(picnn_np.make_fg(p, x))
    o = bundle_np.solve_batch(fg, y0.copy(), nIter=nIter, variant="dual")
    r = be.solveBatch(fg, y0.copy(), nIter=nIter, variant="dual")
    same = (lens(r[1]) == lens(o[1])) & (np.array(r[5]) == np.array(o[5]))
    assert same.mean() >= 0.95
    assert rowdiff(r[0], o[0])[same].max() < 1e-9
    # invariants (SURVEY.md section 8c): lam on the simplex, y = sigma(-G^T lam) for unfinished samples
    for u in range(B):
        lam = r[3][u]
        if lam is None:
            continue
        assert np.all(lam > 0) and abs(lam.sum() - 1) < 1e-9
        if r[5][u] == nIter:
            y = 1.0 / (1.0 + np.exp(np.array(r[1][u], dtype=np.float64).T.dot(lam)))
            np.testing.assert_allclose(y, r[0][u], atol=1e-12)


@pytest.mark.parametrize("B,nIter", [(256, 5), (40, 12)])
def test_k2_rl_matches_oracle(B, nIter):
    from icnn_b200 import bundle_entropy as be
    p, x, y0 = synth.make_inputs("C4", B=B)
    fg = r32(picnn_np.make_fg(p, x, affine=True))
    calls = []
    o = bundle_np.solve_batch(fg, y0.copy(), nIter=nIter, variant="rl")
    r = be.solveBatch(fg, y0.copy(), nIter=nIter, variant="rl", callback=lambda t, f: calls.append((t, f.shape)))
    assert r[0].min() >= 0.03 and r[0].max() <= 0.97          # RL/src/bundle_entropy.py:118
    assert rowdiff(r[0], o[0]).max() < 1e-5
    assert np.median(rowdiff(r[0], o[0])) < 1e-8
    assert calls and calls[0] == (0, (B,))                     # callback(t, fi), :103-104


# c1_rl: the RL copy has no rank test, so on the ReLU toy net duplicate rows make the Newton system
# numerically singular (28 of 122 solves have cond = inf); np.linalg.solve then returns
# rounding-dependent directions that no re-implementation can reproduce -- only the bulk is asked.
GOLD = [("c1_pc", 1e-5, 1e-7), ("c1_dual", 1e-5, 1e-7), ("c1_rl", None, 1e-6), ("c1_boyd", None, None),
        ("c1_pc_long", 1e-5, 1e-7), ("c3_pc", None, 1e-5), ("c3_dual", None, 1e-5), ("c4_rl", 1e-5, 1e-6),
        ("c4_rl_long", 1e-4, 1e-6), ("t_pc", 1e-4, 1e-5), ("t_dual", 1e-4, 1e-5), ("c2_pc", "long", 1e-3),
        ("c5_pc", 1e-4, 1e-5),
        # round 2: the configs' own horizons, judged against the oracle's float32 noise floor measured in the test
        ("c3_pc_full", "floor", None), ("c2_pc_full", "floor", None), ("c5_pc_full", "floor", None)]


@pytest.mark.parametrize("case,maxtol,medtol", GOLD)
def test_k2_against_reference_golden(case, maxtol, medtol, golden_dir):
    """GPU bundle step driven by the float64 oracle fg (rounded to float32 on upload) vs the
    outputs of the UNMODIFIED reference modules on the same inputs."""
    from icnn_b200 import bundle_entropy as be
    gold = np.load(os.path.join(golden_dir, case + ".npz"))
    cfgname = str(gold["config"])
    cfg = synth.CONFIGS[cfgname]
    B, nIter, variant = int(gold["B"]), int(gold["nIter"]), str(gold["variant"])
    p, x, y0 = synth.make_inputs(cfgname, B=B)
    fg = picnn_np.make_fg(p, x, affine=cfg["affine"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        r = be.solveBatch(fg, y0.copy(), nIter=nIter, variant=variant, solver=str(gold["solver"]) or "pc")
    d = rowdiff(r[0], gold["x"])
    if case == "c1_boyd":
        # 'boyd' is accepted and mapped to the converged solve; the reference's 20 damped
        # iterations stop short of the optimum, so only closeness of the objective is asked
        fgv = lambda y: fg(y)[0] + np.sum(y * np.log(y) + (1 - y) * np.log(1 - y), axis=1)  # noqa: E731
        assert np.all(fgv(r[0]) <= fgv(gold["x"]) + 1e-6)
        return
    if maxtol == "floor":
        # Long horizons: the float64 reference itself moves when (f, g) are rounded to float32 (the iterates
        # converge onto ReLU kinks).  Measure that floor here -- the oracle fed the float32-rounded fg against the
        # reference's golden y* -- and require the device to stay within it: fraction of samples off by more
        # than 1e-4 <= floor + max(0.02, 2.5 rows), median <= max(1e-6, 4 x floor median).
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            o32 = bundle_np.solve_batch(r32(fg), y0.copy(), nIter=nIter, variant=variant)
        fl = rowdiff(o32[0], gold["x"])
        print("\n%s: device-vs-reference max %.2e median %.2e frac>1e-4 %.3f | oracle(f32 fg)-vs-reference max %.2e "
              "median %.2e frac>1e-4 %.3f" % (case, d.max(), np.median(d), np.mean(d > 1e-4), fl.max(), np.median(fl),
                                              np.mean(fl > 1e-4)))
        _parity_record(case, d, fl)
        assert np.mean(d > 1e-4) <= np.mean(fl > 1e-4) + max(0.02, 2.5 / B), (np.mean(d > 1e-4), np.mean(fl > 1e-4))
        assert np.median(d) <= max(1e-6, 4 * np.median(fl)), (np.median(d), np.median(fl))
        assert d.max() <= max(1e-4, 10 * fl.max()), (d.max(), fl.max())
        return
    if maxtol == "long":
        # 30 iterations at n=2048: the float64 oracle itself moves by up to 1e-3 under float32
        # rounding of (f, g) (test_fused_vs_oracle prints the floor): the iterates converge onto
        # ReLU kinks, where the active piece flips under any perturbation
        assert d.max() < 5e-3, d
    elif maxtol is not None:
        assert d.max() < maxtol, (d.max(), np.median(d))
    else:
        assert np.mean(d < 1e-4) >= 0.75, np.mean(d < 1e-4)
    assert np.median(d) < medtol, np.median(d)
    if maxtol != "long":      # active-set sizes only compare before the trajectories decorrelate
        agree = np.mean(lens(r[1]) == gold["counts"])
        assert agree >= (0.5 if nIter > 10 else 0.8), agree


# ("T", 160, ...) and ("C2", 70, ...) have >= 64 rows: K1 and the gate precompute run on the wgmma path
FUSED = [("C1", 64, 5, 1e-4), ("C4", 512, 5, 1e-4), ("T", 48, 10, 1e-4), ("T", 160, 10, None), ("C3", 96, 10, None),
         ("C2", 6, 30, None), ("C2", 70, 8, None)]


@pytest.mark.parametrize("name,B,nIter,maxtol", FUSED)
def test_fused_vs_oracle(name, B, nIter, maxtol):
    """The headline parity statement: fused device loop (float32 K1 + float64 K2) vs the float64
    oracle of the variant BASELINE.json names, next to the oracle's own float32 noise floor."""
    import icnn_b200
    from icnn_b200 import bundle_entropy as be
    cfg = synth.CONFIGS[name]
    p, x, y0 = synth.make_inputs(name, B=B)
    variant = cfg["variant"]
    o = bundle_np.solve_batch(picnn_np.make_fg(p, x, affine=cfg["affine"]), y0.copy(), nIter=nIter, variant=variant)
    o32 = bundle_np.solve_batch(picnn_np.make_fg(p, x, affine=cfg["affine"], dtype=np.float32, out_dtype=np.float64),
                                y0.copy(), nIter=nIter, variant=variant)
    net = icnn_b200.PICNN.from_params(p)
    y0c = y0.copy()
    r = be.solveBatch(net.bind(x, affine=cfg["affine"]), y0c, nIter=nIter, variant=variant)
    assert r[0] is y0c                                       # initXs is overwritten in place (:200)
    d = rowdiff(r[0], o[0])
    floor = rowdiff(o32[0], o[0])
    print("\n%s: GPU-vs-oracle max %.2e median %.2e frac>1e-4 %.3f | oracle f32 noise floor max %.2e median %.2e frac>1e-4 %.3f"
          % (name, d.max(), np.median(d), np.mean(d > 1e-4), floor.max(), np.median(floor), np.mean(floor > 1e-4)))
    if maxtol is not None:
        assert d.max() < maxtol
    else:
        assert np.median(d) < max(1e-5, 4 * np.median(floor))
        _parity_record("fused_%s_B%d_it%d" % (name, B, nIter), d, floor)
        # floor + 0.02, or + 2.5 rows when the batch is small: device and float32 oracle are two independent float32
        # realisations, the count of kink-flipped rows fluctuates by ~sqrt(count) between them
        assert np.mean(d > 1e-4) <= np.mean(floor > 1e-4) + max(0.02, 2.5 / B)
    # objective gap: f - H at the GPU solution is as good as the oracle's
    fg64 = picnn_np.make_fg(p, x, affine=cfg["affine"])
    obj = lambda y: fg64(y)[0] + np.sum(y * np.log(y) + (1 - y) * np.log(1 - y), axis=1)  # noqa: E731
    gap = (obj(r[0]) - obj(o[0])) / np.maximum(1.0, np.abs(obj(o[0])))
    assert np.median(np.abs(gap)) < 1e-5 and gap.max() < 1e-3, gap


@pytest.mark.parametrize("name,B,cut,nIter", [("T", 160, 70, 10), ("C4", 200, 77, 5), ("C3", 160, 67, 5)])
def test_shard_concat_equals_unsharded(name, B, cut, nIter):
    """Samples are independent: solving two row blocks separately equals solving the batch at
    once (what the multi-GPU sharding relies on) -- up to float32 summation order in K1, whose
    split-K factor follows the grid size.  Both shards keep >= 64 rows (same K1 path), and the horizons are
    the ones where the float32 noise floor of the workload is below 1 %, so that a
    disagreement would be a sharding bug and not a ReLU-kink flip."""
    import icnn_b200
    from icnn_b200 import bundle_entropy as be
    cfg = synth.CONFIGS[name]
    p, x, y0 = synth.make_inputs(name, B=B)
    net = icnn_b200.PICNN.from_params(p)
    kw = dict(nIter=nIter, variant=cfg["variant"])
    full = be.solveBatch(net.bind(x, affine=cfg["affine"]), y0.copy(), **kw)
    a = be.solveBatch(net.bind(x[:cut], affine=cfg["affine"]), y0[:cut].copy(), **kw)
    b = be.solveBatch(net.bind(x[cut:], affine=cfg["affine"]), y0[cut:].copy(), **kw)
    d = rowdiff(full[0], np.concatenate([a[0], b[0]]))
    assert np.median(d) < 1e-5 and np.mean(d < 1e-4) >= 0.97, (np.median(d), np.mean(d < 1e-4))
    assert np.mean(np.array(full[5]) == np.array(a[5] + b[5])) >= 0.95


def test_fused_properties_at_full_size():
    """Config 3 at BASELINE.json's full size (B=4096, n=159, 10 iterations): size-independent
    properties -- multipliers on the simplex, bundle rows under-estimate the convex f at y*,
    rows are the gradients at the stored iterates, y* inside the box."""
    import icnn_b200
    from icnn_b200 import bundle_entropy as be
    p, x, y0 = synth.make_inputs("C3")
    net = icnn_b200.PICNN.from_params(p)
    fg = net.bind(x)
    y, G, h, lam, ys, nIters = be.solveBatch(fg, y0.copy(), nIter=10)
    assert y.shape == (4096, 159) and np.all(np.isfinite(y)) and y.min() > 0 and y.max() < 1
    f_star, _ = fg(y)
    for u in range(0, 4096, 97):
        k = len(G[u])
        assert 1 <= k <= 10 and len(h[u]) == k and len(ys[u]) == k and lam[u].shape == (k,)
        assert np.all(lam[u] > 1e-8) and abs(lam[u].sum() - 1) < 1e-6
        Gu = np.array(G[u], dtype=np.float64)
        assert np.all(Gu.dot(y[u]) + np.array(h[u]) <= f_star[u] + 1e-3 * max(1, abs(f_star[u])))
    # rows are gradients at the stored iterates (consistency of A / xs, multi-label-cls/icnn_ebundle.py:300-305).
    # Evaluated through the SAME bound fg: late iterates sit on ReLU kinks, so gates recomputed
    # for another batch size (cuBLAS is not batch-invariant) would select a different piece.
    us = list(range(0, 4096, 512))
    Y = y0.copy()
    for u in us:
        Y[u] = ys[u][-1]
    _, gchk = fg(Y)
    for u in us:
        np.testing.assert_allclose(G[u][-1], gchk[u], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("name", ["C2", "C4", "T", "C5"])
def test_fused_properties_at_full_size_other_configs(name):
    """BASELINE.json's remaining configs (and the north-star target shape) at their FULL sizes --
    C2 400 x 2048 x 30 its, C4 65 536 x 6 (RL variant), T 4096 x 512 x 10, C5 8192 x 4096 x 50 --
    through size-independent properties: finite iterate inside the box (RL: inside the clip
    [.03, .97], RL/src/bundle_entropy.py:118), multipliers on the simplex, every kept row an
    under-estimator of the convex f at y*, bookkeeping lists consistent."""
    import icnn_b200
    from icnn_b200 import bundle_entropy as be
    cfg = synth.CONFIGS[name]
    p, x, y0 = synth.make_inputs(name)
    B, n, nIter = cfg["B"], cfg["n"], cfg["nIter"]
    net = icnn_b200.PICNN.from_params(p)
    fg = net.bind(x, affine=cfg["affine"])
    y, G, h, lam, ys, nIters = be.solveBatch(fg, y0.copy(), nIter=nIter, variant=cfg["variant"])
    assert y.shape == (B, n) and np.all(np.isfinite(y))
    if cfg["variant"] == "rl":
        assert y.min() >= 0.03 - 1e-12 and y.max() <= 0.97 + 1e-12
    else:
        assert y.min() > 0 and y.max() < 1
    assert len(G) == B and len(nIters) == B
    f_star, _ = fg(y)
    step = max(1, B // 41)
    for u in range(0, B, step):
        k = len(G[u])
        assert 1 <= k <= min(nIter, n) + 1 and len(h[u]) == k and len(ys[u]) == k and lam[u].shape == (k,)
        assert np.all(lam[u] >= 0) and abs(lam[u].sum() - 1) < 1e-6
        Gu = np.array(G[u], dtype=np.float64)
        assert np.all(Gu.dot(y[u]) + np.array(h[u]) <= f_star[u] + 1e-3 * max(1, abs(f_star[u])))


FULLSIZE = [("C3", 64), ("T", 64), ("C4", 64), ("C2", 48), ("C5", 16)]


@pytest.mark.parametrize("name,nsub", FULLSIZE)
def test_full_size_subsample_matches_oracle(name, nsub):
    """BASELINE.json's configs at FULL size and FULL horizon (C5: 8192 x 4096, 50 iterations, 51 slots): the
    samples are independent (lib/bundle_entropy.py:211), so a random subsample of the device result is compared
    with the float64 oracle run on exactly those rows, next to the oracle's own noise floor on the same rows (the
    larger of: float32-arithmetic fg; float64 fg with 2e-6 relative noise = the device's measured f/g accuracy).  Tolerance: fraction of rows off by more than 1e-4 <= floor + max(0.02, 2.5 rows), median <=
    max(1e-5, 4 x floor median); at the short horizons (C3 / C4 / T) the floor is ~0 and this is the 1e-4 statement."""
    import icnn_b200
    from icnn_b200 import bundle_entropy as be
    cfg = synth.CONFIGS[name]
    p, x, y0 = synth.make_inputs(name)
    B, nIter, variant = cfg["B"], cfg["nIter"], cfg["variant"]
    net = icnn_b200.PICNN.from_params(p)
    r = be.solveBatch(net.bind(x, affine=cfg["affine"]), y0.copy(), nIter=nIter, variant=variant)
    rows = np.sort(np.random.RandomState(7).choice(B, size=nsub, replace=False))
    xs, ys = x[rows], y0[rows]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        o = bundle_np.solve_batch(picnn_np.make_fg(p, xs, affine=cfg["affine"]), ys.copy(), nIter=nIter, variant=variant)
        o32 = bundle_np.solve_batch(picnn_np.make_fg(p, xs, affine=cfg["affine"], dtype=np.float32, out_dtype=np.float64),
                                    ys.copy(), nIter=nIter, variant=variant)
        # second floor: the float64 oracle under a relative perturbation of (f, g) of the size of the device's
        # measured f/g error (<= 2e-6: tests/test_gpu_picnn.py::test_long_reductions_carry_no_systematic_bias) --
        # SURVEY.md section 8c asks for both floors; with 12-64 rows one realisation alone is a noisy estimate
        rsn = np.random.RandomState(123)
        fg64n = picnn_np.make_fg(p, xs, affine=cfg["affine"])

        def fg_noisy(y):
            f, g = fg64n(y)
            return f * (1.0 + 2e-6 * rsn.randn(*f.shape)), g * (1.0 + 2e-6 * rsn.randn(*g.shape))
        on = bundle_np.solve_batch(fg_noisy, ys.copy(), nIter=nIter, variant=variant)
    d = rowdiff(r[0][rows], o[0])
    floor32 = rowdiff(o32[0], o[0])
    floorn = rowdiff(on[0], o[0])
    floor = floorn if np.mean(floorn > 1e-4) > np.mean(floor32 > 1e-4) else floor32     # the larger of the two floors
    kdev = lens([r[1][int(u)] for u in rows])
    print("\n%s full size, %d-row subsample: device-vs-oracle max %.2e median %.2e frac>1e-4 %.3f | oracle f32 floor max "
          "%.2e median %.2e frac>1e-4 %.3f | active rows device mean %.1f oracle mean %.1f"
          % (name, nsub, d.max(), np.median(d), np.mean(d > 1e-4), floor.max(), np.median(floor), np.mean(floor > 1e-4),
             kdev.mean(), lens(o[1]).mean()))
    _parity_record("fullsize_%s" % name, d, floor, {"B": B, "nIter": nIter, "KS": (nIter if variant == "rl" else min(nIter, cfg["n"])) + 1,
                                                   "floor_f32_arithmetic_frac_gt_1e-4": float(np.mean(floor32 > 1e-4)),
                                                   "floor_2e-6_noise_frac_gt_1e-4": float(np.mean(floorn > 1e-4)),
                                                   "floor_f32_arithmetic_median": float(np.median(floor32)),
                                                   "floor_2e-6_noise_median": float(np.median(floorn)),
                                                   "active_rows_device_mean": float(kdev.mean()),
                                                   "active_rows_oracle_mean": float(lens(o[1]).mean())})
    assert np.mean(d > 1e-4) <= np.mean(floor > 1e-4) + max(0.02, 2.5 / nsub), (np.mean(d > 1e-4), np.mean(floor > 1e-4))
    assert np.median(d) <= max(1e-5, 4 * np.median(floor)), (np.median(d), np.median(floor))
    # objective: f - H at the device solution is as good as the oracle's on those rows
    fg64 = picnn_np.make_fg(p, xs, affine=cfg["affine"])
    obj = lambda y: fg64(y)[0] + np.sum(y * np.log(y) + (1 - y) * np.log(1 - y), axis=1)  # noqa: E731
    gap = (obj(r[0][rows]) - obj(o[0])) / np.maximum(1.0, np.abs(obj(o[0])))
    assert np.median(np.abs(gap)) < 1e-5 and gap.max() < 1e-3, gap


def test_edge_cases_and_error_paths():
    import icnn_b200
    from icnn_b200 import bundle_entropy as be
    p, x, y0 = synth.make_inputs("C1", B=9)
    net = icnn_b200.PICNN.from_params(p)
    fg = net.bind(x)
    # nIter = 1: one row, y = PC solution of a single cut; compare with the oracle
    r = be.solveBatch(fg, y0.copy(), nIter=1)
    o = bundle_np.solve_batch(picnn_np.make_fg(p, x), y0.copy(), nIter=1)
    assert rowdiff(r[0], o[0]).max() < 1e-5 and r[5] == o[5]
    # empty batch: the reference's loops simply do nothing
    e = be.solveBatch(lambda yy: (np.zeros(0), np.zeros((0, 8))), np.zeros((0, 8)), nIter=3)
    assert e[0].shape == (0, 8) and len(e[1]) == 0 and e[5] == []
    # B = 1
    r1 = be.solveBatch(net.bind(x[:1]), y0[:1].copy(), nIter=5)
    # (the x-path gates come from cuBLAS, which is not batch-invariant -> float32-level noise)
    np.testing.assert_allclose(r1[0], be.solveBatch(fg, y0.copy(), nIter=5)[0][:1], atol=2e-5)
    # unknown solver -> RuntimeError like lib/bundle_entropy.py:232
    with pytest.raises(RuntimeError, match="Solver unknown"):
        be.solveBatch(fg, y0.copy(), solver="nope")
    # callback(t, f, x) is invoked once per executed iteration with the live iterate
    seen = []
    be.solveBatch(fg, y0.copy(), nIter=5, callback=lambda t, f, xx: seen.append((t, f.shape, xx.shape)))
    assert seen[0] == (0, (9,), (9, 8)) and [s[0] for s in seen] == list(range(len(seen)))
    # non-finite fg: flagged, not propagated silently
    def bad(y):
        f, g = picnn_np.make_fg(p, x)(y)
        g[3, 2] = np.nan
        return f, g
    with pytest.warns(UserWarning, match="non-finite"):
        rb = be.solveBatch(bad, y0.copy(), nIter=3, return_state=True)
    assert rb[-1].status_host[3] == 4 and np.all(np.isfinite(rb[0][[0, 1, 2, 4]]))
    with pytest.raises(RuntimeError):
        be.solveBatch(bad, y0.copy(), nIter=3, strict=True)


def test_slot_cap_float64_callback_stats_and_state_reuse():
    """Round-2 API surface: the 64-slot cap is reported up front; a float64 fg keeps its f in float64 for the cut
    offsets (the reference forms b = f - sum(g x) in float64, lib/bundle_entropy.py:205-207); per-iteration
    statistics; a reused BundleState reproduces the result bit for bit."""
    import icnn_b200
    from icnn_b200 import bundle_entropy as be
    p, x, y0 = synth.make_inputs("C3", B=40)
    fg64 = picnn_np.make_fg(p, x)
    # nIter > 63 with n_y >= 64: min(nIter, n) + 1 > 64 slots -> clear error instead of a launch failure
    with pytest.raises(ValueError, match="64"):
        be.solveBatch(fg64, y0.copy(), nIter=70)
    # float64 f with bits below float32 resolution, float32-representable rows: the offsets must follow the float64 f
    def fg_f64(y):
        f, g = fg64(y)
        return f + 1e-9 * np.arange(1, len(f) + 1), g.astype(np.float32).astype(np.float64)
    o = bundle_np.solve_batch(fg_f64, y0.copy(), nIter=4)
    r = be.solveBatch(fg_f64, y0.copy(), nIter=4)
    for u in (0, 7, 39):
        np.testing.assert_allclose(np.array(r[2][u]), np.array(o[2][u]), rtol=0, atol=1e-11)   # h = f - g.y from the f64 f
    assert rowdiff(r[0], o[0]).max() < 1e-9
    # per-iteration statistics + state reuse on the fused path
    net = icnn_b200.PICNN.from_params(p)
    fgd = net.bind(x)
    seen = []
    r1 = be.solveBatch(fgd, y0.copy(), nIter=6, return_state=True, stats=True,
                       callback=lambda t, f, xx: seen.append(float(np.mean(f + np.sum(xx * np.log(xx) + (1 - xx) * np.log(1 - xx), axis=1)))))
    st = r1[-1]
    sd = st.stats()
    assert sd["entering"][0] == 40 and np.all(np.diff(sd["entering"]) <= 0)
    np.testing.assert_allclose(sd["mean_f_minus_H"][:len(seen)][sd["entering"][:len(seen)] == 40],
                               np.array(seen)[sd["entering"][:len(seen)] == 40], rtol=1e-5, atol=1e-4)
    assert np.all(sd["inner_its"][:len(seen)] >= sd["entering"][:len(seen)] - sd["stopped"][:len(seen)])
    ya = be.solveBatch(fgd, y0.copy(), nIter=6)[0]
    yb = be.solveBatch(fgd, y0.copy(), nIter=6, state=st)[0]          # reused buffers, no allocation
    assert np.array_equal(ya, yb)


def test_early_exit_when_all_finished():
    """Once every sample hit the rank stop the remaining iterations are device-side no-ops
    (the reference returns early, lib/bundle_entropy.py:239)."""
    import icnn_b200
    from icnn_b200 import bundle_entropy as be
    p, x, y0 = synth.make_inputs("C1", B=16)
    net = icnn_b200.PICNN.from_params(p)
    r = be.solveBatch(net.bind(x), y0.copy(), nIter=40, return_state=True)
    na = r[-1].nactive.cpu().numpy()
    o = bundle_np.solve_batch(picnn_np.make_fg(p, x), y0.copy(), nIter=40)
    assert na[0] == 16 and na[-1] == 0 and max(r[5]) < 39
    assert rowdiff(r[0], o[0]).max() < 1e-4


@pytest.mark.parametrize("name,B,nIter,env", [("C2", 5, 12, {"ICNN_K2_RESIDENT": "1"}),
                                              ("C2", 5, 12, {"ICNN_K2_RESIDENT": "1", "ICNN_K2_CS": "2"}),
                                              ("T", 20, 10, {"ICNN_K2_RESIDENT": "1"}),
                                              ("C3", 20, 10, {"ICNN_K2_RESIDENT": "1"}),
                                              ("C5", 3, 12, {"ICNN_K2_RESIDENT": "1", "ICNN_K2_CS": "8"}),
                                              ("C5", 3, 12, {"ICNN_K2_WPS": "16"}),      # 512-thread CTA per sample
                                              ("C2", 5, 12, {"ICNN_K2_WPS": "16"})])
def test_resident_cluster_variant_matches_streaming(name, B, nIter, env, monkeypatch):
    """The optional K2 launch variants (rows resident in shared memory, sample split over a
    thread-block cluster with DSMEM exchanges, 16 warps per sample) compute the same thing as the
    default streaming kernel.  The launch configuration is read from the environment at every launch.
    These variables select among five-sweep builds, which the PC solver takes only under ICNN_K2_PC=legacy at these
    shapes; icnn_k2_last_launch shows that both arms ran the five-sweep kernel and that the variant ran in the second
    (tests/test_gpu_k2_builds.py compares each variant with the float64 oracle)."""
    import ctypes as C
    from icnn_b200 import _capi, bundle_entropy as be

    def ran():
        out = (C.c_int32 * _capi.K2_PLAN_LEN)()
        assert _capi.lib.icnn_k2_last_launch(out) == 0
        return tuple(out)
    p, x, y0 = synth.make_inputs(name, B=B)
    fg = r32(picnn_np.make_fg(p, x))
    for k_ in ("ICNN_K2_RESIDENT", "ICNN_K2_CS", "ICNN_K2_WPS", "ICNN_K2_SMALL"):
        monkeypatch.delenv(k_, raising=False)
    monkeypatch.setenv("ICNN_K2_PC", "legacy")
    ref = be.solveBatch(fg, y0.copy(), nIter=nIter)
    streaming = ran()
    assert streaming[0] == 2 and streaming[2] == 1 and streaming[5] == 0, streaming    # five-sweep, no cluster, streamed
    for k_, v_ in env.items():
        monkeypatch.setenv(k_, v_)
    alt = be.solveBatch(fg, y0.copy(), nIter=nIter)
    variant = ran()
    assert variant[0] == 2 and variant != streaming, (variant, streaming)
    if env.get("ICNN_K2_RESIDENT") == "1":
        assert variant[5] == 1, variant
    if "ICNN_K2_CS" in env:
        assert variant[2] == int(env["ICNN_K2_CS"]), variant
    if "ICNN_K2_WPS" in env:
        assert variant[1] == int(env["ICNN_K2_WPS"]), variant
    same = (lens(ref[1]) == lens(alt[1])) & (np.array(ref[5]) == np.array(alt[5]))
    assert same.mean() >= 0.8
    assert rowdiff(ref[0], alt[0])[same].max() < 1e-9


@pytest.mark.parametrize("name,B,nIter,env_ref,env_alt", [
    ("C5", 3, 12, {"ICNN_PC_V3": "0"}, {}),                  # n_y = 4096: three-vector build is the default
    ("C5", 3, 45, {"ICNN_PC_V3": "0"}, {}),                  # deep horizon: k up to ~35 rows, every row-block shape of sweep A
])
def test_three_vector_pc_kernel_matches_four_vector(name, B, nIter, env_ref, env_alt, monkeypatch):
    """The V3 build of the predictor-corrector kernel (y, ry, du in shared memory; u = ry - logit(y) and dy recomputed
    in the update; two samples per SM at n_y = 4096) walks the same interior-point iterates as the four-vector build
    up to FP64 rounding of the recovered u."""
    from icnn_b200 import bundle_entropy as be
    p, x, y0 = synth.make_inputs(name, B=B)
    fg = r32(picnn_np.make_fg(p, x))
    for k_, v_ in env_ref.items():
        monkeypatch.setenv(k_, v_)
    ref = be.solveBatch(fg, y0.copy(), nIter=nIter)
    for k_ in env_ref:
        monkeypatch.delenv(k_)
    for k_, v_ in env_alt.items():
        monkeypatch.setenv(k_, v_)
    alt = be.solveBatch(fg, y0.copy(), nIter=nIter)
    same = (lens(ref[1]) == lens(alt[1])) & (np.array(ref[5]) == np.array(alt[5]))
    assert same.mean() >= 0.6
    assert rowdiff(ref[0], alt[0])[same].max() < 1e-9
    assert np.all((alt[0] > 0) & (alt[0] < 1))


def test_loop_graph_replays_the_fused_loop_bit_for_bit():
    """solveBatch(graph=True): the nIter x (K1, K2) launches captured once into a CUDA graph (icnn_loop_graph_*)
    and replayed with one launch give the same bits as the eager enqueue, call after call; the capture is keyed on
    the buffers it bakes in (a new bind -> a new capture, never a stale replay)."""
    import icnn_b200
    from icnn_b200 import _capi, bundle_entropy as be
    for name, B, nIter in (("C3", 48, 6), ("C4", 300, 5), ("T", 70, 5)):
        cfg = synth.CONFIGS[name]
        p, x, y0 = synth.make_inputs(name, B=B)
        net = icnn_b200.PICNN.from_params(p)
        fgd = net.bind(x, affine=cfg["affine"])
        kw = dict(nIter=nIter, variant=cfg["variant"])
        r0 = be.solveBatch(fgd, y0.copy(), return_state=True, **kw)
        st = r0[-1]
        g1 = be.solveBatch(fgd, y0.copy(), state=st, graph=True, **kw)
        assert len(st._graphs) == 1
        nodes = _capi.lib.icnn_loop_graph_nodes(next(iter(st._graphs.values())))
        assert nodes >= 2 * nIter + 1
        g2 = be.solveBatch(fgd, y0.copy(), state=st, graph=True, **kw)      # replay
        assert len(st._graphs) == 1
        assert np.array_equal(r0[0], g1[0]) and np.array_equal(r0[0], g2[0])
        assert r0[5] == g1[5] == g2[5]
        # other inputs through the same captured graph: the graph reads y0 / the gates from the baked-in buffers
        y1 = np.clip(y0 + 0.05, 0.01, 0.99)
        e1 = be.solveBatch(fgd, y1.copy(), **kw)
        g3 = be.solveBatch(fgd, y1.copy(), state=st, graph=True, **kw)
        assert np.array_equal(e1[0], g3[0])
        # a second bind has its own gate buffers -> its own capture
        fgd2 = net.bind(x[::-1].copy(), affine=cfg["affine"])
        e2 = be.solveBatch(fgd2, y0.copy(), **kw)
        g4 = be.solveBatch(fgd2, y0.copy(), state=st, graph=True, **kw)
        assert np.array_equal(e2[0], g4[0])


@pytest.mark.parametrize("name,B,nIter,variant", [("C1", 64, 5, "lib"), ("C1", 64, 8, "dual"), ("C4", 300, 5, "rl")])
def test_thread_per_sample_kernel_matches_group_kernel(name, B, nIter, variant, monkeypatch):
    """n_y <= 8 runs the one-thread-per-sample K2 (bundle_step_small.cu); ICNN_K2_SMALL=0 forces the
    warp-per-sample kernel.  Same algorithm, different summation order."""
    from icnn_b200 import bundle_entropy as be
    cfg = synth.CONFIGS[name]
    p, x, y0 = synth.make_inputs(name, B=B)
    fg = r32(picnn_np.make_fg(p, x, affine=cfg["affine"]))
    small = be.solveBatch(fg, y0.copy(), nIter=nIter, variant=variant)
    monkeypatch.setenv("ICNN_K2_SMALL", "0")
    group = be.solveBatch(fg, y0.copy(), nIter=nIter, variant=variant)
    same = (lens(small[1]) == lens(group[1])) & (np.array(small[5]) == np.array(group[5]))
    assert same.mean() >= 0.9
    # the RL Newton stops on |tau d| < 1e-10 / 20 iterations, so summation-order noise shows at 1e-7
    assert rowdiff(small[0], group[0])[same].max() < (1e-6 if variant == "rl" else 1e-9)


def test_callback_mode_mirrors_numpy_rank_tolerance_dtype():
    """np.linalg.matrix_rank scales its tolerance with the row dtype; a float32 fg therefore stops
    samples earlier in the reference (lib/bundle_entropy.py:219).  Callback mode reproduces that."""
    from icnn_b200 import bundle_entropy as be
    p, x, y0 = synth.make_inputs("C2", B=6)
    fg32 = picnn_np.make_fg(p, x, dtype=np.float32, out_dtype=np.float32)
    o = bundle_np.solve_batch(fg32, y0.copy(), nIter=30)            # float32 rows -> eps32 rank test
    r = be.solveBatch(fg32, y0.copy(), nIter=30)
    assert np.mean(np.abs(np.array(r[5]) - np.array(o[5])) <= 2) >= 0.6, (r[5], o[5])
    assert np.median(rowdiff(r[0], o[0])) < 1e-4
    assert max(r[5]) <= max(o[5]) + 2 and min(r[5]) < 30            # early stops do happen


def test_single_sample_solve_alias():
    """lib/bundle_entropy_dual.py:87-127 `solve`: one sample, fg(x [n]) -> (f, g [n])."""
    from icnn_b200 import bundle_entropy as be
    p, x, y0 = synth.make_inputs("C3", B=1)
    fgb = picnn_np.make_fg(p, x)
    fg1 = lambda y: tuple(v[0] for v in fgb(y[None, :]))  # noqa: E731
    seen = []
    xs = be.solve(fg1, y0[0], nIter=6, callback=lambda t, f, xx: seen.append(t))
    o = bundle_np.solve_batch(fgb, y0.copy(), nIter=6, variant="dual")
    assert xs.shape == (159,) and seen == list(range(len(seen))) and len(seen) >= 1
    assert np.abs(xs - o[0][0]).max() < 1e-5


def test_callback_mode_with_a_conv_picnn_fg():
    """SURVEY.md section 8d config 2: the reference's Olivetti energy is CONVOLUTIONAL
    (completion/icnn_ebundle.py:337-452); the fused path covers fully-connected PICNNs, and any other
    architecture goes through callback mode -- fg is the user's own callable (here a torch conv-PICNN on
    the GPU, float32 like the TF fetch), the per-sample bundle work runs in K2.  Checked against the
    oracle driven by the SAME float32 fg (what the library is responsible for: identical (f, g) in,
    identical y* out), at the Olivetti dims (y = the 64 x 32 left half, n_y = 2048); the distance to
    the float64 evaluation of the network is printed (1e-6 with FP32 convolutions; with torch's
    default TF32 convolutions the user's g carries 1e-3 relative noise and half the samples move by
    2e-2 -- a property of that fg, which is why TF32 is switched off here)."""
    import torch
    from conv_picnn import ConvPICNN
    from icnn_b200 import bundle_entropy as be
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    B, H, W, nIter = 8, 64, 32, 6
    net64 = ConvPICNN(H, W, seed=1, dtype=torch.float64)
    rs = np.random.RandomState(0)
    x = rs.uniform(size=(B, H * W))
    y0 = np.full((B, H * W), 0.5)
    net32 = net64.to(torch.float32, "cuda")
    yo, Go, _, lo, _, _ = bundle_np.solve_batch(net32.make_fg(x), y0.copy(), nIter=nIter)
    y64 = bundle_np.solve_batch(net64.make_fg(x), y0.copy(), nIter=nIter)[0]
    trace = []
    for as_numpy in (True, False):          # numpy (f, g) like the reference, or CUDA tensors (no host hop for g)
        y, G, h, lam, ys, nIters = be.solveBatch(net32.make_fg(x, as_numpy=as_numpy), y0.copy(), nIter=nIter,
                                                 callback=lambda t, fi, xi: trace.append((t, float(np.mean(fi)))))
        d = np.abs(y - yo).max(axis=1)
        print("conv-PICNN callback mode vs oracle on the same fg: max %.2e median %.2e; vs float64 network: max %.2e"
              % (d.max(), np.median(d), np.abs(y - y64).max()), [len(g) for g in G])
        assert np.median(d) < 1e-6 and np.mean(d < 1e-4) >= 0.75, d
        for u in range(B):
            assert abs(lam[u].sum() - 1) < 1e-6 and 1 <= len(G[u]) <= nIter
    assert [t for t, _ in trace[:nIter]] == list(range(nIter))
