"""Every K2 build the dispatch can select, against the float64 oracle, with the build that ran asserted.

Callback mode: the oracle and K2 are fed the same float32-representable (f, g), so K2 is isolated (as in
test_gpu_bundle.py::test_k2_pc_matches_oracle).  Each case
  * asserts with icnn_k2_last_launch that the build it names ran (family, warps, chunks | cluster size, V3, 16-byte
    rows, resident rows), and that icnn_k2_plan predicts the same build;
  * asserts >= 95 % of the samples with the oracle's counts and nIters, y* within 1e-9 on those and lambda / h / rows /
    xs as test_k2_pc_matches_oracle does;
  * asserts that the bundle reached the k range the case was written for (max len(G[u])): k >= 33 runs the
    two-rows-per-lane k x k stage (K32 = false); k + 2 > 40 (two-sweep) and k > 40 (five-sweep) the Gram
    composition of rb >= 6 row blocks.

The fgs are piecewise linear (a maximum of affine pieces, like the workload PICNNs), rounded to float32: a bundle row
is one piece's slope, so the oracle and the device store the same rows bit for bit and the trajectories agree to 1e-9.
  * random pieces (max_affine_fg): bundles stop on an exactly repeated row after 10-20 iterations, which is enough for
    the warp counts, launch variables and limits;
  * near-orthogonal pieces, a_m = 8 e_(i_m) + 2 w + N(0, 0.05^2 / n) on distinct coordinates (orthogonal_fg): nearly
    every iteration adds a row, so k reaches 33-63, and G D G^T (D = y (1 - y)) stays below cond ~10.  These cases reach k >= 33 (the
    two-rows-per-lane k x k stage, K32 = false) and k >= 41 (Gram composition of rb >= 6 row blocks) in every build
    and are held to the same 1e-9.
A sample whose trajectory leaves the oracle's may be set aside only when its final G D G^T has cond > 1e9, at most one
per case.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import argmin_grad_np, bundle_np

pytestmark = pytest.mark.gpu
np.seterr(all="ignore")

SMALL, TWO, FIVE = 0, 1, 2
ENV = ("ICNN_K2_SMALL", "ICNN_K2_PC", "ICNN_PC_V3", "ICNN_K2_WPS", "ICNN_K2_CS", "ICNN_K2_RESIDENT", "ICNN_PC_LEGACY")


def five(wps, cs=1, vec=1, res=0):
    return (FIVE, wps, cs, 0, vec, res)


def two(wps, nch, vec=1, v3=0):
    return (TWO, wps, nch, v3, vec, 0)


def r32(a):
    return a.astype(np.float32).astype(np.float64)


def lse_fg(n, B, M=300, temp=1.0, scale=10.0, seed=0):
    """Per sample f(y) = temp * logsumexp((A y + b) / temp) over M pieces, slopes N(0, scale^2 / n); f and g rounded
    to float32 (both sides see the same numbers)."""
    rs = np.random.RandomState(seed)
    A = r32(rs.randn(B, M, n) * scale / np.sqrt(n))
    b = r32(rs.randn(B, M))

    def fg(y):
        v = (np.einsum("bmn,bn->bm", A, y) + b) / temp
        mx = v.max(1, keepdims=True)
        e = np.exp(v - mx)
        s = e.sum(1, keepdims=True)
        return r32(temp * (np.log(s[:, 0]) + mx[:, 0])), r32(np.einsum("bm,bmn->bn", e / s, A))
    return fg


def max_affine_fg(n, B, M=2000, scale=10.0, seed=0):
    """Per sample f(y) = max_m (a_m . y + b_m), g = the slope of the maximising piece; slopes N(0, scale^2 / n)."""
    rs = np.random.RandomState(seed)
    A = rs.randn(B, M, n).astype(np.float32)
    A *= np.float32(scale / np.sqrt(n))
    A = A.astype(np.float64)
    b = r32(rs.randn(B, M))
    rows = np.arange(B)

    def fg(y):
        v = np.einsum("bmn,bn->bm", A, y) + b
        i = v.argmax(1)
        return r32(v[rows, i]), A[rows, i].copy()
    return fg


def orthogonal_fg(n, B, P=64, seed=0):
    """Per sample f(y) = max_m (a_m . y + b_m) over min(P, n) pieces a_m = 8 e_(i_m) + 2 w + N(0, 0.05^2 / n) with
    distinct coordinates i_m, one unit vector w shared by every piece and b_m = N(0, 0.1^2): the bundle gains one
    well-separated row per iteration.  The shared 2 w leaves the maximising piece unchanged and couples every pair of
    rows, so the Cholesky factor of G D G^T has off-diagonal entries of a few % (a solve that drops one is visibly
    wrong) while cond(G D G^T) stays below ~10."""
    P = min(P, n)
    rs = np.random.RandomState(seed)
    A = np.zeros((B, P, n))
    for u in range(B):
        A[u, np.arange(P), rs.choice(n, P, replace=False)] = 8.0
    w = rs.randn(n)
    A = r32(A + rs.randn(B, P, n) * 0.05 / np.sqrt(n) + 2.0 * w / np.linalg.norm(w))
    b = r32(0.1 * rs.randn(B, P))
    rows = np.arange(B)

    def fg(y):
        v = np.einsum("bmn,bn->bm", A, y) + b
        i = v.argmax(1)
        return r32(v[rows, i]), A[rows, i].copy()
    return fg


@pytest.fixture(autouse=True)
def clean_env(monkeypatch):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)


def last_launch():
    from icnn_b200 import _capi
    out = (C.c_int32 * _capi.K2_PLAN_LEN)()
    assert _capi.lib.icnn_k2_last_launch(out) == 0
    return tuple(out)


def planned(n, KS, variant):
    from icnn_b200 import _capi
    out = (C.c_int32 * _capi.K2_PLAN_LEN)()
    solver = _capi.SOLVER_PC if variant == "lib" else _capi.SOLVER_NEWTON
    assert _capi.lib.icnn_k2_plan(n, KS, solver, _capi.VARIANT[variant], out) == 0, _capi.lib.icnn_last_error()
    return tuple(out)


def lens(rows):
    return np.array([len(r) for r in rows])


def cond_gdg(y, G):
    G = np.array(G, dtype=np.float64)
    return np.linalg.cond((G * (y * (1.0 - y))).dot(G.T)) if len(G) else 1.0


def solve_both(fg, n, B, nIter, variant):
    from icnn_b200 import bundle_entropy as be
    y0 = np.full((B, n), 0.5)
    kw = dict(solver="pc") if variant == "lib" else {}
    o = bundle_np.solve_batch(fg, y0.copy(), nIter=nIter, variant=variant, **kw)
    r = be.solveBatch(fg, y0.copy(), nIter=nIter, variant=variant, return_state=True, **kw)
    return o, r


def check_against_oracle(o, r, kmin, ytol=1e-9):
    """The assertions of test_k2_pc_matches_oracle plus the cond > 1e9 set-aside and the bundle-size check."""
    B = len(o[5])
    same = (lens(r[1]) == lens(o[1])) & (np.array(r[5]) == np.array(o[5]))
    d = np.abs(r[0] - o[0]).max(axis=1)
    off = np.flatnonzero(~same | (d >= ytol))
    aside = [u for u in off if cond_gdg(o[0][u], o[1][u]) > 1e9]
    for u in off:
        print("sample %d: k device %d oracle %d, nIters %d / %d, |dy*| %.2e, cond(G D G^T) %.2e"
              % (u, len(r[1][u]), len(o[1][u]), r[5][u], o[5][u], d[u], cond_gdg(o[0][u], o[1][u])))
    assert len(aside) <= 1 and len(aside) == len(off), (off, aside)
    keep = np.setdiff1d(np.arange(B), aside)
    assert same[keep].mean() >= 0.95
    assert d[keep].max() < ytol
    for u in keep[:8]:
        if len(o[1][u]):
            np.testing.assert_allclose(r[3][u], o[3][u], atol=1e-8)
            np.testing.assert_allclose(np.array(r[2][u]), np.array(o[2][u]), atol=1e-9)
            np.testing.assert_allclose(np.array(r[1][u]), np.array(o[1][u]), atol=0)
            np.testing.assert_allclose(np.array(r[4][u]), np.array(o[4][u]), atol=1e-9)
    kmax = max(lens(r[1]))
    assert kmax >= kmin, (kmax, kmin, list(lens(r[1])))
    return kmax


def run_case(n, B, nIter, variant, want, kmin, env, monkeypatch, fg=None, **fgkw):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    KS = (nIter if variant == "rl" else min(nIter, n)) + 1
    plan = planned(n, KS, variant)
    assert plan[:6] == want, (plan, want)
    o, r = solve_both(fg or lse_fg(n, B, **fgkw), n, B, nIter, variant)
    ran = last_launch()
    assert ran == plan, (ran, plan)
    print("n_y %d KS %d %s: ran %s, k device %s" % (n, KS, variant, ran, list(lens(r[1]))))
    return o, r


# id -> (n_y, B, nIter, variant, build, k reached, environment); piecewise-linear fg
CASES = {
    # five-sweep kernel, PC and dual Newton, at every warp count
    "five-1w-pc": (100, 8, 20, "lib", five(1), 3, {"ICNN_K2_PC": "legacy"}),
    "five-2w-pc": (300, 8, 20, "lib", five(2), 3, {}),
    "five-4w-pc": (800, 6, 20, "lib", five(4), 3, {}),
    "five-8w-pc": (1500, 3, 20, "lib", five(8), 3, {"ICNN_K2_PC": "legacy"}),
    "five-16w-pc": (5000, 2, 12, "lib", five(16), 3, {"ICNN_K2_PC": "legacy"}),
    "five-1w-dual": (100, 8, 20, "dual", five(1), 2, {}),
    "five-2w-dual": (300, 8, 20, "dual", five(2), 2, {}),
    "five-4w-dual": (800, 6, 20, "dual", five(4), 2, {}),
    "five-8w-dual": (1500, 3, 20, "dual", five(8), 2, {}),
    "five-16w-dual": (4096, 2, 40, "dual", five(16), 2, {}),
    # eight one-warp samples per CTA hold at most 35 slots at n_y = 100: 41 slots take 2 warps, 4 samples per CTA
    "five-2w-ks41-dual": (100, 8, 40, "dual", five(2), 2, {}),
    # n_y % 4 != 0 above 1024: SIMT Gram, PC falls back to the five-sweep kernel
    "five-8w-simt-1025-pc": (1025, 3, 20, "lib", five(8, vec=0), 3, {}),
    "five-8w-simt-2050-pc": (2050, 3, 20, "lib", five(8, vec=0), 3, {}),
    "five-8w-simt-2050-dual": (2050, 3, 20, "dual", five(8, vec=0), 2, {}),
    # two-sweep kernel, every build
    "two-1x1": (100, 8, 20, "lib", two(1, 1), 3, {}),
    "two-1x1-scalar": (90, 8, 20, "lib", two(1, 1, vec=0), 3, {}),
    "two-1x2": (200, 8, 20, "lib", two(1, 2), 3, {}),
    "two-1x2-scalar": (198, 8, 20, "lib", two(1, 2, vec=0), 3, {}),
    "two-8x2": (1500, 3, 20, "lib", two(8, 2), 3, {}),
    "two-v3-8x4": (3000, 2, 20, "lib", two(8, 4, v3=1), 3, {}),
    "two-16x2": (4096, 2, 52, "lib", two(16, 2), 3, {}),
    "two-16x4": (5000, 2, 20, "lib", two(16, 4), 3, {}),
    # thread-per-sample kernel boundary
    "small-n8": (8, 16, 8, "lib", (SMALL, 0, 0, 0, 0, 0), 1, {}),
    "two-n9": (9, 16, 9, "lib", two(1, 1, vec=0), 1, {}),
}


@pytest.mark.parametrize("cid", list(CASES))
def test_k2_build_matches_oracle(cid, monkeypatch):
    n, B, nIter, variant, want, kmin, env = CASES[cid]
    o, r = run_case(n, B, nIter, variant, want, kmin, env, monkeypatch, fg=max_affine_fg(n, B))
    check_against_oracle(o, r, kmin)


# id -> (n_y, B, nIter, variant, build, k reached, environment); near-orthogonal fg, k = nIter
LARGE = {
    # five-sweep kernel: one warp holds at most 35 slots at n_y = 100 (k = 34); 2 / 4 / 8 / 16 warps with k >= 41
    "five-1w-k34-pc": (100, 4, 34, "lib", five(1), 33, {"ICNN_K2_PC": "legacy"}),
    "five-1w-k34-dual": (100, 4, 34, "dual", five(1), 33, {}),
    "five-2w-k45-pc": (300, 4, 45, "lib", five(2), 41, {}),
    "five-8w-k45-pc": (1500, 2, 45, "lib", five(8), 41, {"ICNN_K2_PC": "legacy"}),
    "five-16w-k40-dual": (4096, 2, 40, "dual", five(16), 33, {}),
    # KS = 63 / 64 with PC: the natural five-sweep fallback (4 warps at small n_y: 8 / 4 samples do not fit a CTA)
    "five-4w-ks63-n100": (100, 4, 62, "lib", five(4), 41, {}),
    "five-4w-ks64-n200": (200, 4, 63, "lib", five(4), 41, {}),
    "five-8w-ks63-n1500": (1500, 2, 62, "lib", five(8), 41, {}),
    "five-16w-ks64-n2048": (2048, 2, 63, "lib", five(16), 41, {}),
    # two-sweep kernel, every build: k + 2 > 40 sweep rows (rb = 6 ... 8)
    "two-1x1": (100, 4, 61, "lib", two(1, 1), 41, {}),
    "two-1x1-scalar": (90, 4, 61, "lib", two(1, 1, vec=0), 41, {}),
    "two-1x2": (200, 4, 61, "lib", two(1, 2), 41, {}),
    "two-1x2-scalar": (198, 4, 61, "lib", two(1, 2, vec=0), 41, {}),
    "two-8x2": (1500, 2, 45, "lib", two(8, 2), 41, {}),
    "two-v3-8x4": (3000, 2, 45, "lib", two(8, 4, v3=1), 41, {}),
    "two-16x2": (4096, 2, 52, "lib", two(16, 2), 41, {}),
    "two-16x4": (5000, 2, 45, "lib", two(16, 4), 41, {}),
}


@pytest.mark.parametrize("cid", list(LARGE))
def test_k2_large_bundle_build_matches_oracle(cid, monkeypatch):
    n, B, nIter, variant, want, kmin, env = LARGE[cid]
    o, r = run_case(n, B, nIter, variant, want, kmin, env, monkeypatch, fg=orthogonal_fg(n, B))
    check_against_oracle(o, r, kmin)


# The launch variables of the five-sweep kernel, where they take effect: the PC solver under ICNN_K2_PC=legacy, or the
# dual Newton solver.  Rows resident in shared memory, the sample split over a 2 / 4 / 8-CTA cluster (DSMEM exchanges),
# 16 warps per sample.
VARIANTS = {
    "resident-1w-pc": (159, 8, 10, "lib", five(1, vec=0, res=1), {"ICNN_K2_PC": "legacy", "ICNN_K2_RESIDENT": "1"}),
    "resident-2w-pc": (512, 8, 10, "lib", five(2, res=1), {"ICNN_K2_PC": "legacy", "ICNN_K2_RESIDENT": "1"}),
    "resident-cs2-dual": (2048, 3, 12, "dual", five(8, cs=2, res=1), {"ICNN_K2_RESIDENT": "1"}),
    "resident-cs8-pc": (4096, 2, 12, "lib", five(8, cs=8, res=1),
                        {"ICNN_K2_PC": "legacy", "ICNN_K2_RESIDENT": "1", "ICNN_K2_CS": "8"}),
    "cs2-pc": (2048, 3, 12, "lib", five(8, cs=2), {"ICNN_K2_PC": "legacy", "ICNN_K2_CS": "2"}),
    "cs4-dual": (2048, 3, 12, "dual", five(8, cs=4), {"ICNN_K2_CS": "4"}),
    "cs8-dual": (2048, 3, 12, "dual", five(8, cs=8), {"ICNN_K2_CS": "8"}),
    "wps16-pc": (2048, 3, 12, "lib", five(16), {"ICNN_K2_PC": "legacy", "ICNN_K2_WPS": "16"}),
    "wps16-dual": (2048, 3, 12, "dual", five(16), {"ICNN_K2_WPS": "16"}),
}


@pytest.mark.parametrize("cid", list(VARIANTS))
def test_k2_launch_variant_matches_oracle(cid, monkeypatch):
    n, B, nIter, variant, want, env = VARIANTS[cid]
    o, r = run_case(n, B, nIter, variant, want, 2, env, monkeypatch, fg=max_affine_fg(n, B))
    check_against_oracle(o, r, 2)


@pytest.mark.parametrize("nIter,want", [(9, (SMALL, 0, 0, 0, 0, 0)), (10, five(1, vec=0))])
def test_rl_small_kernel_boundary(nIter, want, monkeypatch):
    """RL at n_y = 6: KS = nIter + 1 = 10 slots is the thread-per-sample kernel, 11 the five-sweep kernel.  The RL
    Newton stops on |tau d| < 1e-10 / 20 iterations and has no rank test, so summation-order noise shows at 1e-7 on
    this smooth fg (measured: median 1e-8 and 9e-8, max 6e-6); the bound is the 1e-6 that
    test_gpu_bundle.py::test_thread_per_sample_kernel_matches_group_kernel allows RL, max as
    test_k2_rl_matches_oracle."""
    o, r = run_case(6, 64, nIter, "rl", want, 1, {}, monkeypatch, M=20)
    d = np.abs(r[0] - o[0]).max(axis=1)
    assert r[0].min() >= 0.03 and r[0].max() <= 0.97
    assert d.max() < 1e-5 and np.median(d) < 1e-6, (d.max(), np.median(d))


def test_shared_memory_edge_at_8192(monkeypatch):
    """n_y = 8192: the five-sweep kernel holds at most 41 slots.  nIter = 40 (KS = 41) matches the oracle; nIter = 41
    is refused at the first bundle step with the library's message, and the refused step enqueues nothing."""
    import torch
    from icnn_b200 import bundle_entropy as be
    o, r = run_case(8192, 2, 40, "lib", five(16), 4, {}, monkeypatch, fg=max_affine_fg(8192, 2, M=500))
    check_against_oracle(o, r, 4)
    before = last_launch()
    y0 = np.full((2, 8192), 0.5)
    with pytest.raises(RuntimeError, match=r"shared memory does not fit \(n=8192, KS=42\)"):
        be.solveBatch(max_affine_fg(8192, 2, M=500), y0, nIter=41)
    torch.cuda.synchronize()
    assert last_launch() == before


# K3 on states the K3 test of test_gpu_argmin_grad.py does not reach: k >= 33 (gram_pass at rb >= 5, the warp LU with
# m = k + 1 > 32) at 1, 2, 4 and 8 warps per sample, and 63 slots at n_y = 100, where eight one-warp samples no longer
# fit a CTA and K3 takes 4 warps per sample.  Against oracle/argmin_grad_np.py on the device's own state.
@pytest.mark.parametrize("n,B,nIter", [(100, 4, 34), (300, 4, 45), (800, 4, 45), (1500, 2, 45), (100, 4, 62)],
                         ids=["n100-1warp-k34", "n300-2warps-k45", "n800-4warps-k45", "n1500-8warps-k45", "n100-ks63-k62"])
@pytest.mark.parametrize("loss", ["xent", "mse"])
def test_argmin_grad_matches_oracle(n, B, nIter, loss):
    from icnn_b200 import argmin_grad, bundle_entropy as be
    fg = orthogonal_fg(n, B)
    yN, G, h, lam, ys, nIters, st = be.solveBatch(fg, np.full((B, n), 0.5), nIter=nIter, return_state=True)
    assert max(lens(G)) >= 33, list(lens(G))
    trueY = (np.random.RandomState(17).uniform(size=yN.shape) < 0.3).astype(np.float64)
    cy, clam, ct = argmin_grad.argmin_grad(st, trueY, loss=loss, assemble=False)
    checked = 0
    for u in range(B):
        Gu = np.array(G[u], dtype=np.float64)
        ocy, oclam, oct = argmin_grad_np.argmin_grad(yN[u], trueY[u], Gu, loss)
        zinv = 1.0 / (1.0 / np.clip(yN[u], 1e-8, 1 - 1e-8) + 1.0 / (1.0 - np.clip(yN[u], 1e-8, 1 - 1e-8)))
        c = np.linalg.cond((Gu * zinv).dot(Gu.T))
        if c > 1e9:          # the criterion of test_gpu_argmin_grad.py
            print("sample %d (k = %d): cond %.2e, only finiteness checked" % (u, len(Gu), c))
            assert np.all(np.isfinite(cy[u]))
            continue
        checked += 1
        tol = 1e-7 * max(1.0, np.abs(ocy).max(), np.abs(oclam).max())
        np.testing.assert_allclose(cy[u], ocy, atol=tol)
        np.testing.assert_allclose(clam[u][:len(Gu)], oclam, atol=tol)
        np.testing.assert_allclose(ct[u], oct[0], atol=tol)
    assert checked >= B // 2
