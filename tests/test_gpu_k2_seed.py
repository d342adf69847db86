"""The two-sweep K2 kernel's seeded interior-point iteration 0 and its skipped dependency pass, against ICNN_PC_SEED=0.

By default every solve starts from M0 = 0.25 G G^T, w = 0.5 rowsum and q = M0 z0 taken from the stored unweighted Gram
(no sweep A at it = 0), and the dependency test skips its residual pass when the last pivot of the bordered Cholesky
puts the new row far from the span of the others.  ICNN_PC_SEED=0 runs sweep A at it = 0 and the residual pass
always.  M0, q and w at it = 0 are the same sums in another FP64 order, so the two agree to rounding, and every
decision (counts, permutation, status, iterations) is the same.
"""
import numpy as np
import pytest

from test_gpu_k2_builds import CASES, LARGE, last_launch, max_affine_fg, orthogonal_fg, planned, r32

pytestmark = pytest.mark.gpu
np.seterr(all="ignore")

ENV = ("ICNN_K2_SMALL", "ICNN_K2_PC", "ICNN_PC_V3", "ICNN_K2_WPS", "ICNN_K2_CS", "ICNN_K2_RESIDENT", "ICNN_PC_LEGACY",
       "ICNN_PC_PREFETCH", "ICNN_PC_SEED")
ST_RANK_STOP = 2


@pytest.fixture(autouse=True)
def clean_env(monkeypatch):
    for k in ENV:
        monkeypatch.delenv(k, raising=False)


def solve(fg, n, B, nIter, monkeypatch, seed, **kw):
    """solveBatch (PC, callback mode) with the seeded path on or off; returns the outcome and the build that ran."""
    from icnn_b200 import bundle_entropy as be
    if seed:
        monkeypatch.delenv("ICNN_PC_SEED", raising=False)
    else:
        monkeypatch.setenv("ICNN_PC_SEED", "0")
    r = be.solveBatch(fg, np.full((B, n), 0.5), nIter=nIter, return_state=True, **kw)
    st = r[6]
    out = dict(y=np.array(r[0]), lam=st.lam.cpu().numpy(), count=st.count.cpu().numpy(), perm=st.perm.cpu().numpy(),
               status=st.status.cpu().numpy(), finished=st.finished.cpu().numpy(), nIters=np.array(r[5]))
    return out, last_launch()


def assert_same_decisions(a, b):
    for key in ("count", "perm", "status", "finished", "nIters"):
        np.testing.assert_array_equal(a[key], b[key], err_msg=key)


# every two-sweep build of test_gpu_k2_builds.py, with its piecewise-linear fg (k >= 41 in the LARGE cases)
BUILDS = {"%s-random" % c: CASES[c] + (max_affine_fg,) for c in CASES if c.startswith("two-")}
BUILDS.update({"%s-k%d" % (c, LARGE[c][2]): LARGE[c] + (orthogonal_fg,) for c in LARGE if c.startswith("two-")})


@pytest.mark.parametrize("cid", list(BUILDS))
def test_seeded_iteration_matches_explicit_passes(cid, monkeypatch):
    n, B, nIter, variant, want, kmin, env, make_fg = BUILDS[cid]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    KS = min(nIter, n) + 1
    plan = planned(n, KS, variant)
    assert plan[:6] == want, (plan, want)
    new, ran = solve(make_fg(n, B), n, B, nIter, monkeypatch, True)
    assert ran == plan, (ran, plan)
    ref, ran0 = solve(make_fg(n, B), n, B, nIter, monkeypatch, False)
    assert ran0 == plan, (ran0, plan)
    assert_same_decisions(new, ref)
    assert new["count"].max() >= kmin, (new["count"], kmin)
    dy, dl = np.abs(new["y"] - ref["y"]).max(), np.abs(new["lam"] - ref["lam"]).max()
    print("%s: ran %s, counts %s, max |dy*| %.2e, max |dlambda| %.2e" % (cid, ran, list(new["count"]), dy, dl))
    assert dy <= 1e-12 and dl <= 1e-12, (dy, dl)


def near_span_fg(n, B, m, dists, conds, seed=0):
    """Sample u gets m rows whose Gram has condition number conds[u] (singular values of the row matrix geometric from
    1 to conds[u]^-1/2, scaled by 10), then, at call m, a row at relative distance dists[u] from their span (a random
    combination of them plus dists[u] times its norm along a unit vector orthogonal to the span); afterwards random
    rows.  Rows are float32-representable (returned as float64, so the default rank_tol stays the float64 one); f = g y
    + 1 (every cut offset h = 1)."""
    rs = np.random.RandomState(seed)
    rows = np.zeros((B, m + 1, n))
    for u in range(B):
        U, _ = np.linalg.qr(rs.randn(m, m))
        V, _ = np.linalg.qr(rs.randn(n, m + 1))
        sv = 10.0 * np.geomspace(1.0, conds[u] ** -0.5, m)
        R = r32((U * sv).dot(V[:, :m].T))
        c = rs.randn(m)
        base = c.dot(R)
        rows[u, :m] = R
        rows[u, m] = r32(base + dists[u] * np.linalg.norm(base) * V[:, m])
    calls = [0]

    def fg(y):
        t = calls[0]
        calls[0] += 1
        g = rows[:, t] if t <= m else r32(rs.randn(B, n))
        return np.einsum("bn,bn->b", g, y) + 1.0, g.copy()
    return fg


@pytest.mark.parametrize("n", [100, 3000], ids=["1x1", "v3-8x4"])
@pytest.mark.parametrize("tol", ["default", "float32", "rl"])
def test_dependency_decision_near_thresholds(n, tol, monkeypatch):
    """New rows at relative distance 1e-1 ... 1e-9 from the span of 6 rows whose Gram has cond 1 ... 1e6, under the
    default rank_tol (16 max(KS, n) eps64), the float32 value max(KS, n) eps32 and the RL value 1e-3: the same
    statuses, counts and permutations as the explicit residual pass."""
    m, nIter = 6, 9
    dists = 10.0 ** -np.arange(1, 10)
    conds = 10.0 ** np.arange(0, 7, 2)
    dd, cc = [a.ravel() for a in np.meshgrid(dists, conds)]
    B = len(dd)
    KS = min(nIter, n) + 1
    rank_tol = {"default": None, "float32": max(KS, n) * np.finfo(np.float32).eps, "rl": 1e-3}[tol]
    new, _ = solve(near_span_fg(n, B, m, dd, cc), n, B, nIter, monkeypatch, True, rank_tol=rank_tol)
    ref, _ = solve(near_span_fg(n, B, m, dd, cc), n, B, nIter, monkeypatch, False, rank_tol=rank_tol)
    assert_same_decisions(new, ref)
    stopped = new["status"] == ST_RANK_STOP
    print("rank_tol %s, n_y %d: rank stops at (dist, cond) %s" % (tol, n, list(zip(dd[stopped], cc[stopped]))))
    assert not stopped.all()
    if tol != "default":   # float32 rows sit ~1e-7 off any span: only the larger tolerances stop on them
        assert stopped.any()


def zero_rd_fg(n, B, seed=0):
    """Rows with an exactly zero sum (entries +-a in pairs) and f = g y (float64), so h = f - g y is 0 to rounding and
    rd = w + h - t + s = 0.5 rowsum + h is at the start of every interior-point solve: sqrt(dr) < 1e-6, the seeded
    iteration 0 is declined and the sample takes sweep A at it = 0."""
    rs = np.random.RandomState(seed)

    def fg(y):
        a = r32(rs.uniform(0.5, 1.0, (B, n // 2)) * rs.choice([-1.0, 1.0], (B, n // 2)))
        g = np.concatenate([a, -a], axis=1)[:, rs.permutation(n)]
        return np.einsum("bn,bn->b", g, y), g
    return fg


@pytest.mark.parametrize("n", [100, 3000], ids=["1x1", "v3-8x4"])
def test_zero_dual_residual_takes_the_explicit_passes(n, monkeypatch):
    """rd = 0 at it = 0: the result is the explicit passes' bit for bit (the dependency test's skipped residual pass
    does not change a result, only a decision, and the decisions are equal)."""
    B, nIter = 4, 8
    new, ran = solve(zero_rd_fg(n, B), n, B, nIter, monkeypatch, True)
    ref, _ = solve(zero_rd_fg(n, B), n, B, nIter, monkeypatch, False)
    print("n_y %d: ran %s, counts %s, nIters %s" % (n, ran, list(new["count"]), list(new["nIters"])))
    assert_same_decisions(new, ref)
    np.testing.assert_array_equal(new["y"], ref["y"])
    np.testing.assert_array_equal(new["lam"], ref["lam"])
