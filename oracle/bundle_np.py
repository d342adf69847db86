"""numpy float64 restatement of the reference's bundle-entropy inner loop (all three copies).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py): the checker for the CUDA path and the timed
CPU baseline of bench.py.  Written from the algorithms in SURVEY.md Appendix C, following
(paths relative to the locuslab/icnn repository):

  variant 'lib'  : lib/bundle_entropy.py        solveBatch :192-242, pdipm_pc :5-78,
                                                 pdipm_boyd :80-156, get_step :158-163
  variant 'dual' : lib/bundle_entropy_dual.py   solveBatch :129-179, proj_newton_logistic :15-85
  variant 'rl'   : RL/src/bundle_entropy.py     solveBatch :85-136,  proj_newton_logistic :14-83

Pinned against the reference itself: oracle/gen_golden.py imports the three reference modules
unchanged (they only need numpy/scipy), runs them on seeded inputs and commits the outputs
under tests/golden/; tests/test_oracle_golden.py checks this file against those vectors.

Deliberate restatement differences (documented, result-preserving):
  * the per-sample weight matrix diag(y(1-y)) is never materialised as a dense n x n array
    (the reference does, lib/bundle_entropy.py:17-18) -- identical arithmetic up to BLAS
    summation order, O(kn) instead of O(kn^2); ``dense_diag=True`` re-enables the reference's
    cost model for baseline timing;
  * nothing is printed (the reference prints one line per interior-point iteration, :34-36).
"""
from __future__ import annotations

import numpy as np

# --------------------------------------------------------------------------------------------
# per-sample solvers
# --------------------------------------------------------------------------------------------


def max_step(v, dv):
    """Largest a with v + a*dv >= 0 over entries with dv < 0, else 1 (lib/bundle_entropy.py:158-163)."""
    neg = dv < 0
    if np.any(neg):
        return np.min(-v[neg] / dv[neg])
    return 1.0


def pdipm_pc(G, h, dense_diag=False, stats=None, verbose=False):
    """Mehrotra predictor-corrector for
         min_{y in (0,1)^n, t}  t + sum y log y + (1-y) log(1-y)   s.t.  G y + h <= t 1
    (lib/bundle_entropy.py:5-78).  Returns (y, z) with z the multipliers (= lambda)."""
    k, n = G.shape
    z = np.ones(k) / k
    y = np.full(n, 0.5)
    s = np.ones(k)
    t = 1.0
    ones = np.ones(k)
    for it in range(20):
        ry = np.log(y) - np.log(1.0 - y) + G.T.dot(z)
        rt = 1.0 - np.sum(z)
        rc = z
        rd = G.dot(y) + h - t * ones + s
        pri = np.linalg.norm(np.concatenate([ry, [rt]]))
        dua = np.linalg.norm(rd)
        if pri < 1e-8 and dua < 1e-8:
            if stats is not None:
                stats.append(it)
            return y, z
        if verbose:   # the reference prints this line every iteration (lib/bundle_entropy.py:30-36)
            d_ = z / s
            print(("primal_res = {0:.5g}, dual_res = {1:.5g}, " + "gap = {2:.5g}, kappa(d) = {3:.5g}").format(
                pri, dua, s.dot(z) / k, min(d_) / max(d_)))
        w = 1.0 / (1.0 / y + 1.0 / (1.0 - y))
        if dense_diag:
            # the reference's cost model: BOTH dense n x n diagonal matrices are built every iteration
            # (lib/bundle_entropy.py:17-18) and G.dot(hess_negH_inv) is a dense k x n x n product (:41,46)
            hess_negH = np.diag(1.0 / y + 1.0 / (1.0 - y))   # noqa: F841  (built and unused, as in the reference)
            Dm = np.diag(w)
            GD = G.dot(Dm)
        else:
            GD = G * w
        M = GD.dot(G.T) + np.diag(s / z)
        Lc = np.linalg.cholesky(M)

        def csolve(r):
            return np.linalg.solve(Lc.T, np.linalg.solve(Lc, r))

        Minv1 = csolve(ones)

        def kkt(ry_, rt_, rc_, rd_):
            if dense_diag:   # :46 recomputes G.dot(hess_negH_inv) in every solve, :50 multiplies by the dense matrix
                r = rd_ - G.dot(Dm).dot(ry_) - (s / z) * rc_
            else:
                r = rd_ - GD.dot(ry_) - (s / z) * rc_
            dt = (r.dot(Minv1) - rt_) / Minv1.sum()
            dz = csolve(r - dt)
            ds = -(s / z) * (rc_ + dz)
            dy = -Dm.dot(ry_ + G.T.dot(dz)) if dense_diag else -w * (ry_ + G.T.dot(dz))
            return dt, dz, ds, dy

        dt_a, dz_a, ds_a, dy_a = kkt(ry, rt, rc, rd)
        alpha = min(max_step(z, dz_a), max_step(s, ds_a), max_step(y, dy_a),
                    max_step(1.0 - y, -dy_a), 1.0)
        sig = (np.dot(s + alpha * ds_a, z + alpha * dz_a) / np.dot(s, z)) ** 3
        mu = np.dot(s, z) / k
        rc2 = -(mu * sig * ones - ds_a * dz_a) / s
        dt_c, dz_c, ds_c, dy_c = kkt(np.zeros(n), 0.0, rc2, np.zeros(k))
        dy, dt, ds, dz = dy_a + dy_c, dt_a + dt_c, ds_a + ds_c, dz_a + dz_c
        alpha = max(0.0, min(1.0, 0.99 * min(max_step(s, ds), max_step(z, dz),
                                             max_step(y, dy), max_step(1.0 - y, -dy))))
        y = y + alpha * dy
        t = t + alpha * dt
        s = s + alpha * ds
        z = z + alpha * dz
    if stats is not None:
        stats.append(20)
    return y, z


def pdipm_boyd(G, h):
    """Alternative PDIPM (Boyd & Vandenberghe p.612) on the full KKT system
    (lib/bundle_entropy.py:80-156).  O((n+2k)^3): small cases only."""
    alpha, beta, mu = 0.05, 0.5, 10.0
    k, n = G.shape
    z = np.ones(k) / k
    y = np.full(n, 0.5)
    t = np.max(G.dot(y) + h) + 1.0
    s = -G.dot(y) - h + t

    for _ in range(20):
        gap = s.dot(z) / k
        u = mu / gap

        def res(y_, t_, s_, z_):
            return (np.log(y_) - np.log(1.0 - y_) + G.T.dot(z_), 1.0 - np.sum(z_),
                    s_ * z_ + 1.0 / u, G.dot(y_) + h - t_ + s_)

        ry, rt, rc, rd = res(y, t, s, z)
        if np.linalg.norm(np.concatenate([ry, [rt]])) < 1e-8 and np.linalg.norm(rd) < 1e-8:
            return y, z
        N = n + 1 + 2 * k
        A = np.zeros((N, N))
        A[:n, :n] = np.diag(1.0 / y + 1.0 / (1.0 - y))
        A[:n, n + 1 + k:] = G.T
        A[n, n + 1 + k:] = -1.0
        A[n + 1:n + 1 + k, n + 1:n + 1 + k] = np.diag(z)
        A[n + 1:n + 1 + k, n + 1 + k:] = np.diag(s)
        A[n + 1 + k:, :n] = G
        A[n + 1 + k:, n] = -1.0
        A[n + 1 + k:, n + 1:n + 1 + k] = np.eye(k)
        r = np.concatenate([ry, [rt], rc, rd])
        dvec = np.linalg.solve(A, -r)
        dy, dt, ds, dz = np.split(dvec, [n, n + 1, n + 1 + k])
        dt = dt[0]
        step = min(1.0, 0.99 * min(max_step(s, ds), max_step(z, dz), max_step(y, dy),
                                   max_step(1.0 - y, -dy)))

        def upd(st):
            return y + st * dy, t + st * dt, s + st * ds, z + st * dz

        def infeasible(st):
            yp, tp, sp_, zp = upd(st)
            return np.all(G.dot(yp) + h - tp + sp_ >= 0)

        def insufficient(st):
            rp = np.concatenate([np.atleast_1d(v) for v in res(*upd(st))])
            return np.linalg.norm(rp) > (1.0 - alpha * st) * np.linalg.norm(r)

        while infeasible(step):
            step *= beta
        while insufficient(step):
            step *= beta
        y, t, s, z = upd(step)
    return y, z


def softplus(x):
    """Numerically stable log(1+exp(x)) (lib/bundle_entropy_dual.py:6-12)."""
    out = np.empty_like(x)
    big = x > 1
    out[big] = np.log1p(np.exp(-x[big])) + x[big]
    out[~big] = np.log1p(np.exp(x[~big]))
    return out


class NewtonFailure(Exception):
    pass


def proj_newton_logistic(A, b, rl=False, line_search=None, stats=None):
    """min_{lam in simplex} -(A 1 + b)^T lam + sum_j log(1 + exp((A^T lam)_j)) by projected
    Newton with the simplex eliminated through the pivot p = argmax(lam).
    lib/bundle_entropy_dual.py:15-85; ``rl=True`` gives RL/src/bundle_entropy.py:14-83
    (20 iterations, line search on, pre-scaled first step, 10 backtracks, swallowed solve
    failure)."""
    if line_search is None:
        line_search = bool(rl)
    k = A.shape[0]
    c = np.sum(A, axis=1) + b
    e = np.ones(k)
    lam = np.ones(k) / k
    n_outer = 20 if rl else 100
    n_back = 10 if rl else 50
    for it in range(n_outer):
        a = A.T.dot(lam)
        zz = 1.0 / (1.0 + np.exp(-a))
        F = -c.dot(lam) + np.sum(softplus(a))
        g = -c + A.dot(zz)
        H = (A * (zz * (1.0 - zz))).dot(A.T)
        p = int(np.argmax(lam))
        yv = lam.copy()
        yv[p] = 1.0
        e[p] = 0.0
        g0 = g - e * g[p]
        H0 = H - np.outer(e, H[:, p]) - np.outer(H[:, p], e) + H[p, p] * np.outer(e, e)
        bound = (yv <= 1e-12) & (g0 > 0)
        bound[p] = True
        free = ~bound
        if np.linalg.norm(g0[free]) < 1e-10:
            if stats is not None:
                stats.append(it)
            return lam
        d = np.zeros(k)
        try:
            d[free] = np.linalg.solve(H0[free][:, free], -g0[free])
        except np.linalg.LinAlgError:
            if rl:
                break
            raise NewtonFailure("singular reduced Hessian")
        tau = min(1.0 / np.max(np.abs(d)), 1.0) if rl else 1.0
        lam_n = lam
        for _ in range(n_back):
            yn = np.maximum(yv + tau * d, 0.0)
            yn[p] = 1.0
            lam_n = yn.copy()
            lam_n[p] = 1.0 - e.dot(yn)
            if lam_n[p] >= 0:
                if line_search:
                    Fn = -c.dot(lam_n) + np.sum(softplus(A.T.dot(lam_n)))
                    if Fn < F + tau * 1e-5 * d.dot(g0):
                        break
                else:
                    break
            small = (np.max(tau * np.abs(d)) < 1e-10) if rl else (tau < 1e-10)
            if small:
                if stats is not None:
                    stats.append(it + 1)
                return lam_n
            tau *= 0.5
        e[p] = 1.0
        lam = lam_n.copy()
    if stats is not None:
        stats.append(n_outer)
    return lam


# --------------------------------------------------------------------------------------------
# batch driver
# --------------------------------------------------------------------------------------------


def solve_batch(fg, initXs, nIter=None, callback=None, solver="pc", variant="lib",
                dense_diag=False, line_search=None, stats=None, verbose=False):
    """The outer bundle loop shared by the three copies (SURVEY.md Appendix C.2).

    variant 'lib'  -> lib/bundle_entropy.py:192-242   (PC / Boyd solve, prune lam <= 1e-8,
                                                       SVD rank stop, callback(t, f, x))
    variant 'dual' -> lib/bundle_entropy_dual.py:129-179 (dual Newton, k=1 shortcut, prune lam<=0)
    variant 'rl'   -> RL/src/bundle_entropy.py:85-136 (nIter 5, clip [.03,.97], |dy|<1e-6 stop,
                                                       no rank test, callback(t, f))
    ``initXs`` is mutated in place exactly like the reference (x = initXs, :200).
    Returns (x, A, b, lam, xs, nIters)."""
    if variant not in ("lib", "dual", "rl"):
        raise ValueError(variant)
    if nIter is None:
        nIter = 5 if variant == "rl" else 10
    if variant == "lib" and solver not in ("pc", "boyd"):
        raise RuntimeError("Solver unknown: " + solver)
    B = initXs.shape[0]
    A = [[] for _ in range(B)]
    b = [[] for _ in range(B)]
    xs = [[] for _ in range(B)]
    lam = [None] * B
    thr = 1e-8 if variant == "lib" else 0.0
    x = initXs
    finished = np.zeros(B, dtype=bool)
    nIters = [nIter] * B
    for t in range(nIter):
        fi, gi = fg(x)
        bi = fi - np.sum(gi * x, axis=1)
        if callback is not None:
            if variant == "rl":
                callback(t, fi)
            else:
                callback(t, fi, x)
        for u in range(B):
            if finished[u]:
                continue
            A[u].append(gi[u])
            b[u].append(bi[u])
            xs[u].append(np.copy(x[u]))
            Au = np.array(A[u])
            if variant != "rl" and np.linalg.matrix_rank(Au) < len(A[u]):
                del A[u][-1], b[u][-1], xs[u][-1]
                finished[u] = True
                nIters[u] = t - 1
                continue
            bu = np.array(b[u])
            if variant == "lib":
                if solver == "pc":
                    x[u], lam[u] = pdipm_pc(Au, bu, dense_diag=dense_diag, stats=stats, verbose=verbose)
                else:
                    x[u], lam[u] = pdipm_boyd(Au, bu)
            else:
                prev = x[u].copy()
                if len(A[u]) > 1:
                    lam[u] = proj_newton_logistic(Au, bu, rl=(variant == "rl"),
                                                  line_search=line_search, stats=stats)
                    x[u] = 1.0 / (1.0 + np.exp(Au.T.dot(lam[u])))
                else:
                    lam[u] = np.array([1.0])
                    x[u] = 1.0 / (1.0 + np.exp(A[u][0]))
                if variant == "rl":
                    x[u] = np.clip(x[u], 0.03, 0.97)
                    if np.max(np.abs(prev - x[u])) < 1e-6:
                        finished[u] = True
            keep = lam[u] > thr
            A[u] = [r for r, kk in zip(A[u], keep) if kk]
            b[u] = [r for r, kk in zip(b[u], keep) if kk]
            xs[u] = [r for r, kk in zip(xs[u], keep) if kk]
            lam[u] = lam[u][keep]
        if finished.all():
            break
    return x, A, b, lam, xs, nIters


def neg_entropy(y):
    """sum y log y + (1-y) log(1-y)  (lib/bundle_entropy.py:165-166)."""
    return np.sum(y * np.log(y) + (1.0 - y) * np.log(1.0 - y))
