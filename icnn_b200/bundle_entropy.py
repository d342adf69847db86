"""Drop-in ``solveBatch`` of the reference's bundle-entropy library, running on an H100.

Reference surfaces reproduced (paths relative to the locuslab/icnn repository):
    lib/bundle_entropy.py:192        solveBatch(fg, initXs, nIter=10, callback=None, solver='pc')
    lib/bundle_entropy_dual.py:129   solveBatch(fg, initXs, nIter=10, callback=None)
    RL/src/bundle_entropy.py:85      solveBatch(fg, initXs, nIter=5,  callback=None)
returning ``(x, A, b, lam, xs, nIters)`` (callers name A, b as G, h:
multi-label-cls/icnn_ebundle.py:225).

Two ways to supply ``fg``:
  * fused mode   -- ``fg`` is a :class:`icnn_b200.BoundPICNN` (``PICNN.bind(x)``): the whole loop
                    (K1 PICNN f/grad kernel + K2 bundle step) runs on the device, no host round
                    trip per iteration;
  * callback mode -- ``fg`` is any Python callable ``fg(x ndarray[B,n]) -> (f[B], g[B,n])``
                    (e.g. a conv-PICNN in torch): one host hop per iteration like the reference,
                    the per-sample bundle work (K2) still runs on the device.
There is no CPU implementation here: without the native library / a CUDA device this raises.
"""
from __future__ import annotations

import ctypes as C
import warnings

import numpy as np
import torch

from . import _capi
from .picnn import BoundPICNN, default_device

__all__ = ["solveBatch", "solve", "BundleState", "VARIANT_DEFAULTS"]

# reference defaults per copy: (nIter, solver, line_search, prune_thr)
VARIANT_DEFAULTS = {
    "lib": dict(nIter=10, line_search=True, prune_thr=1e-8),
    "dual": dict(nIter=10, line_search=False, prune_thr=0.0),
    "rl": dict(nIter=5, line_search=True, prune_thr=0.0),
}
_EPS64 = float(np.finfo(np.float64).eps)


class _Rows:
    """Lazy list-of-lists view over the dense device bundle buffers.  ``rows[u]`` is a Python
    list (what the reference returns) built on first access; fetching everything at once would
    be a multi-GB device->host copy at the stress sizes (SURVEY.md section 7, hard part 7)."""

    def __init__(self, state, kind):
        self._s, self._kind = state, kind
        self._cache = {}

    def __len__(self):
        return self._s.B

    def __getitem__(self, u):
        if isinstance(u, slice):
            return [self[i] for i in range(*u.indices(len(self)))]
        if u < 0:
            u += len(self)
        if not 0 <= u < len(self):
            raise IndexError(u)
        if u not in self._cache:
            self._cache[u] = self._s._fetch(self._kind, u)
        return self._cache[u]

    def __iter__(self):
        return (self[u] for u in range(len(self)))


class BundleState:
    """Device buffers of one solveBatch call (icnn_bundle_bufs in include/icnn_b200.h)."""

    def __init__(self, B, n, KS, device, keep_xs=True, nIter=10, stats=False, keep_f64=False):
        self.B, self.n, self.KS, self.device = int(B), int(n), int(KS), device
        self.nIter, self.keep_xs = int(nIter), bool(keep_xs)
        f32, f64, i32 = torch.float32, torch.float64, torch.int32
        e = lambda *shape, dtype: torch.empty(*shape, dtype=dtype, device=device)  # noqa: E731
        self.y = e(B, n, dtype=f64)
        self.y32 = e(B, n, dtype=f32)
        self.f = e(B, dtype=f32)
        self.G = e(B, KS, n, dtype=f32)
        self.ys = e(B, KS, n, dtype=f64) if keep_xs else None
        self.h = torch.zeros(B, KS, dtype=f64, device=device)
        self.lam = torch.zeros(B, KS, dtype=f64, device=device)
        self.rsum = torch.zeros(B, KS, dtype=f64, device=device)
        self.gram = torch.zeros(B, KS, KS, dtype=f64, device=device)
        self.perm = e(B, KS, dtype=i32)
        self.count = e(B, dtype=i32)
        self.status = e(B, dtype=i32)
        self.finished = e(B, dtype=i32)
        self.nIters = e(B, dtype=i32)
        self.nactive = e(nIter + 1, dtype=i32)
        self.newton_its = e(B, dtype=i32)
        self.ksum = e(B, dtype=i32)
        # optional: float64 f of a float64 callback fg; per-iteration statistics (include/icnn_b200.h)
        self.f64 = e(B, dtype=f64) if keep_f64 else None
        self.iter_stats = torch.zeros(nIter, _capi.NSTAT, dtype=torch.float64, device=device) if stats else None
        # scratch for the measured-and-rejected variant of the predictor-corrector kernel that keeps the per-sample
        # n-vectors in L2 instead of shared memory (include/icnn_b200.h: vec_ws): only
        # allocated when the exploration knob ICNN_PC_GV is set
        import os
        self.vec_ws = e(B, 4, (n + 15) & ~15, dtype=f64) if os.environ.get("ICNN_PC_GV") else None
        p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        self.c = _capi.BundleBufs(self.B, self.n, self.KS, p(self.y), p(self.y32), p(self.f), p(self.G),
                                  p(self.ys), p(self.h), p(self.lam), p(self.rsum), p(self.gram),
                                  p(self.perm), p(self.count), p(self.status), p(self.finished),
                                  p(self.nIters), p(self.nactive), p(self.newton_its), p(self.ksum),
                                  p(self.f64), p(self.iter_stats), p(self.vec_ws))
        self._host = None
        self._pin_y = None
        self._graphs = {}   # captured device loops (solveBatch(graph=True)), keyed on everything the capture bakes in

    _MAX_GRAPHS = 4

    def loop_graph(self, fg, cfg):
        """Captured CUDA graph of the fused loop for (this state, fg's buffers, cfg); captured on first use.
        The key holds every device address / value the capture bakes in, so a hit is always a valid replay."""
        key = (id(fg.net), fg.net._pack_gen, fg.net._h.value, fg.ws.data_ptr(), fg.B,
               tuple(None if t is None else t.data_ptr() for lst in (fg.cy, fg.cz, fg.d) for t in lst),
               (fg.c_gates.in_scale, fg.c_gates.in_shift, fg.c_gates.g_scale),
               bytes(cfg), self.c.iter_stats, self.c.f64)
        g = self._graphs.get(key)
        if g is None:
            while len(self._graphs) >= self._MAX_GRAPHS:
                _, old = self._graphs.popitem()
                _capi.lib.icnn_loop_graph_destroy(old)
            g = C.c_void_p()
            _capi.check(_capi.lib.icnn_loop_graph_create(fg.net._h, C.byref(fg.c_gates), C.byref(cfg), C.byref(self.c),
                                                         fg.ws.data_ptr(), C.byref(g)))
            self._graphs[key] = g
        return g

    def __del__(self):
        for g in getattr(self, "_graphs", {}).values():
            try:
                _capi.lib.icnn_loop_graph_destroy(g)
            except Exception:
                pass
        self._graphs = {}

    def compatible(self, B, n, KS, device, keep_xs, nIter, stats, keep_f64):
        """True if this state can be reused (``solveBatch(..., state=st)``) for a problem of that shape."""
        return (self.B == B and self.n == n and self.KS == KS and self.device == device
                and self.nIter >= nIter and (self.ys is not None) == bool(keep_xs)
                and (self.iter_stats is not None or not stats) and (self.f64 is not None or not keep_f64))

    def reset_views(self):
        self._host = None

    def stats(self):
        """Per-outer-iteration statistics as a dict of numpy arrays [nIter] (None if not requested):
        what the reference prints per iteration / what ebundle-vs-gd.py:94-99 plots (mean f - H)."""
        if self.iter_stats is None:
            return None
        a = self.iter_stats.cpu().numpy()
        ent = np.maximum(a[:, 0], 1.0)
        return dict(entering=a[:, 0], sum_k=a[:, 1], inner_its=a[:, 2], sum_its_k2=a[:, 3], sum_its_k=a[:, 4],
                    stopped=a[:, 5], mean_f_minus_H=a[:, 6] / ent)

    def y_host(self, out=None):
        """y* on the host.  ``out``: a float64 CPU tensor / array to fill in place (pinned memory makes
        the copy asynchronous-capable and ~4x faster than pageable); else a pinned staging buffer owned
        by this state is used and a numpy copy is returned."""
        if out is not None and isinstance(out, torch.Tensor) and out.dtype == torch.float64 and not out.is_cuda \
                and out.is_contiguous():
            out.copy_(self.y, non_blocking=out.is_pinned())
            torch.cuda.current_stream().synchronize()
            return out.numpy()
        if self._pin_y is None:
            try:
                self._pin_y = torch.empty(self.B, self.n, dtype=torch.float64, pin_memory=True)
            except RuntimeError:
                self._pin_y = torch.empty(self.B, self.n, dtype=torch.float64)
        self._pin_y.copy_(self.y, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return self._pin_y.numpy().copy()

    # ---- ragged outputs ---------------------------------------------------------------------
    def _host_small(self):
        if self._host is None:
            self._host = dict(perm=self.perm.cpu().numpy(), count=self.count.cpu().numpy(),
                              h=self.h.cpu().numpy(), lam=self.lam.cpu().numpy())
        return self._host

    def _fetch(self, kind, u):
        hs = self._host_small()
        k = int(hs["count"][u])
        slots = hs["perm"][u, :k]
        if kind == "lam":
            return hs["lam"][u, slots].copy() if k else None
        if kind == "b":
            return [float(v) for v in hs["h"][u, slots]]
        src = self.G if kind == "A" else self.ys
        if src is None:
            raise RuntimeError("xs were not kept (keep_xs=False)")
        if k == 0:
            return []
        idx = torch.as_tensor(slots.astype(np.int64), device=self.device)
        rows = src[u].index_select(0, idx).cpu().numpy()
        return [rows[j] for j in range(k)]


class _EmptyState:
    """State of a zero-row call (an empty shard of a sample-sharded batch, icnn_b200/dist.py)."""

    def __init__(self, n, KS, device):
        self.B, self.n, self.KS, self.device = 0, int(n), int(KS), device
        self.y = torch.empty(0, n, dtype=torch.float64, device=device)
        self.nactive = torch.zeros(1, dtype=torch.int32, device=device)
        self.ys = self.iter_stats = self.f64 = None
        self.status_host = np.zeros(0, dtype=np.int32)

    def stats(self):
        return None


def _make_cfg(variant, solver, nIter, line_search, rank_tol, max_inner, n, KS):
    dflt = VARIANT_DEFAULTS[variant]
    if variant == "lib":
        if solver == "pc":
            sol = _capi.SOLVER_PC
        elif solver in ("newton", "boyd"):
            # 'boyd' (lib/bundle_entropy.py:80-156) solves the same strictly convex subproblem on
            # the full KKT system; it is accepted and mapped to the converged dual Newton solve.
            sol = _capi.SOLVER_NEWTON
        else:
            raise RuntimeError("Solver unknown: " + str(solver))  # lib/bundle_entropy.py:232
    else:
        sol = _capi.SOLVER_NEWTON
    ls = dflt["line_search"] if line_search is None else bool(line_search)
    if rank_tol is None:
        # np.linalg.matrix_rank: tol = sigma_max * max(k, n) * eps (float64 rows); x16 margin for
        # the explicit-residual test that replaces the SVD (DESIGN.md, "rank stop")
        rank_tol = 16.0 * max(KS, n) * _EPS64
    return _capi.BundleCfg(_capi.VARIANT[variant], sol, int(ls), int(max_inner), float(dflt["prune_thr"]),
                           float(rank_tol), int(nIter), 0)


def _dtype_of(a):
    if isinstance(a, torch.Tensor):
        return {torch.float32: np.float32, torch.float64: np.float64}.get(a.dtype, None)
    return np.asarray(a).dtype.type


def _to_numpy(a):
    if isinstance(a, torch.Tensor):
        return a.detach().cpu().numpy()
    return np.asarray(a)


def _nvtx(name):
    return torch.cuda.nvtx.range(name)


def solveBatch(fg, initXs, nIter=None, callback=None, solver="pc", *, variant="lib", line_search=None,
               rank_tol=None, max_inner=0, keep_xs=True, device=None, strict=False, return_state=False,
               state=None, stats=False, graph=False):
    """argmin_y f(x, y) - H(y) over [0,1]^n by the bundle-entropy method, on the GPU.

    Positional/keyword arguments are the reference's; keyword-only extras select which of the
    reference's three copies is reproduced (``variant`` in {'lib', 'dual', 'rl'}) and tuning.
    ``solver``: 'pc' (Mehrotra predictor-corrector, the reference default), 'boyd' (accepted,
    mapped to the same optimum) or 'newton' (converged dual projected Newton).
    Returns ``(x, A, b, lam, xs, nIters)``; A/b/xs are lazy list-of-lists views, lam a lazy list
    of arrays.  ``initXs`` (numpy float64, or a float64 CPU torch tensor) is overwritten with the
    result like the reference does (lib/bundle_entropy.py:200,228).
    ``state``: a BundleState of a previous call with the same shape to reuse (no device allocation;
    the lazy A/b/lam/xs views of that earlier call become invalid).  ``stats=True`` collects the
    per-iteration statistics (``return_state=True`` -> ``state.stats()``).
    ``graph=True`` (fused mode): the nIter x (K1, K2) launches are captured into a CUDA graph on first use and
    replayed with one launch afterwards; the capture is cached on ``state`` and keyed on the device addresses of
    ``fg``'s buffers, so it pays off when ``state`` is reused and ``fg`` keeps its buffers (same results, bit for bit).
    NVTX ranges ``icnn:h2d``, ``icnn:loop``, ``icnn:d2h`` bracket the phases for nsys / ncu.
    """
    if variant not in VARIANT_DEFAULTS:
        raise ValueError("variant must be one of %s" % sorted(VARIANT_DEFAULTS))
    if variant != "lib":
        solver = "newton"
    if nIter is None:
        nIter = VARIANT_DEFAULTS[variant]["nIter"]
    nIter = int(nIter)
    if not torch.cuda.is_available():
        raise RuntimeError("icnn_b200.solveBatch needs a CUDA device (no CPU fallback)")
    fused = isinstance(fg, BoundPICNN)
    dev = fg.net.device if fused else (torch.device(device) if device is not None else default_device())
    x0 = initXs
    B, n = x0.shape
    if B == 0 or nIter < 1:
        out = (_to_numpy(x0), [[] for _ in range(B)], [[] for _ in range(B)], [None] * B,
               [[] for _ in range(B)], [nIter] * B)
        if return_state:   # an empty shard of a sharded batch still gets a (zero-row) state
            KS0 = max((nIter if variant == "rl" else min(max(nIter, 1), n)) + 1, 2)
            return out + (_EmptyState(n, KS0, dev),)
        return out
    # slot capacity: active rows <= min(nIter, n) for the rank-tested copies, + 1 free slot
    KS = (nIter if variant == "rl" else min(nIter, n)) + 1
    KS = max(KS, 2)
    if KS > 64:
        # the per-sample k x k algebra lives in one warp's registers / shared memory (include/icnn_b200.h)
        raise ValueError("solveBatch: min(nIter, n_y) + 1 = %d bundle slots requested, the device solver "
                         "holds at most 64 (nIter <= 63); the reference has no cap (lib/bundle_entropy.py:192)"
                         % KS)
    cfg = _make_cfg(variant, solver, nIter, line_search, rank_tol, max_inner, n, KS)
    f64_cb = False
    rows_inexact = False
    with torch.cuda.device(dev):
        need = (B, n, KS, dev, keep_xs, nIter, stats, False)
        if state is not None and state.compatible(*need):
            st = state
            st.reset_views()
            if st.iter_stats is not None:      # a reused state collects statistics (atomics) only when this call asks
                st.c.iter_stats = st.iter_stats.data_ptr() if stats else None
        else:
            st = BundleState(B, n, KS, dev, keep_xs=keep_xs, nIter=nIter, stats=stats)
        with _nvtx("icnn:h2d"):
            if isinstance(x0, torch.Tensor):
                st.y.copy_(x0.to(device=dev, dtype=torch.float64, non_blocking=True))
            else:
                st.y.copy_(torch.from_numpy(np.ascontiguousarray(x0, dtype=np.float64)), non_blocking=False)
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        loop_rng = _nvtx("icnn:loop")
        loop_rng.__enter__()
        if fused and callback is None:
            if fg.B != B or fg.net.n != n:
                raise ValueError("fg is bound to a [%d, %d] problem, initXs is %s" % (fg.B, fg.net.n, (B, n)))
            if graph:
                _capi.check(_capi.lib.icnn_loop_graph_launch(st.loop_graph(fg, cfg), stream))
            else:
                _capi.check(_capi.lib.icnn_solve_batch_fused(fg.net._h, C.byref(fg.c_gates), C.byref(cfg),
                                                             C.byref(st.c), fg.ws.data_ptr(), stream))
        else:
            _capi.check(_capi.lib.icnn_bundle_init(C.byref(st.c), nIter, stream))
            for t in range(nIter):
                if fused:
                    _capi.check(_capi.lib.icnn_picnn_fg(
                        fg.net._h, C.byref(fg.c_gates), st.y32.data_ptr(), st.f.data_ptr(),
                        st.G.data_ptr(), 0, st.perm.data_ptr(), st.count.data_ptr(), KS,
                        fg.ws.data_ptr(), None, stream))
                    if callback is not None:
                        fi = st.f.cpu().numpy()
                        xi = st.y.cpu().numpy()
                        if variant == "rl":
                            callback(t, fi)          # RL/src/bundle_entropy.py:103-104
                        else:
                            callback(t, fi, xi)      # lib/bundle_entropy.py:208-209
                else:
                    xi = st.y.cpu().numpy()
                    fi, gi = fg(xi)
                    if t == 0:
                        f64_cb = (_dtype_of(gi) == np.float64 or _dtype_of(fi) == np.float64)
                        if f64_cb and st.f64 is None:
                            # a float64 fg: keep f in float64 for the cut offsets h = f - g.y, like the
                            # reference (lib/bundle_entropy.py:205-207); the rows themselves are stored
                            # in float32 (documented deviation, DESIGN.md section 2)
                            st.f64 = torch.empty(B, dtype=torch.float64, device=dev)
                            st.c.f64 = st.f64.data_ptr()
                        if rank_tol is None and variant != "rl" and _dtype_of(gi) == np.float32:
                            # np.linalg.matrix_rank scales its tolerance with the dtype of the rows: a
                            # float32 fg (the reference's TF fetch) stops samples at max(k, n) * eps32
                            cfg.rank_tol = float(max(KS, n) * np.finfo(np.float32).eps)
                    if callback is not None:
                        if variant == "rl":
                            callback(t, _to_numpy(fi))
                        else:
                            callback(t, _to_numpy(fi), xi)
                    if f64_cb:
                        fd = torch.as_tensor(fi, device=dev).to(torch.float64).contiguous().reshape(B)
                        gd = torch.as_tensor(gi, device=dev).to(torch.float64).contiguous().reshape(B, n)
                        if rank_tol is None and variant != "rl" and not rows_inexact \
                                and bool((gd.to(torch.float32).to(torch.float64) != gd).any()):
                            # genuinely float64 rows do not survive the float32 row storage exactly: from here
                            # on the dependency test works at the storage precision, max(k, n) * eps32, so
                            # that rows dependent in float64 are still detected after rounding (rows that are
                            # float32-representable keep the reference's float64 tolerance)
                            rows_inexact = True
                            cfg.rank_tol = float(max(KS, n) * np.finfo(np.float32).eps)
                        _capi.check(_capi.lib.icnn_bundle_put_fg_f64(C.byref(st.c), fd.data_ptr(), gd.data_ptr(), stream))
                    else:
                        fd = torch.as_tensor(fi, device=dev).to(torch.float32).contiguous().reshape(B)
                        gd = torch.as_tensor(gi, device=dev).to(torch.float32).contiguous().reshape(B, n)
                        _capi.check(_capi.lib.icnn_bundle_put_fg(C.byref(st.c), fd.data_ptr(), gd.data_ptr(), stream))
                _capi.check(_capi.lib.icnn_bundle_step(C.byref(cfg), C.byref(st.c), t, stream))
                if int(st.nactive[t + 1].item()) == 0:   # lib/bundle_entropy.py:239
                    break
        loop_rng.__exit__(None, None, None)
        with _nvtx("icnn:d2h"):
            x = st.y_host(out=x0 if isinstance(x0, torch.Tensor) else None)
            status = st.status.cpu().numpy()
    if np.any(status == _capi.ST_NONFINITE) or np.any(status == _capi.ST_SOLVE_FAIL):
        msg = "solveBatch: %d samples non-finite, %d with a failed inner solve" % (
            int(np.sum(status == _capi.ST_NONFINITE)), int(np.sum(status == _capi.ST_SOLVE_FAIL)))
        if strict:
            raise RuntimeError(msg)
        warnings.warn(msg)   # the reference runs under np.seterr(all='warn')
    if isinstance(x0, np.ndarray) and x0.dtype == np.float64:
        x0[...] = x
        x = x0
    nIters = st.nIters.cpu().numpy().tolist()     # a Python list like the reference's (ndarray.tolist: 65 536 rows in ~1 ms)
    st.status_host = status
    out = (x, _Rows(st, "A"), _Rows(st, "b"), _Rows(st, "lam"), _Rows(st, "xs"), nIters)
    if return_state:
        return out + (st,)
    return out


def solve(fg, initX, nIter=10, callback=None, *, variant="dual", **kw):
    """Single-sample form of the reference (lib/bundle_entropy_dual.py:87-127 ``solve``; the
    ``solve`` of lib/bundle_entropy.py:168-190 is dead code there): ``fg(x [n]) -> (f, g [n])``,
    returns the final iterate.  Runs as a batch of one through :func:`solveBatch`."""
    x0 = np.array(initX, dtype=np.float64).reshape(1, -1)

    def fg1(xb):
        f, g = fg(xb[0])
        return np.atleast_1d(np.asarray(f, dtype=np.float64)), np.asarray(g, dtype=np.float64).reshape(1, -1)

    cb = None if callback is None else (lambda t, f, x=None: callback(t, f[0], None if x is None else x[0]))
    out = solveBatch(fg1, x0, nIter=nIter, callback=cb, variant=variant, **kw)
    return out[0][0]
