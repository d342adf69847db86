"""numpy float64 restatement of the fully-connected PICNN energy f(x, y; theta) and df/dy.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  The reference builds this function as a
TensorFlow graph (TensorFlow/tflearn absent here), so it is restated from the cited lines; tflearn
``fully_connected`` is ``out = in @ W + b`` with W laid out ``[in, out]``.

Follows (paths relative to the locuslab/icnn repository):
  * multi-label-cls/icnn_ebundle.py:316-388  (Model.f: ReLU PICNN, ``nLabels`` appended to szs)
  * RL/src/icnn.py:325-404                   (Agent.negQ: leaky-ReLU PICNN, szs = [l1, l2])
  * multi-label-cls/icnn_ebundle.py:146      (dE_dy_ = tf.gradients(E_, y_))
  * RL/src/icnn.py:148-158                   (affine wrapper x in [0,1] -> a = 2x-1, grad *= 2)
  * multi-label-cls/icnn-back.py:116-131     (momentum gradient-descent inner loop)

Parity status of THIS file: TensorFlow / tflearn are not installed, so the reference's graph cannot run on
the real libraries.  It is pinned three ways (tests/test_oracle_picnn.py, tests/test_oracle_tfshim.py):
(i) **the reference's own code** -- Model.__init__/f of both multi-label scripts and Agent.negQ /
Agent.bundle_entropy, cut out of the reference files unmodified -- executed on a stand-in that restates only the
TF / tflearn PRIMITIVES (oracle/tf_shim.py; goldens tests/golden/picnn_tfshim.npz by oracle/gen_golden_tfshim.py):
f, df/dy, gates with batch-norm, momentum GD and the RL wrapper agree to 1e-10; (ii) a finite-difference check of
the analytic gradient; (iii) an independently written torch-autograd forward.  What stays restated rather than
executed is the primitives' semantics (``fully_connected`` = ``x @ W + b``, batch-norm epsilon 1e-5, leaky-ReLU).

Index convention: z-layers i = 0..L, widths s_0..s_{L-1} = ``hidden``, s_L = 1.
"""
from __future__ import annotations

import numpy as np


from icnn_b200.workloads import PicnnParams, synth_params  # noqa: E402,F401  (data generator only)


def gates(p: PicnnParams, x):
    """x-path: returns (cz, cy, d) lists indexed by z-layer (cz[0] is None).
    multi-label-cls/icnn_ebundle.py:339-347 (u path; inference-mode batch-norm after the ReLU when
    ``p.bn[i]`` is given, as the per-feature affine map (scale, shift) -- tflearn's epsilon / moving
    averages are the caller's, SURVEY.md section 8c), :354-356 (cz), :363-365 (cy), :372-373 (d)."""
    x = np.asarray(x, dtype=np.float64)
    L = p.L
    us = []
    prev = x
    for i in range(L):
        u = prev @ p.Wu[i] + p.bu[i]
        if i < L - 1:
            u = np.maximum(u, 0.0)
            bn = getattr(p, "bn", None)
            if bn is not None and bn[i] is not None:     # :343-345  u = bn(relu(fc(prevU)))
                u = u * np.asarray(bn[i][0], dtype=np.float64) + np.asarray(bn[i][1], dtype=np.float64)
        us.append(u)
        prev = u
    cz, cy, d = [None] * (L + 1), [None] * (L + 1), [None] * (L + 1)
    for i in range(L + 1):
        P = x if i == 0 else us[i - 1]
        if i > 0:
            cz[i] = np.maximum(P @ p.Wzu[i] + p.bzu[i], 0.0)
        cy[i] = P @ p.Wyu[i] + p.byu[i]
        d[i] = P @ p.Wzx[i] + p.bzx[i]
    return cz, cy, d


def fg_gated(p: PicnnParams, gts, y, dtype=np.float64):
    """Energy f [B] and gradient df/dy [B, n] for iterate y [B, n] given precomputed gates.
    Forward  multi-label-cls/icnn_ebundle.py:349-387 / RL/src/icnn.py:356-404;
    gradient = what tf.gradients(E_, y_) (:146) evaluates, written out by hand.
    (``np.asarray(.., dtype)`` is a no-op on operands already of ``dtype``: make_fg casts weights and gates once.)"""
    cz, cy, d = gts
    c = lambda a: np.asarray(a, dtype=dtype)          # noqa: E731
    y = c(y)
    L, a = p.L, p.alpha
    zs = []
    z = None
    for i in range(L + 1):
        pre = (y * c(cy[i])) @ c(p.Wy[i]) + c(d[i])
        if i > 0:
            pre = pre + (z * c(cz[i])) @ c(p.Wz[i])
        if i < L:
            z = np.where(pre > 0, pre, a * pre)
        else:
            z = pre
        zs.append(z)
    f = zs[L][:, 0]
    delta = np.ones_like(zs[L])
    g = np.zeros_like(y)
    for i in range(L, -1, -1):
        g += c(cy[i]) * (delta @ c(p.Wy[i]).T)
        if i > 0:
            dact = np.where(zs[i - 1] > 0, 1.0, a).astype(dtype)
            delta = dact * c(cz[i]) * (delta @ c(p.Wz[i]).T)
    return f, g


class _Cast:
    """The z-path weights of ``p`` cast to ``dtype`` once (the reference's TF graph holds float32 variables; it does
    not convert them per sess.run)."""

    def __init__(self, p, dtype):
        self.L, self.alpha = p.L, p.alpha
        self.Wy = [np.asarray(w, dtype=dtype) for w in p.Wy]
        self.Wz = [None if w is None else np.asarray(w, dtype=dtype) for w in p.Wz]


def make_fg(p: PicnnParams, x, dtype=np.float64, out_dtype=None, affine=False):
    """Closure fg(y) -> (f, g) with the reference's callback contract
    (multi-label-cls/icnn_ebundle.py:218-221).  ``dtype=np.float32`` mimics the TF graph's
    arithmetic, ``out_dtype=np.float32`` mimics the float32 fetch.  ``affine=True`` applies the
    RL wrapper (RL/src/icnn.py:148-153): the solver variable is x in [0,1], a = 2x-1, grad *= 2."""
    gts = gates(p, x)
    if np.dtype(dtype) != np.float64:                 # cast weights and gates once, not per call
        gts = tuple([None if g_ is None else g_.astype(dtype) for g_ in gs] for gs in gts)
        p = _Cast(p, dtype)

    def fg(y):
        yy = 2.0 * np.asarray(y) - 1.0 if affine else y
        f, g = fg_gated(p, gts, yy, dtype=dtype)
        if affine:
            g = 2.0 * g
        if out_dtype is not None:
            f, g = f.astype(out_dtype), g.astype(out_dtype)
        return f, g

    return fg


def momentum_gd(fg, y0, nIter, lr, momentum):
    """Unrolled momentum gradient descent, multi-label-cls/icnn-back.py:120-131
    (= completion/icnn.back.py:133-147): v' = m v - lr g(y); y' = y - m v + (1+m) v'.
    No projection.  Returns (y_n, f(y_n))."""
    y = np.array(y0, dtype=np.float64)
    v = np.zeros_like(y)
    for _ in range(nIter):
        _, g = fg(y)
        v_new = momentum * v - lr * np.asarray(g, dtype=np.float64)
        y = y - momentum * v + (1.0 + momentum) * v_new
        v = v_new
    f, _ = fg(y)
    return y, np.asarray(f, dtype=np.float64)


def entr(y):
    """Sum_j -y log y - (1-y) log(1-y) with 0 log 0 = 0 (multi-label-cls/ebundle-vs-gd.py:38-41)."""
    y = np.asarray(y, dtype=np.float64)
    with np.errstate(all="ignore"):
        z = -y * np.log(y) - (1.0 - y) * np.log(1.0 - y)
    z[z != z] = 0.0
    return z.sum(axis=1)
