"""numpy float64 restatement of the bundle-entropy training gradient d F / d theta.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

What the reference computes: ``opt.compute_gradients(F_, theta_)`` (multi-label-cls/icnn_ebundle.py:153-156) of

    F_ = c * E(x, y) + sum_j v_j dE/dy_j                       (:148, dE_dy_ = tf.gradients(E_, y_) :146)

summed over the ``train_step_fd`` rows (:296-314), one per (sample, bundle point).  TensorFlow is absent here, so
this file writes the double backprop out by hand from the layer recurrences of one row (gates from the row's x):

    forward    pre_l = (y o cy_l) Wy_l + (z_{l-1} o cz_l) Wz_l + d_l,   z_l = act(pre_l) (l < L),  E = pre_L
    backward   delta_L = 1,   g = sum_l cy_l o (delta_l Wy_l^T),
               delta_{l-1} = act'(pre_{l-1}) o cz_l o (delta_l Wz_l^T)
    F = c E + v . g

Reverse mode of F: the adjoint of g is v, the adjoint of E is c.  The backward recurrence is reversed from l = 0
upwards (act'' = 0 almost everywhere for ReLU / leaky-ReLU, which is what TensorFlow's ReluGrad gradient gives):

    bar_delta_l = (v o cy_l) Wy_l + (t_{l-1} o cz_l) Wz_l,   t_l = act'(pre_l) o bar_delta_l

and every use of a parameter / gate in either recurrence contributes its term:

    from  g += cy_l o (delta_l Wy_l^T):          dWy_l += (v o cy_l)^T delta_l,     dcy_l += v o (delta_l Wy_l^T)
    from  delta_{l-1} = ... (delta_l Wz_l^T):    dWz_l += (t_{l-1} o cz_l)^T delta_l,  dcz_l += t_{l-1} o (delta_l Wz_l^T)
    from  c * E through the forward:             dWy_l += c (y o cy_l)^T delta_l,   dcy_l += c y o (delta_l Wy_l^T)
                                                 dWz_l += c (z_{l-1} o cz_l)^T delta_l,  dcz_l += c z_{l-1} o (delta_l Wz_l^T)
                                                 dd_l  += c delta_l

The x-path parameters follow from the per-sample gate adjoints (dcy, dcz, dd) by dense-layer backprop of
multi-label-cls/icnn_ebundle.py:339-373.  Every gradient is returned PER SAMPLE (the sum over that sample's rows),
stacked as [B, ...]; summing over axis 0 gives the minibatch gradient.  Pinned by tests/test_oracle_bundle_grad.py
against the reference's own ``Model`` executed on oracle/tf_shim.py (tests/golden/training/bundle_grad.npz), an
independent torch double backprop, central finite differences and linearity in (V, c).
"""
from __future__ import annotations

import numpy as np

from oracle import picnn_np

PARAMS = ("Wy", "Wz", "Wu", "bu", "Wzu", "bzu", "Wyu", "byu", "Wzx", "bzx")


def _rows_of(counts):
    counts = np.asarray(counts, dtype=np.int64)
    return np.repeat(np.arange(len(counts)), counts)


def row_pass(p, x, Y, V, c, counts):
    """Per-row forward, backward and reversed backward.  Returns (gates of the rows, zs, deltas, ts, pres)."""
    iu = _rows_of(counts)
    cz, cy, d = picnn_np.gates(p, np.asarray(x, dtype=np.float64))
    cz = [None if a is None else a[iu] for a in cz]
    cy = [a[iu] for a in cy]
    d = [a[iu] for a in d]
    Y, V, c = (np.asarray(a, dtype=np.float64) for a in (Y, V, c))
    L, al = p.L, p.alpha
    Wy = [np.asarray(w, dtype=np.float64) for w in p.Wy]
    Wz = [None] + [np.asarray(w, dtype=np.float64) for w in p.Wz[1:]]
    pres, zs, z = [], [], None
    for l in range(L + 1):
        pre = (Y * cy[l]) @ Wy[l] + d[l]
        if l > 0:
            pre = pre + (z * cz[l]) @ Wz[l]
        z = np.where(pre > 0, pre, al * pre) if l < L else pre
        pres.append(pre)
        zs.append(z)
    dact = [np.where(pres[l] > 0, 1.0, al) for l in range(L)]
    delta = [None] * (L + 1)
    delta[L] = np.ones((Y.shape[0], 1))
    for l in range(L, 0, -1):
        delta[l - 1] = dact[l - 1] * cz[l] * (delta[l] @ Wz[l].T)
    ts, t = [], None
    for l in range(L):
        bar = (V * cy[l]) @ Wy[l]
        if l > 0:
            bar = bar + (t * cz[l]) @ Wz[l]
        t = dact[l] * bar
        ts.append(t)
    return (cz, cy, d), zs, delta, ts, pres


def _per_sample(rows_arr, iu, B):
    out = np.zeros((B,) + rows_arr.shape[1:])
    np.add.at(out, iu, rows_arr)
    return out


def bundle_grad(p, x, Y, V, c, counts, per_sample=True):
    """Gradients of sum_r F_r: dict name -> list over layers, for the parameters ``PARAMS`` (Wz[0], Wzu[0], bzu[0]
    are None) and the gate adjoints 'dcy', 'dcz', 'dd'.  Gate adjoints are always per sample ([B, .]); parameter
    gradients are per sample ([B, ...]) with ``per_sample``, else summed over the minibatch."""
    B = len(counts)
    iu = _rows_of(counts)
    off = np.concatenate([[0], np.cumsum(np.asarray(counts, dtype=np.int64))])
    (cz, cy, d), zs, delta, ts, _ = row_pass(p, x, Y, V, c, counts)
    Y, V, c = (np.asarray(a, dtype=np.float64) for a in (Y, V, c))
    cc = c[:, None]
    L = p.L
    Wy = [np.asarray(w, dtype=np.float64) for w in p.Wy]
    Wz = [None] + [np.asarray(w, dtype=np.float64) for w in p.Wz[1:]]

    def wsum(A, D):                 # sum over rows of A_r^T D_r: per sample or over everything
        if not per_sample:
            return A.T @ D
        out = np.zeros((B, A.shape[1], D.shape[1]))
        for u in range(B):
            out[u] = A[off[u]:off[u + 1]].T @ D[off[u]:off[u + 1]]
        return out

    g = {k: [None] * (L + 1) for k in ("Wy", "Wz", "dcy", "dcz", "dd")}
    for l in range(L + 1):
        # v . g term and c E term of every use of the layer's parameters / gates
        g["Wy"][l] = wsum(V * cy[l], delta[l]) + wsum(cc * Y * cy[l], delta[l])
        bw = delta[l] @ Wy[l].T
        g["dcy"][l] = _per_sample(V * bw + cc * Y * bw, iu, B)
        g["dd"][l] = _per_sample(cc * delta[l], iu, B)
        if l > 0:
            zw = delta[l] @ Wz[l].T
            g["Wz"][l] = wsum(ts[l - 1] * cz[l], delta[l]) + wsum(cc * zs[l - 1] * cz[l], delta[l])
            g["dcz"][l] = _per_sample(ts[l - 1] * zw + cc * zs[l - 1] * zw, iu, B)
    g.update(xpath_backward(p, x, g["dcy"], g["dcz"], g["dd"], per_sample))
    return g


def xpath_backward(p, x, dcy, dcz, dd, per_sample=True):
    """Dense-layer backprop of the per-sample gate adjoints [B, .] into the x-path parameters, per sample or summed
    (no batch-norm: ``p.bn`` must be empty or folded)."""
    x = np.asarray(x, dtype=np.float64)
    L = p.L
    W = lambda ws: [None if w is None else np.asarray(w, dtype=np.float64) for w in ws]  # noqa: E731
    Wu, Wzu, Wyu, Wzx = W(p.Wu), W(p.Wzu), W(p.Wyu), W(p.Wzx)
    if per_sample:
        outer = lambda a, b: np.einsum("bi,bj->bij", a, b)                 # noqa: E731
        bsum = lambda a: a.copy()                                          # noqa: E731
    else:
        outer = lambda a, b: a.T @ b                                       # noqa: E731
        bsum = lambda a: a.sum(0)                                          # noqa: E731
    us, pres, prev = [], [], x
    for i in range(L):
        pre = prev @ Wu[i] + p.bu[i]
        u = np.maximum(pre, 0.0) if i < L - 1 else pre
        pres.append(pre); us.append(u); prev = u
    out = {k: [None] * (L + 1) for k in ("Wzu", "bzu", "Wyu", "byu", "Wzx", "bzx")}
    out.update(Wu=[None] * L, bu=[None] * L)
    dU = [np.zeros_like(u) for u in us]
    for i in range(L, -1, -1):
        P = x if i == 0 else us[i - 1]
        out["Wyu"][i], out["byu"][i] = outer(P, dcy[i]), bsum(dcy[i])
        out["Wzx"][i], out["bzx"][i] = outer(P, dd[i]), bsum(dd[i])
        dP = dcy[i] @ Wyu[i].T + dd[i] @ Wzx[i].T
        if i > 0:
            pz = dcz[i] * ((P @ Wzu[i] + p.bzu[i]) > 0)
            out["Wzu"][i], out["bzu"][i] = outer(P, pz), bsum(pz)
            dU[i - 1] += dP + pz @ Wzu[i].T
    for i in range(L - 1, -1, -1):
        du = dU[i] * (pres[i] > 0) if i < L - 1 else dU[i]
        P = x if i == 0 else us[i - 1]
        out["Wu"][i], out["bu"][i] = outer(P, du), bsum(du)
        if i > 0:
            dU[i - 1] += du @ Wu[i].T
    return out


def objective(p, x, Y, V, c, counts):
    """sum_r F_r = sum_r c_r E(x_u, y_r) + v_r . dE/dy(x_u, y_r)  (the scalar the gradient is of)."""
    (cz, cy, d), zs, delta, _, _ = row_pass(p, x, Y, V, c, counts)
    Y, V, c = (np.asarray(a, dtype=np.float64) for a in (Y, V, c))
    g = sum(cy[l] * (delta[l] @ np.asarray(p.Wy[l], dtype=np.float64).T) for l in range(p.L + 1))
    return float(np.sum(c * zs[p.L][:, 0]) + np.sum(V * g))


def min_rel_preact(p, x, Y, counts):
    """Per row: min over the hidden layers of min_j |pre_l[j]| / max_j |pre_l[j]| -- how close the row sits to a kink
    of the piecewise-linear energy (a float32 evaluation can land on the other side of it)."""
    _, _, _, _, pres = row_pass(p, x, Y, np.zeros_like(np.asarray(Y, dtype=np.float64)), np.zeros(len(Y)), counts)
    out = np.full(len(Y), np.inf)
    for l in range(p.L):
        a = np.abs(pres[l])
        out = np.minimum(out, a.min(axis=1) / np.maximum(a.max(axis=1), 1e-300))
    return out
