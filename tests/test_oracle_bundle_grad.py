"""oracle/bundle_grad_np.py -- the float64 bundle-entropy training gradient d (sum_r F_r) / d theta -- against the
reference's own Model executed on the TF shim (tests/golden/training/bundle_grad.npz, oracle/gen_golden_bundle_grad.py), an
independent torch double backprop, central finite differences, and linearity in (V, c).  CPU only."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle import bundle_grad_np as bg
from oracle.gen_golden_bundle_grad import CASES, LOSSES, case_inputs
from icnn_b200.workloads import synth_params

PNAMES = bg.PARAMS


@pytest.mark.parametrize("tag", list(CASES))
@pytest.mark.parametrize("loss", LOSSES)
def test_oracle_matches_reference_model_golden(tag, loss, golden_dir):
    gold = np.load(os.path.join(golden_dir, "training", "bundle_grad.npz"))
    p, x, _y0, _tY, _nIter, _sizes = case_inputs(tag)
    key = "%s_%s_" % (tag, loss)
    counts = gold[tag + "_counts"]
    g = bg.bundle_grad(p, x, gold[key + "Y"], gold[key + "V"], gold[key + "c"], counts)
    stored = [k for k in gold.files if k.startswith(key + "grad_")]
    assert len(stored) >= (35 if tag == "small" else 13)
    for k in stored:
        name = k[len(key + "grad_"):]
        pname, layer = name.rstrip("0123456789"), int(name[len(name.rstrip("0123456789")):])
        ref = gold[k]
        mine = g[pname][layer]
        assert mine.shape == ref.shape, (k, mine.shape, ref.shape)
        err = np.abs(mine - ref).max()
        assert err <= 1e-9 * max(1.0, np.abs(ref).max()), (k, err)


def _torch_grads(p, x, Y, V, c, counts):
    """Independent double backprop: E per row from the PICNN forward, dE/dy with create_graph=True, F = c E + v.g,
    then d sum F / d theta by autograd."""
    T = {k: [None if a is None else torch.tensor(np.asarray(a, dtype=np.float64), requires_grad=True)
             for a in getattr(p, k)] for k in PNAMES}
    L = p.L
    xr = torch.tensor(np.repeat(np.asarray(x, dtype=np.float64), counts, axis=0))
    y = torch.tensor(np.asarray(Y, dtype=np.float64), requires_grad=True)
    us, prev = [], xr
    for i in range(L):
        u = prev @ T["Wu"][i] + T["bu"][i]
        if i < L - 1:
            u = torch.relu(u)
        us.append(u)
        prev = u
    prevU, prevZ = xr, None
    for i in range(L + 1):
        z = (y * (prevU @ T["Wyu"][i] + T["byu"][i])) @ T["Wy"][i] + prevU @ T["Wzx"][i] + T["bzx"][i]
        if i > 0:
            z = z + (prevZ * torch.relu(prevU @ T["Wzu"][i] + T["bzu"][i])) @ T["Wz"][i]
        if i < L:
            z = torch.nn.functional.leaky_relu(z, p.alpha) if p.alpha else torch.relu(z)
        prevU = us[i] if i < L else None
        prevZ = z
    E = z.reshape(-1)
    (g,) = torch.autograd.grad(E.sum(), y, create_graph=True)
    F = torch.tensor(np.asarray(c, dtype=np.float64)) * E + (g * torch.tensor(np.asarray(V, dtype=np.float64))).sum(1)
    flat = [(k, i, t) for k in PNAMES for i, t in enumerate(T[k]) if t is not None]
    gs = torch.autograd.grad(F.sum(), [t for _, _, t in flat], allow_unused=True)
    out = {k: [None] * len(T[k]) for k in PNAMES}
    for (k, i, _), gr in zip(flat, gs):
        out[k][i] = np.zeros(tuple(T[k][i].shape)) if gr is None else gr.numpy()
    return out


def _case(seed, m, n, hidden, B, alpha=0.0, maxk=4):
    p = synth_params(seed, m, n, hidden, alpha=alpha)
    rs = np.random.RandomState(seed + 7)
    for i in range(p.L):
        p.bu[i] = 0.3 * rs.randn(p.hidden[i])
    for i in range(p.L + 1):
        if i > 0:
            p.bzu[i] = 0.3 * rs.randn(p.sizes[i - 1])
        p.byu[i] = 0.5 + 0.3 * rs.randn(n)
        p.bzx[i] = 0.3 * rs.randn(p.sizes[i])
    x = rs.randn(B, m)
    counts = rs.randint(0, maxk + 1, size=B)
    R = int(counts.sum())
    return p, x, rs.uniform(0.05, 0.95, size=(R, n)), rs.randn(R, n), rs.randn(R), counts


@pytest.mark.parametrize("alpha", [0.0, 0.01])
def test_oracle_matches_torch_double_backprop(alpha):
    p, x, Y, V, c, counts = _case(3, 7, 6, [9, 5, 6], 10, alpha=alpha)
    g = bg.bundle_grad(p, x, Y, V, c, counts, per_sample=False)
    t = _torch_grads(p, x, Y, V, c, counts)
    for k in PNAMES:
        for i, (a, b) in enumerate(zip(g[k], t[k])):
            if b is None:
                assert a is None, (k, i)
                continue
            np.testing.assert_allclose(a, b, rtol=0, atol=1e-10 * max(1.0, np.abs(b).max()), err_msg="%s%d" % (k, i))


def test_oracle_matches_central_finite_differences():
    """d sum F / d theta_e by central differences on entries whose +-h perturbation moves no pre-activation (of the
    z path or of an x-path ReLU) across zero."""
    p, x, Y, V, c, counts = _case(5, 6, 5, [8, 5], 8)
    g = bg.bundle_grad(p, x, Y, V, c, counts, per_sample=False)
    rs = np.random.RandomState(0)
    h = 1e-6
    checked = 0
    for k in PNAMES:
        for i, w in enumerate(getattr(p, k)):
            if w is None:
                continue
            for _ in range(3):
                idx = tuple(rs.randint(s) for s in np.shape(w))
                vals, masks = [], []
                for sgn in (1.0, -1.0):
                    q = copy.deepcopy(p)
                    arr = np.array(getattr(q, k)[i], dtype=np.float64)
                    arr[idx] += sgn * h
                    getattr(q, k)[i] = arr
                    vals.append(bg.objective(q, x, Y, V, c, counts))
                    _, _, _, _, pres = bg.row_pass(q, x, Y, V, c, counts)
                    from oracle import picnn_np
                    gz = picnn_np.gates(q, x)[0]
                    masks.append([pr[:, :] > 0 for pr in pres[:-1]] + [gz[j] > 0 for j in range(1, q.L + 1)])
                if any((a != b).any() for a, b in zip(*masks)):
                    continue
                fd = (vals[0] - vals[1]) / (2 * h)
                an = g[k][i][idx]
                assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)), (k, i, idx, fd, an)
                checked += 1
    assert checked >= 20


def test_gradient_is_linear_in_v_and_c():
    p, x, Y, V1, c1, counts = _case(8, 5, 4, [6, 4], 9)
    rs = np.random.RandomState(1)
    V2, c2 = rs.randn(*V1.shape), rs.randn(*c1.shape)
    a = bg.bundle_grad(p, x, Y, V1, c1, counts, per_sample=False)
    b = bg.bundle_grad(p, x, Y, V2, c2, counts, per_sample=False)
    s = bg.bundle_grad(p, x, Y, 2.0 * V1 - 3.0 * V2, 2.0 * c1 - 3.0 * c2, counts, per_sample=False)
    z = bg.bundle_grad(p, x, Y, 0 * V1, 0 * c1, counts, per_sample=False)
    for k in s:
        for ga, gb, gs, gz in zip(a[k], b[k], s[k], z[k]):
            if gs is None:
                continue
            np.testing.assert_allclose(gs, 2.0 * ga - 3.0 * gb, rtol=0, atol=1e-11 * max(1.0, np.abs(gs).max()))
            assert not np.any(gz)
