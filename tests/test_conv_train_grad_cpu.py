"""CPU checks of the conv-PICNN training gradient: the C ABI struct matches the header and null arguments are refused
before any device is touched; the float64 oracle (oracle/conv_train_grad_torch.py) evaluates the energy of
tests/conv_energy.py (pinned to the reference's graph) and its gradient agrees with central finite differences."""
import ctypes as C
import os
import re

import numpy as np
import torch

from oracle import conv_train_grad_torch as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_struct_layout_matches_the_header():
    from icnn_b200 import _capi
    hdr = open(os.path.join(ROOT, "include", "icnn_b200.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} icnn_conv_train_grads;", hdr).group(1)
    fields = re.findall(r"float\* const\* (\w+);", body)
    assert fields == [f for f, _ in _capi.ConvTrainGrads._fields_]
    assert C.sizeof(_capi.ConvTrainGrads) == len(fields) * C.sizeof(C.c_void_p)


def test_null_arguments_are_refused_without_the_gpu():
    from icnn_b200 import _capi
    lib = _capi.lib
    assert lib.icnn_conv_train_grad(None, None, None, None, None, None, None, None, None) == -1
    assert b"null" in lib.icnn_last_error()
    off = (C.c_int64 * 2)(0, 0)
    gates = _capi.Gates()
    grads = _capi.ConvTrainGrads()          # all seven pointer arrays NULL
    ws = C.c_void_p(16)                     # never dereferenced: the call is refused first
    assert lib.icnn_conv_train_grad(C.c_void_p(8), C.byref(gates), off, None, None, None, C.byref(grads), ws,
                                    None) == -1
    assert b"null gradient array" in lib.icnn_last_error()
    assert lib.icnn_conv_train_grad_workspace_bytes(None, 4, 10) == 0


def _tiny(seed=1):
    from icnn_b200.conv_picnn import parse_variables
    H, W, convs, fcs = 7, 5, [(3, 3, 2), (4, 2, 1)], [5, 1]
    v = O.make_variables(H, W, convs, fcs, seed=seed)
    spec = parse_variables(v, H, W, strides=[2, 1])
    rs = np.random.RandomState(seed)
    counts = np.array([2, 0, 3])
    R = int(counts.sum())
    return spec, rs.uniform(size=(3, H * W)), rs.uniform(size=(R, H * W)), rs.randn(R, H * W), rs.randn(R), counts


def test_oracle_energy_is_the_reference_energy():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import conv_energy
    spec, x, Y, _V, _c, counts = _tiny()
    iu = np.repeat(np.arange(len(counts)), counts)
    V64 = {k: torch.as_tensor(a, dtype=torch.float64) for k, a in spec.vars.items()}
    cz, cy, d = O.gates(V64, spec, torch.as_tensor(x))
    rg = lambda lst: [None if t is None else t[iu] for t in lst]    # noqa: E731
    E, _, _ = O.y_energy(V64, spec, rg(cz), rg(cy), rg(d), torch.as_tensor(Y))
    ref = conv_energy.energy(spec, x[iu], torch.as_tensor(Y))
    np.testing.assert_allclose(E.numpy(), ref.numpy(), rtol=1e-12, atol=1e-14)


def test_oracle_matches_central_differences():
    """F = sum_r c_r E + V_r . dE/dy, with dE/dy from autograd, differenced in a few entries of every variable."""
    spec, x, Y, V, c, counts = _tiny()
    grads, adj, rel, _ = O.train_grad(spec, x, Y, V, c, counts)
    assert rel.min() > 1e-4                      # no row near a kink: F is smooth around theta
    assert set(grads) == set(O.trainable(list(spec.vars), 2, 2))
    assert len(adj["dcy"]) == 2 and adj["dcz"][0] is None and len(adj["dd"]) == 4
    iu = np.repeat(np.arange(len(counts)), counts)

    def F(vars_):
        V64 = {k: torch.as_tensor(a, dtype=torch.float64) for k, a in vars_.items()}
        cz, cy, d = O.gates(V64, spec, torch.as_tensor(x))
        rg = lambda lst: [None if t is None else t[iu] for t in lst]    # noqa: E731
        y = torch.as_tensor(Y).requires_grad_()
        E, _, _ = O.y_energy(V64, spec, rg(cz), rg(cy), rg(d), y)
        (g,) = torch.autograd.grad(E.sum(), y)
        return float((torch.as_tensor(c) * E).sum() + (torch.as_tensor(V) * g).sum())

    rs = np.random.RandomState(0)
    h = 1e-6
    for k, g in grads.items():
        for _ in range(2):
            idx = tuple(rs.randint(s) for s in g.shape)
            vp = {kk: np.array(a, dtype=np.float64) for kk, a in spec.vars.items()}
            vm = {kk: np.array(a, dtype=np.float64) for kk, a in spec.vars.items()}
            vp[k][idx] += h
            vm[k][idx] -= h
            fd = (F(vp) - F(vm)) / (2 * h)
            assert abs(fd - g[idx]) <= 1e-6 * max(1.0, abs(g).max()), (k, idx, fd, g[idx])
