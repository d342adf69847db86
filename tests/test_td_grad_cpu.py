"""CPU checks of the RL TD training gradient: the C ABI entries and their refusals before any device is touched, the
Python argument errors, and properties of the float64 oracle (oracle/td_grad_np.py)."""
import ctypes as C

import numpy as np
import pytest

from oracle import td_grad_np as tg


def test_abi_entries():
    from icnn_b200 import _capi
    for name in ("icnn_td_grad_workspace_bytes", "icnn_td_grad"):
        assert name in _capi.SYMBOLS
        getattr(_capi.lib, name)
    text = open(_capi.LIB_PATH.replace("icnn_b200/libicnn_b200.so", "include/icnn_b200.h")).read()
    assert "int icnn_td_grad(" in text and "size_t icnn_td_grad_workspace_bytes(" in text


def test_workspace_query_and_refusals_without_a_device():
    from icnn_b200 import _capi
    lib = _capi.lib
    assert lib.icnn_td_grad_workspace_bytes(None, 256) == 0
    assert lib.icnn_td_grad_workspace_bytes(C.c_void_p(8), 0) == 0
    assert lib.icnn_td_grad_workspace_bytes(C.c_void_p(8), 65537) == 0
    assert lib.icnn_td_grad(None, None, None, None, None, None, None, 0.99, None, None, None, None, None) == -1
    assert b"null" in lib.icnn_last_error()
    gates, grads, p = _capi.Gates(), _capi.TrainGrads(), C.c_void_p(16)   # never dereferenced: refused first
    assert lib.icnn_td_grad(C.c_void_p(8), C.byref(gates), p, p, p, p, p, 0.99, p, p, C.byref(grads), p, None) == -1
    assert b"null gradient array" in lib.icnn_last_error()


def test_python_argument_errors():
    from icnn_b200.picnn import BoundPICNN
    from icnn_b200.td_grad import td_grad
    z = np.zeros((2, 3))
    with pytest.raises(TypeError, match="BoundPICNN"):
        td_grad(object(), object(), z, z, np.zeros(2), z, np.zeros(2, bool))
    fg = BoundPICNN.__new__(BoundPICNN)
    fg.affine = True
    with pytest.raises(ValueError, match="affine"):
        td_grad(fg, fg, z, z, np.zeros(2), z, np.zeros(2, bool))


def _small(B=10, seed=3):
    p, pt = tg.make_net("small", 3), tg.make_net("small", 4)
    return p, pt, tg.make_rows(p, pt, B, seed)


def test_terminal_row_ignores_the_target():
    p, pt, (obs, act, rew, ob2, act2, term) = _small()
    term = np.ones_like(term)
    td, _, y0 = tg.td_parts(p, pt, obs, act, rew, ob2, act2, term)
    pt2 = tg.make_net("small", 9)
    td2, _, y02 = tg.td_parts(p, pt2, obs, act, rew, ob2 + 1.0, -act2, term)
    np.testing.assert_array_equal(td, td2)
    np.testing.assert_array_equal(y0, rew)


def test_td_is_clamped():
    p, pt, rows = _small(B=40)
    td, q, y0 = tg.td_parts(p, pt, *rows)
    assert np.abs(td).max() <= 1.0 + 1e-12
    out = np.abs(y0 - q) > 1
    np.testing.assert_allclose(np.abs(td[out]), 1.0, rtol=0, atol=1e-12)


def test_loss_q_gradient_by_finite_differences():
    """Central differences of loss_q with the TD target y held fixed (it is under stop_gradient)."""
    p, pt, rows = _small(B=8)
    obs, act, rew, ob2, act2, term = rows
    _loss, td, g = tg.td_grad(p, pt, *rows)
    _, q, _ = tg.td_parts(p, pt, *rows)
    y = q - td

    def loss_q():
        qq = -(tg.negq(p, obs, act) - tg.entropy(act))
        return float(np.mean((qq - y) ** 2) + tg.L2NORM * tg.l2_loss(p))
    assert abs(loss_q() - _loss) <= 1e-12 * max(1.0, abs(_loss))
    rs = np.random.RandomState(0)
    for k in tg.PARAMS:
        for i, w in enumerate(getattr(p, k)):
            if w is None:
                continue
            w = np.asarray(w, dtype=np.float64)
            for _ in range(3):
                idx = tuple(rs.randint(s) for s in w.shape)
                h = 1e-6
                vals = []
                for s in (1, -1):
                    w2 = w.copy()
                    w2[idx] += s * h
                    getattr(p, k)[i] = w2
                    vals.append(loss_q())
                getattr(p, k)[i] = w
                fd = (vals[0] - vals[1]) / (2 * h)
                an = np.asarray(g[k][i]).reshape(w.shape)[idx]
                assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)), (k, i, idx, fd, an)
