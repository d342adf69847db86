"""CPU checks of the conv-PICNN GD training gradient: the C ABI refuses null and out-of-range arguments before any
device is touched, the library and the binding agree on the ABI version, and the piecewise-linear reduction the device
relies on holds: the literal float64 double backward through the unrolled GD loop (oracle/conv_gd_grad_torch.gd_grad)
equals the conv training gradient on the rows Y = y_i, V = kappa_i a, c = 0 (oracle/conv_gd_grad_torch.kappa_form)."""
import ctypes as C

import numpy as np
import pytest

from oracle import conv_gd_grad_torch as O
from oracle import conv_train_grad_torch as T


def test_abi_version_and_symbols():
    from icnn_b200 import _capi
    assert _capi.lib.icnn_abi_version() == _capi.ABI_VERSION == 9
    for name in ("icnn_conv_gd_backward", "icnn_conv_gd_backward_workspace_bytes"):
        assert name in _capi.SYMBOLS
        getattr(_capi.lib, name)


def test_null_and_bad_arguments_are_refused_without_the_gpu():
    from icnn_b200 import _capi
    lib = _capi.lib
    fake = C.c_void_p(16)                   # never dereferenced: every call below is refused first
    assert lib.icnn_conv_gd_backward(None, None, None, None, 1.0, 1, 0.01, 0.9, None, None, None, None) == -1
    assert b"null" in lib.icnn_last_error()
    gates = _capi.Gates()
    grads = _capi.ConvTrainGrads()          # all seven pointer arrays NULL
    assert lib.icnn_conv_gd_backward(C.c_void_p(8), C.byref(gates), fake, fake, 1.0, 1, 0.01, 0.9, fake,
                                     C.byref(grads), fake, None) == -1
    assert b"null gradient array" in lib.icnn_last_error()
    ptrs = [(C.c_void_p * 8)(*([16] * 8)) for _ in range(7)]
    grads = _capi.ConvTrainGrads(*[C.cast(a, _capi._fpp) for a in ptrs])
    assert lib.icnn_conv_gd_backward(C.c_void_p(8), C.byref(gates), fake, fake, 1.0, -1, 0.01, 0.9, fake,
                                     C.byref(grads), fake, None) == -1
    assert b"nIter < 0" in lib.icnn_last_error()


def test_workspace_query_refuses_what_it_cannot_size():
    from icnn_b200 import _capi
    ws = _capi.lib.icnn_conv_gd_backward_workspace_bytes
    h = C.c_void_p(8)                       # never dereferenced for these arguments
    assert ws(None, 4, 10) == 0
    assert ws(h, 0, 10) == 0
    assert ws(h, -3, 10) == 0
    assert ws(h, 4, -1) == 0
    assert ws(h, 2 ** 16, 2 ** 15) == 0     # 2^31 rows


def _tiny(seed=1, fcs=(5, 1)):
    from icnn_b200.conv_picnn import parse_variables
    H, W, convs = 7, 5, [(3, 3, 2), (4, 2, 1)]
    v = T.make_variables(H, W, convs, list(fcs), seed=seed)
    spec = parse_variables(v, H, W, strides=[2, 1])
    rs = np.random.RandomState(seed)
    B = 3
    return spec, rs.uniform(size=(B, H * W)), rs.uniform(0.2, 0.8, size=(B, H * W)), rs.uniform(size=(B, H * W))


@pytest.mark.parametrize("fcs", [(5, 1), (1,)])
def test_literal_double_backward_equals_the_kappa_form(fcs):
    """The Hessian term of the double backward vanishes (the energy is piecewise linear in y), so d loss / d theta is
    the training gradient of the rows (y_i, kappa_i a, c = 0): gradients and gate adjoints to 1e-10."""
    spec, x, y0, trueY = _tiny(fcs=fcs)
    nIter, lr, m = 6, 0.01, 0.9
    _yN, _loss, lit, ladj, rel = O.gd_grad(spec, x, y0, trueY, nIter, lr, m, loss_scale=3.0)
    assert rel.min() > 1e-6
    kf, kadj = O.kappa_form(spec, x, y0, trueY, nIter, lr, m, loss_scale=3.0)
    Lc, NL = len(spec.convs), len(spec.convs) + len(spec.fcs)
    out_d = {"z%d_u/W" % (NL - 1), "z%d_u/b" % (NL - 1)}
    assert set(lit) == set(kf) - out_d
    for k in out_d:
        assert not np.any(kf[k])
    scale = max(np.abs(g).max() for g in lit.values())
    for k, g in lit.items():
        assert np.abs(g - kf[k]).max() <= 1e-10 * max(1.0, scale), k
    for k in ("dcy", "dcz"):
        for a, b in zip(ladj[k], kadj[k]):
            if a is not None:
                assert np.abs(a - b).max() <= 1e-10 * max(1.0, np.abs(b).max()), k
    for a in kadj["dd"]:
        assert not np.any(a)
    for l in range(Lc - 1):                 # in gv_, exactly zero
        assert not np.any(lit["z%d_y_red/b" % l])
    for i in range(NL - 1):
        assert not np.any(lit["z%d_u/W" % i]) and not np.any(lit["z%d_u/b" % i])


def test_zero_steps_give_zero_gradients():
    spec, x, y0, trueY = _tiny()
    yN, _loss, lit, _adj, _rel = O.gd_grad(spec, x, y0, trueY, 0)
    np.testing.assert_array_equal(yN, y0)
    assert lit == {}
