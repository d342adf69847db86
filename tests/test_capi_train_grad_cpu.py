"""CPU-only checks of the training-gradient entry points of the C ABI: null arguments are rejected with
ICNN_E_INVALID before any device is touched, and the workspace query refuses what it cannot size."""
import ctypes as C


def test_train_grad_rejects_null_arguments_without_touching_the_gpu():
    from icnn_b200 import _capi
    lib = _capi.lib
    assert lib.icnn_train_grad(None, None, None, None, None, None, None, None, None) == -1
    assert b"null" in lib.icnn_last_error()
    off = (C.c_int64 * 2)(0, 0)
    gates = _capi.Gates()
    grads = _capi.TrainGrads()          # all five pointer arrays NULL
    ws = C.c_void_p(16)                 # never dereferenced: the call is refused first
    assert lib.icnn_train_grad(C.c_void_p(8), C.byref(gates), off, None, None, None, C.byref(grads), ws, None) == -1
    assert b"null gradient array" in lib.icnn_last_error()
    assert lib.icnn_train_grad_workspace_bytes(None, 4, 10) == 0
