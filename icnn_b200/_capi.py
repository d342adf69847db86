"""ctypes binding of libicnn_b200.so (include/icnn_b200.h).

This is the thin C-ABI layer the north-star asks for: Python passes raw device pointers (torch
tensors are only the containers/allocators) and a CUDA stream handle.  There is NO fallback: if
the shared library is missing the import fails loudly, and every compute call fails without a
CUDA device.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libicnn_b200.so")

ABI_VERSION = 9
NSTAT = 8
K2_PLAN_LEN = 8     # ICNN_K2_PLAN_LEN: int32 fields of an icnn_k2_plan / icnn_k2_last_launch record

# status / enum mirrors of include/icnn_b200.h
ST_RUNNING, ST_RANK_STOP, ST_SOLVE_FAIL, ST_NONFINITE, ST_CONVERGED = 0, 2, 3, 4, 5
VARIANT = {"lib": 0, "dual": 1, "rl": 2}
SOLVER_PC, SOLVER_NEWTON = 0, 1

# every symbol include/icnn_b200.h declares (tests check the .so exports each of them)
SYMBOLS = [
    "icnn_last_error", "icnn_abi_version", "icnn_device_count",
    "icnn_picnn_create", "icnn_picnn_destroy", "icnn_picnn_workspace_bytes", "icnn_picnn_fg",
    "icnn_bundle_init", "icnn_bundle_put_fg", "icnn_bundle_put_fg_f64", "icnn_bundle_step",
    "icnn_solve_batch_fused", "icnn_gd_solve", "icnn_tc_gemm_selftest", "icnn_argmin_grad",
    "icnn_picnn_set_xpath", "icnn_picnn_gates_workspace_bytes", "icnn_picnn_gates",
    "icnn_adam_workspace_bytes", "icnn_adam_solve",
    "icnn_gd_backward_workspace_bytes", "icnn_gd_backward", "icnn_fp64_mma_probe",
    "icnn_loop_graph_create", "icnn_loop_graph_launch", "icnn_loop_graph_nodes", "icnn_loop_graph_destroy",
    "icnn_tc_set_tuning", "icnn_tc_last_launch", "icnn_k2_plan", "icnn_k2_last_launch",
    "icnn_train_grad_workspace_bytes", "icnn_train_grad",
    "icnn_conv_picnn_create", "icnn_conv_picnn_destroy", "icnn_conv_picnn_workspace_bytes", "icnn_conv_picnn_fg",
    "icnn_conv_solve_batch_fused", "icnn_conv_gd_solve",
    "icnn_conv_train_grad_workspace_bytes", "icnn_conv_train_grad",
    "icnn_conv_gd_backward_workspace_bytes", "icnn_conv_gd_backward",
    "icnn_td_grad_workspace_bytes", "icnn_td_grad",
]

_fpp = C.POINTER(C.c_void_p)


class PicnnDesc(C.Structure):
    _fields_ = [("n", C.c_int32), ("L", C.c_int32), ("hidden", C.POINTER(C.c_int32)),
                ("alpha", C.c_float), ("Wy", _fpp), ("Wz", _fpp)]


class ConvPicnnDesc(C.Structure):
    _fields_ = [("H", C.c_int32), ("W", C.c_int32), ("Lc", C.c_int32), ("C", C.POINTER(C.c_int32)),
                ("k", C.POINTER(C.c_int32)), ("s", C.POINTER(C.c_int32)), ("Ld", C.c_int32),
                ("fcs", C.POINTER(C.c_int32)), ("Wz", _fpp), ("Wy", _fpp), ("Wred", _fpp), ("bred", _fpp)]


class Gates(C.Structure):
    _fields_ = [("B", C.c_int32), ("cy", _fpp), ("cz", _fpp), ("d", _fpp),
                ("in_scale", C.c_float), ("in_shift", C.c_float), ("g_scale", C.c_float)]


class BundleBufs(C.Structure):
    _fields_ = [("B", C.c_int32), ("n", C.c_int32), ("KS", C.c_int32),
                ("y", C.c_void_p), ("y32", C.c_void_p), ("f", C.c_void_p), ("G", C.c_void_p),
                ("ys", C.c_void_p), ("h", C.c_void_p), ("lam", C.c_void_p), ("rsum", C.c_void_p),
                ("gram", C.c_void_p), ("perm", C.c_void_p), ("count", C.c_void_p),
                ("status", C.c_void_p), ("finished", C.c_void_p), ("nIters", C.c_void_p),
                ("nactive", C.c_void_p), ("newton_its", C.c_void_p), ("ksum", C.c_void_p),
                ("f64", C.c_void_p), ("iter_stats", C.c_void_p)]


class BundleCfg(C.Structure):
    _fields_ = [("variant", C.c_int32), ("solver", C.c_int32), ("line_search", C.c_int32),
                ("max_inner", C.c_int32), ("prune_thr", C.c_double), ("rank_tol", C.c_double),
                ("nIter", C.c_int32), ("reserved", C.c_int32)]


class GdGrads(C.Structure):
    _fields_ = [("dWy", _fpp), ("dWz", _fpp), ("dcy", _fpp), ("dcz", _fpp)]


class TrainGrads(C.Structure):
    _fields_ = [("dWy", _fpp), ("dWz", _fpp), ("dcy", _fpp), ("dcz", _fpp), ("dd", _fpp)]


class ConvTrainGrads(C.Structure):
    _fields_ = [("dWz", _fpp), ("dWy", _fpp), ("dWred", _fpp), ("dbred", _fpp), ("dcy", _fpp), ("dcz", _fpp),
                ("dd", _fpp)]


class IcnnError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "icnn_b200: %s not found -- build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'` or `make -C icnn_b200/csrc`.  There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    lib.icnn_last_error.restype = C.c_char_p
    lib.icnn_abi_version.restype = C.c_int
    lib.icnn_device_count.restype = C.c_int
    lib.icnn_picnn_create.argtypes = [C.POINTER(PicnnDesc), C.POINTER(C.c_void_p), C.c_void_p]
    lib.icnn_picnn_destroy.argtypes = [C.c_void_p]
    lib.icnn_picnn_workspace_bytes.argtypes = [C.c_void_p, C.c_int32]
    lib.icnn_picnn_workspace_bytes.restype = C.c_size_t
    lib.icnn_picnn_fg.argtypes = [C.c_void_p, C.POINTER(Gates), C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                  C.c_void_p, C.c_void_p]
    lib.icnn_bundle_init.argtypes = [C.POINTER(BundleBufs), C.c_int32, C.c_void_p]
    lib.icnn_bundle_put_fg.argtypes = [C.POINTER(BundleBufs), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.icnn_bundle_put_fg_f64.argtypes = [C.POINTER(BundleBufs), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.icnn_bundle_step.argtypes = [C.POINTER(BundleCfg), C.POINTER(BundleBufs), C.c_int32, C.c_void_p]
    lib.icnn_solve_batch_fused.argtypes = [C.c_void_p, C.POINTER(Gates), C.POINTER(BundleCfg),
                                           C.POINTER(BundleBufs), C.c_void_p, C.c_void_p]
    lib.icnn_gd_solve.argtypes = [C.c_void_p, C.POINTER(Gates), C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_int32, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
    lib.icnn_tc_gemm_selftest.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                          C.c_void_p, C.c_void_p]
    lib.icnn_tc_set_tuning.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    lib.icnn_tc_last_launch.argtypes = [C.POINTER(C.c_int32)]
    lib.icnn_k2_plan.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32)]
    lib.icnn_k2_last_launch.argtypes = [C.POINTER(C.c_int32)]
    lib.icnn_picnn_set_xpath.argtypes = [C.c_void_p, C.c_int32] + [_fpp] * 8 + [C.c_void_p]
    lib.icnn_picnn_gates_workspace_bytes.argtypes = [C.c_void_p, C.c_int32]
    lib.icnn_picnn_gates_workspace_bytes.restype = C.c_size_t
    lib.icnn_picnn_gates.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, _fpp, _fpp, _fpp, C.c_void_p, C.c_void_p]
    lib.icnn_adam_workspace_bytes.argtypes = [C.c_int32, C.c_int32]
    lib.icnn_adam_workspace_bytes.restype = C.c_size_t
    lib.icnn_adam_solve.argtypes = [C.c_void_p, C.POINTER(Gates), C.c_void_p, C.c_void_p, C.c_int32,
                                    C.POINTER(C.c_int32), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.icnn_argmin_grad.argtypes = [C.POINTER(BundleBufs), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p]
    lib.icnn_gd_backward_workspace_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    lib.icnn_gd_backward_workspace_bytes.restype = C.c_size_t
    lib.icnn_gd_backward.argtypes = [C.c_void_p, C.POINTER(Gates), C.c_void_p, C.c_void_p, C.c_float, C.c_int32,
                                     C.c_float, C.c_float, C.c_void_p, C.POINTER(GdGrads), C.c_void_p, C.c_void_p]
    lib.icnn_train_grad_workspace_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_int64]
    lib.icnn_train_grad_workspace_bytes.restype = C.c_size_t
    lib.icnn_train_grad.argtypes = [C.c_void_p, C.POINTER(Gates), C.POINTER(C.c_int64), C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.POINTER(TrainGrads), C.c_void_p, C.c_void_p]
    lib.icnn_fp64_mma_probe.argtypes = [C.c_int32, C.c_void_p, C.POINTER(C.c_double), C.c_void_p]
    lib.icnn_loop_graph_create.argtypes = [C.c_void_p, C.POINTER(Gates), C.POINTER(BundleCfg), C.POINTER(BundleBufs),
                                           C.c_void_p, C.POINTER(C.c_void_p)]
    lib.icnn_loop_graph_launch.argtypes = [C.c_void_p, C.c_void_p]
    lib.icnn_loop_graph_nodes.argtypes = [C.c_void_p]
    lib.icnn_loop_graph_nodes.restype = C.c_int64
    lib.icnn_loop_graph_destroy.argtypes = [C.c_void_p]
    lib.icnn_conv_picnn_create.argtypes = [C.POINTER(ConvPicnnDesc), C.POINTER(C.c_void_p), C.c_void_p]
    lib.icnn_conv_picnn_destroy.argtypes = [C.c_void_p]
    lib.icnn_conv_picnn_workspace_bytes.argtypes = [C.c_void_p, C.c_int32]
    lib.icnn_conv_picnn_workspace_bytes.restype = C.c_size_t
    lib.icnn_conv_picnn_fg.argtypes = lib.icnn_picnn_fg.argtypes
    lib.icnn_conv_solve_batch_fused.argtypes = lib.icnn_solve_batch_fused.argtypes
    lib.icnn_conv_gd_solve.argtypes = lib.icnn_gd_solve.argtypes
    lib.icnn_conv_train_grad_workspace_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_int64]
    lib.icnn_conv_train_grad_workspace_bytes.restype = C.c_size_t
    lib.icnn_conv_train_grad.argtypes = [C.c_void_p, C.POINTER(Gates), C.POINTER(C.c_int64), C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.POINTER(ConvTrainGrads), C.c_void_p, C.c_void_p]
    lib.icnn_conv_gd_backward_workspace_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    lib.icnn_conv_gd_backward_workspace_bytes.restype = C.c_size_t
    lib.icnn_conv_gd_backward.argtypes = [C.c_void_p, C.POINTER(Gates), C.c_void_p, C.c_void_p, C.c_float, C.c_int32,
                                          C.c_float, C.c_float, C.c_void_p, C.POINTER(ConvTrainGrads), C.c_void_p,
                                          C.c_void_p]
    lib.icnn_td_grad_workspace_bytes.argtypes = [C.c_void_p, C.c_int32]
    lib.icnn_td_grad_workspace_bytes.restype = C.c_size_t
    lib.icnn_td_grad.argtypes = [C.c_void_p, C.POINTER(Gates), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.POINTER(TrainGrads), C.c_void_p,
                                 C.c_void_p]
    for name in SYMBOLS:
        getattr(lib, name)  # AttributeError if the .so does not export it
    if lib.icnn_abi_version() != ABI_VERSION:
        raise ImportError("icnn_b200: ABI version mismatch (%d != %d); rebuild the library"
                          % (lib.icnn_abi_version(), ABI_VERSION))
    return lib


lib = _load()


def check(rc):
    if rc != 0:
        raise IcnnError("libicnn_b200 error %d: %s" % (rc, lib.icnn_last_error().decode()))


def ptr_array(tensors):
    """host array of device pointers (None -> NULL); keeps nothing alive -- caller must."""
    arr = (C.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = None if t is None else t.data_ptr()
    return arr
