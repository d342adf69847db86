"""icnn_b200 -- H100-native inner loop argmin_y f(x, y; theta) of locuslab/icnn.

Public surface (mirrors the reference's, see INTEGRATION.md):
    icnn_b200.bundle_entropy.solveBatch(fg, initXs, nIter, callback, solver, variant=...)
    icnn_b200.PICNN(...).bind(x)         -> the fg object for the fused on-device loop
    icnn_b200.ConvPICNN.from_variables(vars, H, W).bind(x) -> the same for the image-completion conv PICNN
    icnn_b200.gd.solve(...)              -> unrolled momentum gradient descent
    icnn_b200.argmin_grad.argmin_grad(state, trueY, loss) -> crossEntrGrad / mseGrad + train_step_fd feeds
    icnn_b200.gd_grad.gd_grad(fg, y0, trueY, ...) -> d mse / d theta through the unrolled GD loop
    icnn_b200.bundle_grad.bundle_grad(fg, state, trueY, loss) -> the bundle-entropy training gradient dF/dtheta
The compute path is hand-written sm_90a CUDA behind a C ABI (libicnn_b200.so).  Every attribute above
loads the native library on first use and raises ImportError when it is missing -- there is no CPU
fallback.  Only ``icnn_b200.workloads`` (pure-numpy synthetic inputs, shared with the CPU reference arm of
bench.py) imports without it, so that the reference arm maps no native code.
"""
import importlib

_LAZY = {
    "PICNN": ("picnn", "PICNN"), "BoundPICNN": ("picnn", "BoundPICNN"),
    "ConvPICNN": ("conv_picnn", "ConvPICNN"), "BoundConvPICNN": ("conv_picnn", "BoundConvPICNN"),
    "conv_picnn": ("conv_picnn", None),
    "bundle_entropy": ("bundle_entropy", None), "gd": ("gd", None), "argmin_grad": ("argmin_grad", None),
    "adam": ("adam", None), "gd_grad": ("gd_grad", None),
    "bundle_grad": ("bundle_grad", None), "dist": ("dist", None), "_capi": ("_capi", None),
    "workloads": ("workloads", None),
}

__all__ = ["PICNN", "BoundPICNN", "ConvPICNN", "BoundConvPICNN", "conv_picnn", "bundle_entropy", "gd", "argmin_grad", "adam", "gd_grad", "bundle_grad"]


def __getattr__(name):
    if name in _LAZY:
        mod, attr = _LAZY[name]
        m = importlib.import_module("." + mod, __name__)     # ._capi raises ImportError if the .so is missing
        v = m if attr is None else getattr(m, attr)
        globals()[name] = v
        return v
    raise AttributeError("module %r has no attribute %r" % (__name__, name))
