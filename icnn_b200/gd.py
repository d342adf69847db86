"""Unrolled momentum gradient-descent inner loop on the device.

Reproduces the forward inner loop the reference unrolls in its TF graph
(multi-label-cls/icnn-back.py:116-131 = completion/icnn.back.py:133-147 =
synthetic-cls/icnn.py:117-131):   v' = m v - lr * dE/dy(y);  y' = y - m v + (1 + m) v'
with v_0 = 0 and no projection; returns (y_n, E(y_n)).  Defaults are the multi-label script's
(--inference_lr .01 --inference_momentum .3 --inference_nIter 30, icnn-back.py:36-38).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _capi
from .conv_picnn import BoundConvPICNN
from .picnn import BoundPICNN


def solve(fg: BoundPICNN, y0, nIter=30, lr=0.01, momentum=0.3, return_device=False):
    """``fg``: a BoundPICNN or, for the image-completion energy (completion/icnn.back.py:133-147), a
    BoundConvPICNN."""
    if not isinstance(fg, (BoundPICNN, BoundConvPICNN)):
        raise TypeError("gd.solve needs a BoundPICNN (PICNN.bind(x)) or a BoundConvPICNN (ConvPICNN.bind(x)); for "
                        "arbitrary callables use your framework's own loop")
    gd_solve = _capi.lib.icnn_conv_gd_solve if isinstance(fg, BoundConvPICNN) else _capi.lib.icnn_gd_solve
    net = fg.net
    dev = net.device
    with torch.cuda.device(dev):
        if isinstance(y0, torch.Tensor):
            y = y0.to(device=dev, dtype=torch.float32).contiguous().clone()
        else:
            y = torch.as_tensor(np.ascontiguousarray(y0, dtype=np.float32), device=dev)
        assert tuple(y.shape) == (fg.B, net.n)
        v = torch.empty_like(y)
        g = torch.empty_like(y)
        f = torch.empty(fg.B, dtype=torch.float32, device=dev)
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        _capi.check(gd_solve(net._h, C.byref(fg.c_gates), y.data_ptr(), v.data_ptr(),
                                            g.data_ptr(), f.data_ptr(), int(nIter), float(lr),
                                            float(momentum), fg.ws.data_ptr(), stream))
        if return_device:
            return y, f
        return y.cpu().numpy(), f.cpu().numpy()
