"""Host-side handle of a fully-connected PICNN and the `fg` object bound to a minibatch of x.

Mirrors the role of the TF graph + ``fg`` closure in the reference
(multi-label-cls/icnn_ebundle.py:218-221, RL/src/icnn.py:127,150-153): ``PICNN.bind(x)`` returns
a callable ``fg(y) -> (f, g)`` with the reference's numpy contract, which ``solveBatch`` also
recognises to run the whole inner loop on the device without a host round trip.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _capi


def default_device():
    """Device used when the caller names none: ``cuda`` (torch's current device), or -- the device-list environment
    variable of SURVEY.md section 5 -- entry LOCAL_RANK of ``ICNN_DEVICES`` (comma-separated CUDA ordinals, e.g.
    ``ICNN_DEVICES=4,5,6,7`` under torchrun with four ranks, or a single ordinal for a single process)."""
    import os
    lst = [s for s in os.environ.get("ICNN_DEVICES", "").split(",") if s.strip()]
    if lst:
        return torch.device("cuda", int(lst[int(os.environ.get("LOCAL_RANK", "0")) % len(lst)]))
    return torch.device("cuda")


def _dev(a, device):
    if isinstance(a, torch.Tensor):
        return a.to(device=device, dtype=torch.float32).contiguous()
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device=device)


class PICNN:
    """Weights of a fully-connected PICNN on one CUDA device.

    y-path (the hot recurrence; handed to the C library, which keeps its own packed copy):
        Wy[i] [n, s_i], Wz[i] [s_{i-1}, s_i] (Wz[0] None), i = 0..L, s_L = 1
    x-path (once per solveBatch; multi-label-cls/icnn_ebundle.py:339-373):
        Wu/bu, Wzu/bzu, Wyu/byu, Wzx/bzx   -- same names as oracle/picnn_np.PicnnParams
    ``alpha``: leaky-ReLU slope of the z path (0 = ReLU).
    """

    def __init__(self, m, n, hidden, Wy, Wz, Wu, bu, Wzu, bzu, Wyu, byu, Wzx, bzx, alpha=0.0,
                 device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("icnn_b200.PICNN needs a CUDA device (no CPU fallback)")
        self.device = torch.device(device) if device is not None else default_device()
        self.m, self.n, self.hidden, self.alpha = int(m), int(n), [int(s) for s in hidden], float(alpha)
        self.L = len(self.hidden)
        L = self.L
        d = self.device
        self.Wy = [_dev(w, d) for w in Wy]
        self.Wz = [None] + [_dev(w, d) for w in Wz[1:]]
        self.Wu = [_dev(w, d) for w in Wu]
        self.bu = [_dev(w, d) for w in bu]
        self.Wzu = [None] + [_dev(w, d) for w in Wzu[1:]]
        self.bzu = [None] + [_dev(w, d) for w in bzu[1:]]
        self.Wyu = [_dev(w, d) for w in Wyu]
        self.byu = [_dev(w, d) for w in byu]
        self.Wzx = [_dev(w, d) for w in Wzx]
        self.bzx = [_dev(w, d) for w in bzx]
        assert len(self.Wy) == L + 1 and len(self.Wz) == L + 1
        self._h = None
        self._pack()

    def _weight_tensors(self):
        return [t for lst in (self.Wy, self.Wz, self.Wu, self.bu, self.Wzu, self.bzu, self.Wyu, self.byu, self.Wzx, self.bzx)
                for t in lst if t is not None]

    def _pack(self):
        """Hand the current weight tensors to the C library (it keeps its own packed / TF32-split copies)."""
        L = self.L
        if self._h is not None and self._h.value:
            _capi.lib.icnn_picnn_destroy(self._h)
            self._h = None
        hid = (C.c_int32 * L)(*self.hidden)
        wy = _capi.ptr_array(self.Wy)
        wz = _capi.ptr_array(self.Wz)
        desc = _capi.PicnnDesc(self.n, L, hid, self.alpha, C.cast(wy, _capi._fpp), C.cast(wz, _capi._fpp))
        handle = C.c_void_p()
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            _capi.check(_capi.lib.icnn_picnn_create(C.byref(desc), C.byref(handle), C.c_void_p(stream)))
        self._h = handle
        # x-path gate precompute on the library's wgmma GEMM when the shapes allow it
        # (SURVEY.md section 8f row 2); otherwise plain cuBLAS GEMMs through torch.addmm
        self._xpath = False
        with torch.cuda.device(self.device):
            args = [_capi.ptr_array(v) for v in (self.Wu, self.bu, self.Wzu, self.bzu, self.Wyu, self.byu,
                                                  self.Wzx, self.bzx)]
            rc = _capi.lib.icnn_picnn_set_xpath(self._h, self.m, *[C.cast(a, _capi._fpp) for a in args],
                                                C.c_void_p(torch.cuda.current_stream().cuda_stream))
            if rc == 0:
                self._xpath = True
            elif rc != -3:           # -3 = ICNN_E_UNSUPPORTED (width not a multiple of 4 / SIMT-only build)
                _capi.check(rc)
        self._versions = [t._version for t in self._weight_tensors()]
        self._pack_gen = getattr(self, "_pack_gen", 0) + 1   # captured loop graphs bake the packed buffers in

    def update_weights(self):
        """Re-pack after the weight tensors were modified in place (an optimiser step, makeCvx / proj:
        multi-label-cls/icnn_ebundle.py:140-144).  The library works on its own packed copies, so without this
        call K1 / the gate GEMMs would keep using the old values; ``bind`` refuses to run on stale copies."""
        with torch.cuda.device(self.device):
            self._pack()

    def _check_fresh(self):
        if [t._version for t in self._weight_tensors()] != self._versions:
            raise RuntimeError("PICNN: a weight tensor was modified in place after it was packed for the device "
                               "library; call net.update_weights() before bind()")

    @classmethod
    def from_params(cls, p, device=None):
        """Build from any object with the attribute names of oracle/picnn_np.PicnnParams.  An inference-mode
        batch-norm on the u-path (``p.bn``, multi-label-cls/icnn_ebundle.py:343-345) is folded into the
        weights of its consumers (workloads.fold_batchnorm): the handle then holds the folded x-path weights."""
        if any(b is not None for b in getattr(p, "bn", []) or []):
            from .workloads import fold_batchnorm
            p = fold_batchnorm(p)
        return cls(p.m, p.n, p.hidden, p.Wy, p.Wz, p.Wu, p.bu, p.Wzu, p.bzu, p.Wyu, p.byu, p.Wzx,
                   p.bzx, alpha=p.alpha, device=device)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                _capi.lib.icnn_picnn_destroy(h)
            except Exception:
                pass
            self._h = None

    def workspace(self, B):
        nbytes = _capi.lib.icnn_picnn_workspace_bytes(self._h, int(B))
        return torch.empty(max(nbytes, 4), dtype=torch.uint8, device=self.device)

    def gates(self, x):
        """x-path products (cz, cy, d), constant over the inner loop (SURVEY.md section 8f row 2): one wgmma GEMM per
        source activation with a bias / ReLU / scatter epilogue (``icnn_picnn_gates``).  Only when the library reports
        the shape unsupported (``icnn_picnn_set_xpath`` -> ICNN_E_UNSUPPORTED, e.g. ICNN_K1=simt builds of the handle)
        the same products are formed by library GEMMs (torch.addmm -> cuBLAS): a once-per-solveBatch precompute,
        outside the hot loop."""
        x = _dev(x, self.device)
        L = self.L
        if self._xpath:
            B = int(x.shape[0])
            e = lambda w: torch.empty(B, w, dtype=torch.float32, device=self.device)  # noqa: E731
            cz = [None] + [e(self.hidden[i - 1]) for i in range(1, L + 1)]
            cy = [e(self.n) for _ in range(L + 1)]
            d = [e(self.hidden[i]) if i < L else e(1) for i in range(L + 1)]
            nbytes = _capi.lib.icnn_picnn_gates_workspace_bytes(self._h, B)
            ws = torch.empty(max(nbytes, 4), dtype=torch.uint8, device=self.device)
            pz, py, pd = _capi.ptr_array(cz), _capi.ptr_array(cy), _capi.ptr_array(d)
            _capi.check(_capi.lib.icnn_picnn_gates(self._h, x.data_ptr(), B, C.cast(pz, _capi._fpp),
                                                   C.cast(py, _capi._fpp), C.cast(pd, _capi._fpp), ws.data_ptr(),
                                                   C.c_void_p(torch.cuda.current_stream().cuda_stream)))
            self._gates_ws = ws     # keep alive until the stream has consumed it
            return cz, cy, d
        us, prev = [], x
        for i in range(L):
            u = torch.addmm(self.bu[i], prev, self.Wu[i])
            if i < L - 1:
                u = torch.relu(u)
            us.append(u)
            prev = u
        cz, cy, d = [None] * (L + 1), [None] * (L + 1), [None] * (L + 1)
        for i in range(L + 1):
            P = x if i == 0 else us[i - 1]
            if i > 0:
                cz[i] = torch.relu(torch.addmm(self.bzu[i], P, self.Wzu[i])).contiguous()
            cy[i] = torch.addmm(self.byu[i], P, self.Wyu[i]).contiguous()
            d[i] = torch.addmm(self.bzx[i], P, self.Wzx[i]).contiguous()
        return cz, cy, d

    def bind(self, x, affine=False):
        """fg object for a minibatch x [B, m].  ``affine=True`` = the RL wrapper
        (RL/src/icnn.py:148-153): solver variable in [0,1], action a = 2x-1, gradient * 2."""
        self._check_fresh()
        return BoundPICNN(self, x, affine)


class BoundPICNN:
    """``fg`` for one minibatch: callable with the reference's numpy contract, and the handle
    solveBatch uses for the fused device loop."""

    def __init__(self, net: PICNN, x, affine=False):
        self.net = net
        self.affine = bool(affine)
        with torch.cuda.device(net.device):
            self.cz, self.cy, self.d = net.gates(x)
        self.B = int(self.cy[0].shape[0])
        self._cy = _capi.ptr_array(self.cy)
        self._cz = _capi.ptr_array(self.cz)
        self._d = _capi.ptr_array(self.d)
        s, sh, gs = (2.0, -1.0, 2.0) if self.affine else (1.0, 0.0, 1.0)
        self.c_gates = _capi.Gates(self.B, C.cast(self._cy, _capi._fpp), C.cast(self._cz, _capi._fpp),
                                   C.cast(self._d, _capi._fpp), s, sh, gs)
        self.ws = net.workspace(self.B)

    def fg_device(self, y32, f=None, g=None):
        """f [B], g [B, n] (float32 CUDA tensors) for a float32 CUDA iterate y32 [B, n]."""
        net = self.net
        assert y32.is_cuda and y32.dtype == torch.float32 and y32.is_contiguous()
        assert tuple(y32.shape) == (self.B, net.n)
        if f is None:
            f = torch.empty(self.B, dtype=torch.float32, device=net.device)
        if g is None:
            g = torch.empty(self.B, net.n, dtype=torch.float32, device=net.device)
        with torch.cuda.device(net.device):
            stream = torch.cuda.current_stream().cuda_stream
            _capi.check(_capi.lib.icnn_picnn_fg(
                net._h, C.byref(self.c_gates), y32.data_ptr(), f.data_ptr(), g.data_ptr(),
                net.n, None, None, 0, self.ws.data_ptr(), None, C.c_void_p(stream)))
        return f, g

    def __call__(self, y):
        """numpy in, numpy out: fg(y [B,n]) -> (f [B] float32, g [B,n] float32), like the
        reference's TF-backed closure (float32 fetch)."""
        y32 = torch.as_tensor(np.ascontiguousarray(y, dtype=np.float32), device=self.net.device)
        f, g = self.fg_device(y32)
        return f.cpu().numpy(), g.cpu().numpy()
