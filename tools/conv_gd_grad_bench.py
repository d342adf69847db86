"""Conv-PICNN GD training gradient at C2-conv: the reference's completion architecture ((32,8,4), (64,4,2), (64,3,1) /
(512, 1)) at 64 x 32 with the weights of tools/conv_bench.py (oracle/conv_picnn.ConvPICNN(64, 32, seed=2)), the back-
optimisation mode's nIter = 30, lr = 0.01, momentum = 0.9, loss_scale = 2 255^2 / (B n), B = 70 (the reference's
trainBatchSz) and 400.

Per batch and run it prints CUDA-event times of
  solve         gd.solve(fg, y0, 30, 0.01, 0.9) (the forward loop alone, on the device)
  gd_grad       gd_grad(fg, y0, trueY, ...) with return_device=True: icnn_conv_gd_backward + the torch x-path
  library       icnn_conv_gd_backward alone (the loop, the row seeds and the training gradient of B nIter rows)
  torch_f32     eager torch float32 (TF32 off), inputs and weights already on the device: the gates, 30 unrolled steps
                with dE/dy by autograd (create_graph=True), the loss and its gradient over every trainable variable --
                what a user has without this library
and a header line with the card, its power limit and SM clock, read in the same process.
Usage: python tools/conv_gd_grad_bench.py [--batches 70,400] [--reps 5] [--runs 3]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="70,400")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--nIter", type=int, default=30)
    args = ap.parse_args()
    import icnn_b200
    from icnn_b200 import _capi, gd
    from icnn_b200.conv_picnn import _train_grad_buffers, parse_variables
    from icnn_b200.gd_grad import gd_grad
    from conv_bench import card, events_ms
    from oracle.conv_picnn import ConvPICNN as Helper
    from oracle import conv_train_grad_torch as O
    from oracle.gen_golden_tfshim import conv_variables
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    H, W, N, lr, m = 64, 32, args.nIter, 0.01, 0.9
    v = conv_variables(Helper(H, W, seed=2, dtype=torch.float64))
    net = icnn_b200.ConvPICNN.from_variables(v, H, W)
    spec = parse_variables(v, H, W)
    print(json.dumps(dict(card(), record="card")), flush=True)
    y_pix = np.random.RandomState(0).uniform(0.2, 0.8, size=(1, H * W))
    names = O.trainable(list(spec.vars), len(spec.convs), len(spec.fcs))
    dev = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float32), device="cuda").contiguous()   # noqa: E731
    P = {k: dev(a).requires_grad_(k in names) for k, a in spec.vars.items()}
    for B in [int(b) for b in args.batches.split(",")]:
        rs = np.random.RandomState(B)
        x = rs.uniform(size=(B, H * W))
        trueY = rs.uniform(size=(B, H * W))
        y0 = np.tile(y_pix, (B, 1))
        ls = 2 * 255.0 ** 2 / (B * H * W)
        fg = net.bind(x)
        xd, y0d, tYd = dev(x), dev(y0), dev(trueY)

        o, gr, arrs = _train_grad_buffers(fg)
        yN = torch.empty_like(y0d)
        ws = torch.empty(_capi.lib.icnn_conv_gd_backward_workspace_bytes(net._h, B, N), dtype=torch.uint8,
                         device="cuda")

        def library():
            _capi.check(_capi.lib.icnn_conv_gd_backward(
                net._h, C.byref(fg.c_gates), y0d.data_ptr(), tYd.data_ptr(), ls, N, lr, m, yN.data_ptr(),
                C.byref(gr), ws.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream)))

        def torch_f32():
            cz, cy, d = O.gates(P, spec, xd)
            y, vv = y0d.detach().requires_grad_(), 0.0
            for _ in range(N):
                E, _pres, _b = O.y_energy(P, spec, cz, cy, d, y)
                (g,) = torch.autograd.grad(E.sum(), y, create_graph=True)
                vn = m * vv - lr * g
                y, vv = y - m * vv + (1 + m) * vn, vn
            loss = 0.5 * ls * ((y - tYd) ** 2).sum()
            return torch.autograd.grad(loss, [P[k] for k in names], allow_unused=True)

        arms = dict(solve=lambda: gd.solve(fg, y0d, N, lr, m, return_device=True),
                    gd_grad=lambda: gd_grad(fg, y0d, tYd, N, lr, m, ls, return_device=True),
                    library=library, torch_f32=torch_f32)
        for fn in arms.values():      # warm-up
            fn()
        torch.cuda.synchronize()
        for run in range(args.runs):
            ms = {k: round(events_ms(fn, args.reps), 3) for k, fn in arms.items()}
            print(json.dumps(dict(record="conv_gd_grad", B=B, nIter=N, rows=B * N, run=run,
                                  **{k + "_ms": t for k, t in ms.items()},
                                  ws_mb=round(ws.numel() / 2 ** 20, 1))), flush=True)
        del o, arrs


if __name__ == "__main__":
    main()
