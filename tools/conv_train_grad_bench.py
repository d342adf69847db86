"""Conv-PICNN training gradient at C2-conv: the reference's completion architecture ((32,8,4), (64,4,2), (64,3,1) /
(512, 1)) at 64 x 32 with the weights of tools/conv_bench.py (oracle/conv_picnn.ConvPICNN(64, 32, seed=2)), 30 solver
iterations, B = 70 (the reference's trainBatchSz) and 400.

Per batch it prints R (the train_step_fd rows the solve leaves) and CUDA-event times of
  solve         bundle_entropy.solveBatch(fg, y0, nIter=30, return_state=True) (fused on the device)
  bundle_grad   K3 (mse) + the device row gather + icnn_conv_train_grad + the torch x-path (return_device=True)
  library       icnn_conv_train_grad alone on the same rows
  torch_f32     eager torch float32 (TF32 off) on the same rows, inputs and weights already on the device: the gates,
                E, dE/dy (create_graph=True), F = sum_r c_r E_r + V_r . dE/dy and dF/dtheta over every trainable
                variable, no host copies -- what a user has without this library
and a header line with the card, its power limit and SM clock, read in the same process.
Usage: python tools/conv_train_grad_bench.py [--batches 70,400] [--reps 5]
"""
import argparse
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
    ap.add_argument("--nIter", type=int, default=30)
    args = ap.parse_args()
    import icnn_b200
    from icnn_b200 import argmin_grad, bundle_entropy as be
    from icnn_b200.bundle_grad import _conv_launch, bundle_grad
    from icnn_b200.conv_picnn import parse_variables
    from conv_bench import card, events_ms
    from oracle.conv_picnn import ConvPICNN as Helper
    from oracle import conv_train_grad_torch as O
    from oracle.gen_golden_tfshim import conv_variables
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    H, W = 64, 32
    v = conv_variables(Helper(H, W, seed=2, dtype=torch.float64))
    net = icnn_b200.ConvPICNN.from_variables(v, H, W)
    spec = parse_variables(v, H, W)
    print(json.dumps(dict(card(), record="card")), flush=True)
    y_pix = np.random.RandomState(0).uniform(0.2, 0.8, size=(1, H * W))
    for B in [int(b) for b in args.batches.split(",")]:
        rs = np.random.RandomState(B)
        x = rs.uniform(size=(B, H * W))
        trueY = rs.uniform(size=(B, H * W))
        y0 = np.tile(y_pix, (B, 1))
        fg = net.bind(x)
        st = be.solveBatch(fg, y0.copy(), nIter=args.nIter, return_state=True)[-1]
        _cy, _cl, _ct, (fY, fV, fc) = argmin_grad.argmin_grad(st, trueY, loss="mse")
        counts = st.count.cpu().numpy().astype(np.int64)
        offsets = np.concatenate([[0], np.cumsum(counts)])
        dev = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float32), device="cuda").contiguous()   # noqa: E731
        Yd, Vd, cd = dev(fY), dev(fV), dev(fc)
        R = int(offsets[-1])
        names = O.trainable(list(spec.vars), len(spec.convs), len(spec.fcs))
        P = {k: dev(a).requires_grad_(k in names) for k, a in spec.vars.items()}
        xd, iu = dev(x), torch.as_tensor(np.repeat(np.arange(B), counts), device="cuda")

        def torch_f32():
            cz, cy, d = O.gates(P, spec, xd)
            rows = lambda lst: [None if g is None else g[iu] for g in lst]   # noqa: E731
            y = Yd.detach().requires_grad_()
            E, _pres, _b = O.y_energy(P, spec, rows(cz), rows(cy), rows(d), y)
            (gy,) = torch.autograd.grad(E.sum(), y, create_graph=True)
            return torch.autograd.grad((cd * E).sum() + (Vd * gy).sum(), [P[k] for k in names])

        bundle_grad(fg, st, trueY, loss="mse", return_device=True)       # warm-up
        torch_f32()
        solve_ms = events_ms(lambda: be.solveBatch(fg, y0.copy(), nIter=args.nIter, return_state=True), args.reps)
        bg_ms = events_ms(lambda: bundle_grad(fg, st, trueY, loss="mse", return_device=True), args.reps)
        keep = []
        lib_ms = events_ms(lambda: keep.append(_conv_launch(fg, Yd, Vd, cd, offsets)), args.reps)
        torch.cuda.synchronize()
        keep.clear()
        t32_ms = events_ms(torch_f32, args.reps)
        print(json.dumps(dict(record="conv_train_grad", B=B, nIter=args.nIter, R=R, solve_ms=round(solve_ms, 3),
                              bundle_grad_ms=round(bg_ms, 3), library_ms=round(lib_ms, 3),
                              torch_f32_ms=round(t32_ms, 3),
                              ws_mb=round(icnn_b200._capi.lib.icnn_conv_train_grad_workspace_bytes(net._h, B, R) / 2**20,
                                          1))), flush=True)


if __name__ == "__main__":
    main()
