#!/usr/bin/env python
"""Conv-PICNN bundle-entropy solve on the device (ConvPICNN, fused) against callback mode with the torch float32
helper fg (TF32 off), which is how this energy ran before the fused path existed.

Workloads ("C2-conv"): the reference's completion architecture ((32,8,4), (64,4,2), (64,3,1) / (512, 1)) at 64 x 32,
lib PC solver, 30 iterations, B = 400 and the reference's trainBatchSz B = 70.  Weights: tests/conv_picnn.ConvPICNN(64,
32, seed=2) via conv_variables; x ~ U(0, 1); y0 one fixed per-pixel vector from U(0.2, 0.8) for every sample.

Prints one JSON line per (run, workload, arm) and a header line with the card, its power limit and SM clock, read in
the same process.  The two arms alternate, three runs.  FLOPs: 4 x the multiply-adds of one forward (forward +
backward, SURVEY.md section 8d) per sample and fg call, against the 3xTF32 ceiling (one third of the data sheet's
dense TF32 rate).  K2's share is derived: solve time minus nIter fused fg calls.
Usage: python tools/conv_bench.py [--runs 3] [--batches 400,70] [--nIter 30]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

TF32_DENSE_TFLOPS = 495.0     # H100 SXM data sheet, dense TF32; 3xTF32 issues three MMAs per product


def card():
    info = {"gpu": torch.cuda.get_device_name()}
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                                     "--format=csv,noheader"], text=True).splitlines()[0]
        info["power_limit"], info["sm_clock"], info["sm_clock_max"] = [s.strip() for s in q.split(",")]
    except (OSError, subprocess.CalledProcessError) as e:
        info["nvidia_smi"] = "unavailable: %s" % e
    return info


def fg_macs(net):
    """multiply-adds of one forward of the y-path per sample (the backward costs the same)."""
    macs, h, w = 0, net.H, net.W
    cp = 0
    for C, k, s in net.convs:
        h, w = -(-h // s), -(-w // s)
        macs += h * w * k * k * (cp + 1) * C
        cp = C
    prev = h * w * cp
    for sz in net.fcs:
        macs += prev * sz
        prev = sz
    return macs


def events_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batches", default="400,70")
    ap.add_argument("--nIter", type=int, default=30)
    args = ap.parse_args()
    import icnn_b200
    from icnn_b200 import bundle_entropy as be
    from conv_picnn import ConvPICNN as Helper
    from oracle.gen_golden_tfshim import conv_variables
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    H, W, nIter = 64, 32, args.nIter
    helper64 = Helper(H, W, seed=2, dtype=torch.float64)
    net = icnn_b200.ConvPICNN.from_variables(conv_variables(helper64), H, W)
    helper32 = helper64.to(torch.float32, "cuda")
    print(json.dumps(dict(card(), record="card")), flush=True)
    rs = np.random.RandomState(0)
    y_pix = rs.uniform(0.2, 0.8, size=(1, H * W))
    work = {}
    for B in [int(b) for b in args.batches.split(",")]:
        x = np.random.RandomState(B).uniform(size=(B, H * W))
        y0 = np.tile(y_pix, (B, 1))
        fg = net.bind(x)
        cb = helper32.make_fg(x)
        st = be.solveBatch(fg, y0.copy(), nIter=nIter, return_state=True)[-1]     # warm-up, keeps the state
        be.solveBatch(cb, y0.copy(), nIter=nIter)
        work[B] = (x, y0, fg, cb, st)
    flop_fg = 4 * fg_macs(net)
    for run in range(args.runs):
        for B, (x, y0, fg, cb, st) in work.items():
            for arm in ("fused", "callback"):
                y32 = torch.as_tensor(y0, dtype=torch.float32, device="cuda")
                if arm == "fused":
                    solve_ms = events_ms(lambda: be.solveBatch(fg, y0.copy(), nIter=nIter, state=st), 3)
                    fg_ms = events_ms(lambda: fg.fg_device(y32), 20)
                else:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(3):
                        be.solveBatch(cb, y0.copy(), nIter=nIter)
                    torch.cuda.synchronize()
                    solve_ms = (time.perf_counter() - t0) * 1e3 / 3
                    fg_ms = events_ms(lambda: cb(y0), 5)
                rec = dict(record="solve", run=run, workload="C2-conv", B=B, nIter=nIter, arm=arm,
                           ms_per_solve=round(solve_ms, 3), solves_per_s=round(B * 1e3 / solve_ms, 1),
                           ms_per_fg=round(fg_ms, 4))
                if arm == "fused":
                    k2 = max(solve_ms - nIter * fg_ms, 0.0)
                    flops = flop_fg * B * nIter
                    rec.update(k2_ms_derived=round(k2, 3), k2_share=round(k2 / solve_ms, 3),
                               fg_flops_per_solve=flops,
                               fg_tflops=round(flop_fg * B / (fg_ms * 1e-3) / 1e12, 2),
                               fg_share_of_3xtf32_ceiling=round(flop_fg * B / (fg_ms * 1e-3) / 1e12
                                                                / (TF32_DENSE_TFLOPS / 3), 4))
                print(json.dumps(rec), flush=True)
    print(json.dumps(dict(card(), record="card_end")), flush=True)


if __name__ == "__main__":
    main()
