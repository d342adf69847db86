#!/usr/bin/env python
"""Timing of the bundle-entropy training gradient (icnn_b200.bundle_grad) at C3 (B = 4096, 10 iterations) and T
(B = 4096, n = 512), after warm-up, next to the solveBatch and K3 (argmin_grad) that precede it in the reference's
training step (multi-label-cls/icnn_ebundle.py:225-245).  CUDA-event times; prints one JSON line per workload.

  bundle_grad_ms        K3 + row gather + icnn_train_grad + x-path backprop (the whole call, x given)
  train_grad_ms         the icnn_train_grad library call alone on the gathered rows, CUDA events around that call only
                        (buffers and workspace allocated beforehand); the time of the rows/s and FLOP rates
  algorithmic FLOPs     8 * MAC per row: forward, tangent, backward, weight gradient; MAC = n sum s_l +
                        sum s_{l-1} s_l (SURVEY.md section 8d), against the bf16 peak and the 3xTF32 ceiling
                        (bf16 peak / 6) the way bench.py reports K1

Usage: python tools/train_grad_bench.py [C3] [T] [--loss xent|mse]
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import icnn_b200  # noqa: E402
from icnn_b200 import argmin_grad, bundle_entropy as be, workloads  # noqa: E402
from icnn_b200.bundle_grad import _launch, _prepare, bundle_grad  # noqa: E402
from bench import flop_fg, load_peaks  # noqa: E402


def timeit_events(fn, reps=5, warm=2):
    """Mean CUDA-event time of fn() with the events recorded right around each call (host work outside excluded)."""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    total = 0.0
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        total += e0.elapsed_time(e1)
    return total / reps


def timeit(fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def gpu_info():
    name = torch.cuda.get_device_name()
    try:
        idx = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or "0"
        out = subprocess.run(["nvidia-smi", "-i", idx, "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        power = float(out)
    except Exception:
        power = None
    return name, power


def run(name, loss):
    cfg = dict(workloads.CONFIGS[name])
    B, nIter = 4096, cfg["nIter"]
    cfg["B"] = B
    p, x, y0 = workloads.make_inputs(name, B=B)
    tY = (np.random.RandomState(5).uniform(size=y0.shape) < 0.3).astype(np.float64)
    dev = torch.device("cuda")
    fg = icnn_b200.PICNN.from_params(p).bind(x)
    xd = torch.tensor(x, dtype=torch.float32, device=dev)
    tYd = torch.tensor(tY, dtype=torch.float64, device=dev)
    st = {}

    def solve():
        st["s"] = be.solveBatch(fg, y0.copy(), nIter=nIter, return_state=True)[-1]

    ms_solve = timeit(solve, reps=3, warm=1)
    s = st["s"]
    ms_k3 = timeit(lambda: argmin_grad.argmin_grad(s, tYd, loss=loss, assemble=True, return_device=True))
    ms_bg = timeit(lambda: bundle_grad(fg, s, tYd, loss=loss, x=xd, return_device=True))
    # the gathered rows, then icnn_train_grad alone
    _cy, _clam, _ct, (fY, fV, fc) = argmin_grad.argmin_grad(s, tY, loss=loss)
    counts = s.count.cpu().numpy()
    Yd, Vd, cd = (torch.tensor(a, dtype=torch.float32, device=dev) for a in (fY, fV, fc))
    prep = _prepare(fg, np.concatenate([[0], np.cumsum(counts)]))
    ms_tg = timeit_events(lambda: _launch(fg, prep, Yd, Vd, cd))
    R = int(counts.sum())
    flops = 2.0 * flop_fg(cfg) * R          # 8 * MAC per row
    peaks = load_peaks()
    achieved = flops / (ms_tg * 1e-3) / 1e12
    gname, power = gpu_info()
    return {"workload": workloads_string(name, cfg), "loss": loss, "rows": R, "gpu": gname, "power_limit_w": power,
            "solveBatch_ms": round(ms_solve, 3), "argmin_grad_k3_ms": round(ms_k3, 3),
            "bundle_grad_ms": round(ms_bg, 3), "train_grad_ms": round(ms_tg, 3),
            "rows_per_s": round(R / (ms_tg * 1e-3), 1), "algorithmic_tflops": round(achieved, 3),
            "frac_of_bf16_peak": round(achieved / peaks["bf16_sustained"], 4),
            "frac_of_3xtf32_ceiling": round(achieved / (peaks["bf16_sustained"] / 6.0), 4),
            "peak_source": peaks["source"]}


def workloads_string(name, cfg):
    return "%s: m=%d n_y=%d hidden=%s batch=%d nIter=%d" % (name, cfg["m"], cfg["n"], cfg["hidden"], cfg["B"],
                                                            cfg["nIter"])


def main():
    args = sys.argv[1:]
    loss = "xent"
    if "--loss" in args:
        i = args.index("--loss")
        loss = args[i + 1]
        del args[i:i + 2]
    for name in args or ["C3", "T"]:
        print(json.dumps(run(name, loss)), flush=True)


if __name__ == "__main__":
    main()
