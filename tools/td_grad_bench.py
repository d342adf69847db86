#!/usr/bin/env python
"""Timing of one RL training step (RL/src/icnn.py:304-323, '--icnn_opt adam') at C4 dims (m 17, n 6, hidden
[200, 200]) for B = 256 (the reference's minibatch, agent.py:9) and B = 65536, one column per component:

  adam_ms            adam.solve on the target network (the argmin act2; includes its host copy of act2)
  td_grad_ms         icnn_b200.td_grad: the target's K1 at act2, icnn_td_grad, the x-path backprop, the L2 term
  lib_ms             the icnn_td_grad library call alone (buffers and workspace allocated beforehand)
  train_grad_v0_ms   what the dedicated entry replaces: a K1 forward of the online network at act (for negQ) plus
                     icnn_train_grad at Y = act, V = 0, one row per sample (its workspace allocated beforehand)
  torch_ms           a lean eager torch float32 autograd arm of loss_q and d loss_q / d theta (TF32 off)

Every shape is warmed up first; the arms alternate within each round and the median over the rounds is reported.
CUDA events around each call, with the device synchronised before the start event.  Prints one JSON line per B,
with the card's name, power limit and SM clock read in the same run.

Usage: python tools/td_grad_bench.py [B ...] [--rounds R]
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
from icnn_b200 import adam  # noqa: E402
from icnn_b200.bundle_grad import _launch as tg_launch, _prepare  # noqa: E402
from icnn_b200.td_grad import _launch as td_launch, td_grad  # noqa: E402
from oracle import td_grad_np as tgn  # noqa: E402


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name()}
    idx = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or "0"
    try:
        out = subprocess.run(["nvidia-smi", "-i", idx, "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10).stdout
        pl, sm, smax = [s.strip() for s in out.strip().split(",")]
        info.update(power_limit_w=float(pl), sm_clock_mhz=float(sm), sm_clock_max_mhz=float(smax))
    except Exception:
        info.update(power_limit_w=None, sm_clock_mhz=None, sm_clock_max_mhz=None)
    return info


def event_ms(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def torch_arm(net, tnet, obs, act, act2, rew, term, discount=0.99, lam=1e-7):
    """loss_q and its gradient by eager float32 autograd: negQ (RL/src/icnn.py:325-404) on leaf copies of the weights."""
    names = ("Wy", "Wz", "Wu", "bu", "Wzu", "bzu", "Wyu", "byu", "Wzx", "bzx")
    P = {k: [None if t is None else t.detach().requires_grad_(True) for t in getattr(net, k)] for k in names}
    L = net.L

    def negq(Q, x, y):
        us, prev = [], x
        for i in range(L):
            u = prev @ Q["Wu"][i] + Q["bu"][i]
            prev = torch.relu(u) if i < L - 1 else u
            us.append(prev)
        z = None
        for i in range(L + 1):
            Pi = x if i == 0 else us[i - 1]
            a = (y * (Pi @ Q["Wyu"][i] + Q["byu"][i])) @ Q["Wy"][i] + Pi @ Q["Wzx"][i] + Q["bzx"][i]
            if i > 0:
                a = a + (z * torch.relu(Pi @ Q["Wzu"][i] + Q["bzu"][i])) @ Q["Wz"][i]
            z = torch.nn.functional.leaky_relu(a, net.alpha) if i < L else a
        return z.reshape(-1)

    def ent(a):
        p = ((a + 1) / 2).clamp(1e-4, 1 - 1e-4)
        return -(p * p.log() + (1 - p) * (1 - p).log()).sum(1)

    with torch.no_grad():
        T = {k: getattr(tnet, k) for k in names}
        qt = -(negq(T, obs, act2) - ent(act2))
    q = -(negq(P, obs, act) - ent(act))
    y = torch.where(term, rew, rew + discount * qt)
    y = torch.minimum(q + 1, torch.maximum(q - 1, y)).detach()
    loss = ((q - y) ** 2).mean()
    leaves = [t for k in names for t in P[k] if t is not None]
    reg = sum((t ** 2).sum() for k in ("Wy", "Wz", "Wu", "Wzu", "Wyu", "Wzx") for t in P[k] if t is not None)
    loss = loss + lam * 0.5 * reg
    return torch.autograd.grad(loss, leaves)


def run(B, rounds):
    p, pt = tgn.make_net("c4", 7), tgn.make_net("c4", 8)
    rs = np.random.RandomState(B)
    obs, ob2 = rs.randn(B, p.m).astype(np.float32), rs.randn(B, p.m).astype(np.float32)
    act = rs.uniform(-1, 1, (B, p.n)).astype(np.float32)
    rew = rs.randn(B).astype(np.float32)
    term = rs.uniform(size=B) < 0.1
    dev = torch.device("cuda")
    net, tnet = icnn_b200.PICNN.from_params(p, device=dev), icnn_b200.PICNN.from_params(pt, device=dev)
    fg, fgt = net.bind(obs), tnet.bind(ob2)
    act2 = adam.solve(fgt).astype(np.float32)
    d = lambda a, dt=torch.float32: torch.as_tensor(a, device=dev).to(dt).contiguous()  # noqa: E731
    obsd, actd, act2d, rewd, termd = d(obs), d(act), d(act2), d(rew), d(term, torch.bool)
    term8 = termd.to(torch.uint8)
    negq_t, _ = fgt.fg_device(act2d)
    _loss, td, _g = td_grad(fg, fgt, obs, act, rew, act2, term, return_device=True)
    c = (-2.0 * td.double() / B).float()
    prep = _prepare(fg, np.arange(B + 1))
    V0 = torch.zeros_like(actd)
    f_on = torch.empty(B, device=dev)
    g_on = torch.empty(B, p.n, device=dev)
    keep = {}

    def lib():
        keep["r"] = td_launch(fg, actd, negq_t, act2d, rewd, term8, 0.99)

    def train_v0():
        fg.fg_device(actd, f_on, g_on)
        tg_launch(fg, prep, actd, V0, c)

    arms = {"adam_ms": lambda: adam.solve(fgt),
            "td_grad_ms": lambda: td_grad(fg, fgt, obsd, actd, rewd, act2d, termd, return_device=True),
            "lib_ms": lib, "train_grad_v0_ms": train_v0,
            "torch_ms": lambda: torch_arm(net, tnet, obsd, actd, act2d, rewd, termd)}
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for fn in arms.values():           # warm-up of every shape
            fn(); fn()
        times = {k: [] for k in arms}
        for _ in range(rounds):
            for k, fn in arms.items():
                times[k].append(event_ms(fn))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    out = {"workload": "C4 dims: m=17 n=6 hidden=[200, 200] B=%d" % B}
    out.update(gpu_info())
    out.update({k: round(float(np.median(v)), 4) for k, v in times.items()})
    out["spread_lib_ms"] = [round(float(min(times["lib_ms"])), 4), round(float(max(times["lib_ms"])), 4)]
    out["spread_train_grad_v0_ms"] = [round(float(min(times["train_grad_v0_ms"])), 4),
                                      round(float(max(times["train_grad_v0_ms"])), 4)]
    return out


def main():
    args = sys.argv[1:]
    rounds = 20
    if "--rounds" in args:
        i = args.index("--rounds")
        rounds = int(args[i + 1])
        del args[i:i + 2]
    for B in [int(a) for a in args] or [256, 65536]:
        print(json.dumps(run(B, rounds)), flush=True)


if __name__ == "__main__":
    main()
