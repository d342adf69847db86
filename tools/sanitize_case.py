"""Small end-to-end cases for compute-sanitizer (memcheck / racecheck / synccheck):
    compute-sanitizer --tool racecheck python tools/sanitize_case.py
Covers K1 FFMA + cluster split-K, K1 wgmma path, K2 group kernel (WPS 1/2/8, PC + dual + RL Newton),
K2 thread-per-sample kernel, K3, Adam, x-path gates, unaligned widths on the wgmma path (pitch-padded
operands), GD training backward (FFMA and wgmma GDB instantiation, split-K weight-gradient GEMM)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import icnn_b200
from icnn_b200 import bundle_entropy as be, workloads

def run(name, B, nIter, variant=None, **kw):
    cfg = workloads.CONFIGS[name]
    p, x, y0 = workloads.make_inputs(name, B=B)
    net = icnn_b200.PICNN.from_params(p)
    fg = net.bind(x, affine=cfg["affine"])
    out = be.solveBatch(fg, y0.copy(), nIter=nIter, variant=variant or cfg["variant"], return_state=True, **kw)
    print(name, B, nIter, variant or cfg["variant"], "ok, y range", float(out[0].min()), float(out[0].max()), flush=True)
    return net, fg, out

which = sys.argv[1:] or ["c1", "c3", "c3dual", "c4", "c2", "t", "k3", "adam", "odd", "gdgrad", "pc"]
if "c1" in which: run("C1", 16, 4)
if "c3" in which: run("C3", 6, 4)
if "c3dual" in which: run("C3", 6, 4, variant="dual")
if "c4" in which:
    run("C4", 40, 4)
    os.environ["ICNN_K2_SMALL"] = "0"; run("C4", 16, 3); os.environ.pop("ICNN_K2_SMALL")
if "c2" in which: run("C2", 2, 4)
if "t" in which: run("T", 64, 2)
if "k3" in which:
    net, fg, out = run("C3", 6, 4)
    tY = (np.random.RandomState(0).uniform(size=out[0].shape) < 0.3).astype(np.float64)
    icnn_b200.argmin_grad.argmin_grad(out[-1], tY, loss="xent"); print("k3 ok", flush=True)
if "adam" in which:
    p, x, _ = workloads.make_inputs("C4", B=8)
    a, its = icnn_b200.adam.solve(icnn_b200.PICNN.from_params(p).bind(x), max_iter=24, return_iters=True); print("adam ok", its, flush=True)
if "odd" in which:      # widths that are not multiples of 4 on the tensor-core path (B >= 64)
    p = workloads.synth_params(3, 13, 37, [50, 21, 33])
    x = np.random.RandomState(1).randn(70, 13)
    net = icnn_b200.PICNN.from_params(p)
    assert net._xpath
    out = be.solveBatch(net.bind(x), np.full((70, 37), 0.5), nIter=3); print("odd ok", float(out[0].mean()), flush=True)
if "gdgrad" in which:
    for dims, B in (((12, 37, [50, 21, 33]), 40), ((12, 37, [50, 21, 33]), 70), ((24, 64, [320, 96]), 130)):
        p = workloads.synth_params(4, *dims)
        rs = np.random.RandomState(2)
        x = rs.randn(B, dims[0]); tY = (rs.uniform(size=(B, dims[1])) < 0.2).astype(np.float64)
        yN, gr = icnn_b200.gd_grad.gd_grad(icnn_b200.PICNN.from_params(p).bind(x), np.full((B, dims[1]), 0.5), tY,
                                           nIter=3, lr=0.02, momentum=0.5, x=x)
        print("gdgrad ok", dims, B, float(np.abs(gr["Wy"][0]).max()), flush=True)
if "pc" in which:     # round 2: the two-sweep PC kernel in every group size, both alignments, the > 4 row-block sweeps, and
    # the chunked-accumulation wgmma GEMM (T, 64 rows above)
    run("C3", 5, 5)                                     # 1 warp / sample, n_y % 4 != 0 (scalar row loads)
    for w in ("1", "2", "4", "8"):
        os.environ["ICNN_PC_WPS"] = w
        run("T", 3, 4)                                  # n_y = 512 on 1 / 2 / 4 / 8 warps per sample
    os.environ["ICNN_PC_WPS"] = "2"
    run("T", 2, 36)                                     # k + 2 > 32 sweep rows: second triangle + rectangle sweeps
    os.environ.pop("ICNN_PC_WPS")
    run("C5", 2, 6)                                     # 16 warps / sample (n_y = 4096)
    _, _, o = run("C3", 4, 4, stats=True)
    print("stats", o[-1].stats()["entering"], flush=True)
print("done")
