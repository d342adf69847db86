"""Small end-to-end cases for compute-sanitizer (memcheck / racecheck / synccheck):
    compute-sanitizer --tool racecheck python tools/sanitize_case.py
Covers K1 FFMA + cluster split-K, K1 wgmma path, K2 five-sweep group kernel (1 / 2 / 8 warps per sample, PC + dual +
RL Newton), every build of the K2 two-sweep PC kernel the dispatch selects, k > 32 bundles and the cluster variant, K2 thread-per-sample kernel, K3, Adam, x-path gates, unaligned widths on the wgmma path (pitch-padded
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

which = sys.argv[1:] or ["c1", "c3", "c3dual", "c4", "c2", "t", "k3", "adam", "odd", "gdgrad", "pc", "k2builds"]
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
if "pc" in which:     # the two-sweep PC kernel in every build bundle_pc.cu selects, both alignments, the > 4 row-block sweeps
    def pc_shape(n, B, nIter):
        p = workloads.synth_params(5, 16, n, [32, 32])
        x = np.random.RandomState(3).randn(B, 16)
        out = be.solveBatch(icnn_b200.PICNN.from_params(p).bind(x), np.full((B, n), 0.5), nIter=nIter)
        print("pc n_y", n, B, nIter, "ok, y range", float(out[0].min()), float(out[0].max()), flush=True)
    pc_shape(100, 5, 5)                                 # 1 warp / sample, 1 chunk
    pc_shape(90, 5, 5)                                  # the same with n_y % 4 != 0 (scalar row loads)
    pc_shape(200, 5, 5)                                 # 1 warp / sample, 2 chunks
    run("C3", 5, 5)                                     # the same with n_y % 4 != 0
    run("C3", 2, 36)                                    # k + 2 > 32 sweep rows: second triangle + rectangle sweeps
    run("C2", 2, 4)                                     # 8 warps / sample (n_y = 2048)
    run("C5", 2, 6)                                     # three-vector build, 8 warps / sample (n_y = 4096)
    run("C5", 2, 56)                                    # 16 warps / sample, 2 chunks: KS too large for two samples per SM
    pc_shape(5000, 2, 4)                                # 16 warps / sample, 4 chunks
    _, _, o = run("C3", 4, 4, stats=True)
    print("stats", o[-1].stats()["entering"], flush=True)
if "k2builds" in which:   # k > 32 in a two-sweep and a five-sweep build, the cluster variant, dual at 16 warps
    def orthogonal(n, B, P=64):   # one well-separated row per iteration (tests/test_gpu_k2_builds.py)
        rs = np.random.RandomState(0)
        P = min(P, n)
        A = np.zeros((B, P, n))
        for u in range(B):
            A[u, np.arange(P), rs.choice(n, P, replace=False)] = 8.0
        w = rs.randn(n)
        A = (A + rs.randn(B, P, n) * 0.05 / np.sqrt(n) + 2.0 * w / np.linalg.norm(w)).astype(np.float32).astype(np.float64)
        b = (0.1 * rs.randn(B, P)).astype(np.float32).astype(np.float64)
        def fg(y):
            v = np.einsum("bmn,bn->bm", A, y) + b
            i = v.argmax(1)
            return v[np.arange(B), i].astype(np.float32).astype(np.float64), A[np.arange(B), i].copy()
        return fg
    for n, nIter, variant, env in ((100, 45, "lib", {}), (100, 62, "lib", {}), (2048, 12, "dual", {"ICNN_K2_CS": "4"}),
                                   (4096, 40, "dual", {})):
        os.environ.update(env)
        out = be.solveBatch(orthogonal(n, 2), np.full((2, n), 0.5), nIter=nIter, variant=variant)
        for k in env: os.environ.pop(k)
        print("k2builds n_y", n, nIter, variant, env, "k", [len(g) for g in out[1]], flush=True)
print("done")
