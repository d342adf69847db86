"""K2 alone at a workload (default C5), per outer iteration t, for several builds of the bundle step (exploration
tool, not part of bench.py).

    python tools/k2_profile.py [--workload C5] [--reps 2] [--builds v3,v3off] [--json OUT]

The bundle loop is driven through the per-iteration entries (icnn_bundle_init, icnn_picnn_fg, icnn_bundle_step) as in
bench.py's instrumented pass, and only the K2 launch of each t is timed (CUDA events).  The build is picked by the
environment knobs that bundle_pc.cu reads at every launch, so all builds run in one process on the same inputs.

Per t it prints the ms of the K2 launch for each build, the mean active rows k of a solve, the mean interior-point
iterations, and the modelled row bytes over the time of the first build:
    sum over the samples of passes x k x n x 4,  passes = 2 its + PASSES_OUTSIDE
with its the interior-point steps of a solve: sweep B once per step, sweep A once per step counting the iteration that
only detects convergence but not the seeded iteration 0, and PASSES_OUTSIDE = 2 for the append pass and u0 = G^T z0.
The dependency test's residual pass (skipped when the new row is clearly independent) is not modelled; for the
seed0 build (ICNN_PC_SEED=0, sweep A at it = 0 and the residual pass always) set K2_PASSES_OUTSIDE=4."""
import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

BUILDS = {
    "v3": {},                      # the default at 2048 < n_y <= 4096
    "v3off": {"ICNN_PC_V3": "0"},  # 16-warp four-vector kernel, one sample per SM
    "legacy": {"ICNN_PC_LEGACY": "1"},
    "seed0": {"ICNN_PC_SEED": "0"},  # sweep A at it = 0 and the dependency residual pass always
    "twolog": {"ICNN_PC_TWOLOG": "1"},  # V3 update with two logs per element
    # L2 prefetch distances of the V3 row sweeps, "sweep A trips,sweep B rows" (bundle_pc.cu)
    "pf0": {"ICNN_PC_PREFETCH": "0,0"},
    "pfa1": {"ICNN_PC_PREFETCH": "1,0"},
    "pfa2": {"ICNN_PC_PREFETCH": "2,0"},
    "pfb8": {"ICNN_PC_PREFETCH": "0,8"},
    "pfb16": {"ICNN_PC_PREFETCH": "0,16"},
    "pfa1b8": {"ICNN_PC_PREFETCH": "1,8"},
    "pfa2b16": {"ICNN_PC_PREFETCH": "2,16"},
}
KNOBS = sorted({k for e in BUILDS.values() for k in e})
PASSES_OUTSIDE = int(os.environ.get("K2_PASSES_OUTSIDE", "2"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C5")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--builds", default="v3,v3off")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import icnn_b200
    from icnn_b200 import _capi, bundle_entropy, workloads

    builds = a.builds.split(",")
    cfg = workloads.CONFIGS[a.workload]
    p, x, y0 = workloads.make_inputs(a.workload)
    B, n, nIter = x.shape[0], cfg["n"], cfg["nIter"]
    dev = torch.device("cuda")
    net = icnn_b200.PICNN.from_params(p, device=dev)
    fg = net.bind(torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(dev), affine=cfg["affine"])
    KS = (nIter if cfg["variant"] == "rl" else min(nIter, n)) + 1
    ccfg = bundle_entropy._make_cfg(cfg["variant"], "pc", nIter, None, None, 0, n, KS)
    for k in KNOBS:
        os.environ.pop(k, None)
    st = bundle_entropy.BundleState(B, n, KS, dev, keep_xs=True, nIter=nIter, stats=True)
    stats_ptr = st.c.iter_stats
    y0d = torch.from_numpy(y0).to(dev)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def run(env, stats):
        for k in KNOBS:
            os.environ.pop(k, None)
        os.environ.update(env)
        st.c.iter_stats = stats_ptr if stats else None
        if stats:
            st.iter_stats.zero_()
        st.y.copy_(y0d)
        _capi.check(_capi.lib.icnn_bundle_init(C.byref(st.c), nIter, stream))
        evs = []
        for t in range(nIter):
            _capi.check(_capi.lib.icnn_picnn_fg(net._h, C.byref(fg.c_gates), st.y32.data_ptr(), st.f.data_ptr(),
                                                st.G.data_ptr(), 0, st.perm.data_ptr(), st.count.data_ptr(), KS,
                                                fg.ws.data_ptr(), None, stream))
            e1, e2 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e1.record()
            _capi.check(_capi.lib.icnn_bundle_step(C.byref(ccfg), C.byref(st.c), t, stream))
            e2.record()
            evs.append((e1, e2))
        torch.cuda.synchronize()
        for k in env:
            os.environ.pop(k, None)
        return np.array([e1.elapsed_time(e2) for e1, e2 in evs])

    run({}, True)    # warm-up + statistics of the default build
    s = st.iter_stats.cpu().numpy()
    solves = np.maximum(s[:, 0] - s[:, 5], 1)
    mean_k = s[:, 1] / solves
    mean_its = s[:, 2] / solves
    row_bytes = 4.0 * n * (2.0 * s[:, 4] + PASSES_OUTSIDE * s[:, 1])
    ms = {}
    for b in builds:
        run(BUILDS[b], False)   # warm-up of this build's module / attributes
        ms[b] = np.mean([run(BUILDS[b], False) for _ in range(a.reps)], axis=0)
    props = torch.cuda.get_device_properties(dev)
    print("%s on %s: B=%d n=%d nIter=%d, K2 ms per launch (mean of %d runs), passes outside the IPM loop in the byte "
          "model = %d" % (a.workload, props.name, B, n, nIter, a.reps, PASSES_OUTSIDE))
    print("  t   active  mean_k  its  " + "  ".join("%9s" % b for b in builds) + "   GB(model)  GB/s(%s)" % builds[0])
    for t in range(nIter):
        print("%3d  %7d  %6.2f  %4.1f  " % (t, s[t, 0], mean_k[t], mean_its[t]) +
              "  ".join("%9.3f" % ms[b][t] for b in builds) +
              "   %9.2f  %8.0f" % (row_bytes[t] / 1e9, row_bytes[t] / 1e9 / max(ms[builds[0]][t] * 1e-3, 1e-9)))
    print("sum  " + " " * 24 + "  ".join("%9.1f" % ms[b].sum() for b in builds) + "   %9.1f" % (row_bytes.sum() / 1e9))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump({"device": props.name, "workload": a.workload, "mean_k": mean_k.tolist(), "mean_its": mean_its.tolist(),
                       "row_bytes_model": row_bytes.tolist(), "ms": {b: v.tolist() for b, v in ms.items()}}, f)


if __name__ == "__main__":
    main()
