"""Where the cycles of the V3 two-sweep K2 kernel go, per phase and per outer iteration t (exploration tool, not part
of bench.py).

    python tools/k2_phases.py [--workload C5] [--json OUT] [--csrc DIR] [--build-only]

It compiles tools/k2_phases.cu, the V3 kernel of bundle_pc_kernel.cuh with ICNN_PC_PHASES, into a shared object of its
own under build/k2_phases/ (never into the library), and drives the bundle loop through the per-iteration entries
(icnn_bundle_init, icnn_picnn_fg) as tools/k2_profile.py does, with that build as the K2 launch of every t.  Thread 0
of each CTA reads clock64 at the end of each phase (bundle_pc_kernel.cuh, PcPhase); a phase that ends at a barrier
includes the wait for the slowest warp, so the phases add up to the CTA's time.  One warm-up solve, then one measured
solve.  Per t it prints the cycles per phase summed over the samples (G = 1e9), their total, the mean active rows k
and the mean interior-point iterations per solve.

--csrc DIR compiles the kernel from another copy of icnn_b200/csrc (for example the parent commit's, with the phase
marks added) so that two versions can be compared phase by phase.  The workload must be one where the dispatch picks
the V3 build (2048 < n_y <= 4096); the tool checks that with icnn_k2_plan."""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ["append", "seed", "u0", "sweepA", "kxk", "sweepB", "sigma", "dir2", "update", "commit"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def build(csrc):
    src = os.path.join(ROOT, "tools", "k2_phases.cu")
    deps = [src] + sorted(os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h")))
    deps.append(os.path.join(csrc, "..", "..", "include", "icnn_b200.h"))
    h = hashlib.sha1()
    for d in deps:   # named by the sources' contents: a copy of the tree reuses the object built from the same sources
        with open(d, "rb") as f:
            h.update(f.read())
    out = os.path.join(ROOT, "build", "k2_phases", "libk2phases_%s.so" % h.hexdigest()[:12])
    if os.path.exists(out):
        return out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
           "-Xptxas", "-v", "-shared", "-I", csrc, src, "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stderr)
        raise SystemExit("k2_phases: compile failed")
    spill = [ln.strip() for ln in r.stderr.splitlines() if "spill" in ln]
    print("k2_phases: built %s (%s)" % (out, spill[0] if spill else "no spill line"))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C5")
    ap.add_argument("--csrc", default=os.path.join(ROOT, "icnn_b200", "csrc"))
    ap.add_argument("--pf", default="1,8", help="prefetch distances 'sweep A trips,sweep B rows' (library default 1,8)")
    ap.add_argument("--json", default=None)
    ap.add_argument("--build-only", action="store_true")
    a = ap.parse_args()
    so = build(os.path.abspath(a.csrc))
    if a.build_only:
        return
    import numpy as np
    import torch
    import icnn_b200
    from icnn_b200 import _capi, bundle_entropy, workloads

    ph_lib = C.CDLL(so)
    ph_lib.k2ph_launch.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    nph, slots = ph_lib.k2ph_nph(), ph_lib.k2ph_slots()
    assert nph == len(PHASES), (nph, PHASES)
    pfa, pfb = (int(v) for v in a.pf.split(","))

    cfg = workloads.CONFIGS[a.workload]
    p, x, y0 = workloads.make_inputs(a.workload)
    B, n, nIter = x.shape[0], cfg["n"], cfg["nIter"]
    KS = (nIter if cfg["variant"] == "rl" else min(nIter, n)) + 1
    plan = (C.c_int32 * _capi.K2_PLAN_LEN)()
    ccfg = bundle_entropy._make_cfg(cfg["variant"], "pc", nIter, None, None, 0, n, KS)
    _capi.check(_capi.lib.icnn_k2_plan(n, KS, ccfg.solver, ccfg.variant, plan))
    dev = torch.device("cuda")
    net = icnn_b200.PICNN.from_params(p, device=dev)
    fg = net.bind(torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(dev), affine=cfg["affine"])
    st = bundle_entropy.BundleState(B, n, KS, dev, keep_xs=True, nIter=nIter, stats=True)
    y0d = torch.from_numpy(y0).to(dev)
    ph = torch.zeros(nIter * nph * slots, dtype=torch.int64, device=dev)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def run():
        st.iter_stats.zero_()
        ph.zero_()
        st.y.copy_(y0d)
        _capi.check(_capi.lib.icnn_bundle_init(C.byref(st.c), nIter, stream))
        for t in range(nIter):
            _capi.check(_capi.lib.icnn_picnn_fg(net._h, C.byref(fg.c_gates), st.y32.data_ptr(), st.f.data_ptr(),
                                                st.G.data_ptr(), 0, st.perm.data_ptr(), st.count.data_ptr(), KS,
                                                fg.ws.data_ptr(), None, stream))
            rc = ph_lib.k2ph_launch(C.byref(ccfg), C.byref(st.c), t, C.c_void_p(ph.data_ptr()), pfa, pfb, stream)
            if rc != 0:
                raise SystemExit("k2ph_launch: CUDA error %d" % rc)
        torch.cuda.synchronize()

    run()   # warm-up
    run()
    s = st.iter_stats.cpu().numpy()
    cyc = ph.cpu().numpy().view(np.uint64).astype(np.float64).reshape(nIter, nph, slots).sum(axis=2)
    solves = np.maximum(s[:, 0] - s[:, 5], 1)
    mean_k, mean_its = s[:, 1] / solves, s[:, 2] / solves
    props = torch.cuda.get_device_properties(dev)
    print("%s on %s: B=%d n=%d nIter=%d, K2 plan %s; V3 phase-timer build, cycles summed over the samples (G = 1e9)"
          % (a.workload, props.name, B, n, nIter, list(plan)))
    print("  t  active  mean_k   its  " + " ".join("%7s" % h for h in PHASES) + "    total")
    for t in range(nIter):
        print("%3d  %6d  %6.2f  %4.1f  " % (t, s[t, 0], mean_k[t], mean_its[t]) +
              " ".join("%7.3f" % (v / 1e9) for v in cyc[t]) + "  %7.2f" % (cyc[t].sum() / 1e9))
    tot = cyc.sum(axis=0)
    print("sum" + " " * 24 + " ".join("%7.2f" % (v / 1e9) for v in tot) + "  %7.1f" % (tot.sum() / 1e9))
    print("share" + " " * 22 + " ".join("%6.1f%%" % (100 * v / tot.sum()) for v in tot))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump({"device": props.name, "workload": a.workload, "phases": PHASES, "mean_k": mean_k.tolist(),
                       "mean_its": mean_its.tolist(), "cycles": cyc.tolist()}, f)


if __name__ == "__main__":
    main()
