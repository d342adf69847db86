"""Per-iteration CUDA-event timing of K1 / K2 on a workload (exploration tool, not a test)."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import icnn_b200
from icnn_b200 import _capi, bundle_entropy, workloads

name = sys.argv[1] if len(sys.argv) > 1 else "C2"
solver = sys.argv[2] if len(sys.argv) > 2 else "pc"
Bover = int(sys.argv[3]) if len(sys.argv) > 3 else None
cfg = workloads.CONFIGS[name]
p, x, y0 = workloads.make_inputs(name, B=Bover)
B, n, nIter = x.shape[0], cfg["n"], cfg["nIter"]
dev = torch.device("cuda")
net = icnn_b200.PICNN.from_params(p)
fg = net.bind(x, affine=cfg["affine"])
variant = cfg["variant"]
KS = (nIter if variant == "rl" else min(nIter, n)) + 1
ccfg = bundle_entropy._make_cfg(variant, solver, nIter, None, None, 0, n, KS)
st = bundle_entropy.BundleState(B, n, KS, dev, keep_xs=True, nIter=nIter)
y0d = torch.from_numpy(y0).to(dev)
stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
for rep in range(2):
    st.y.copy_(y0d)
    _capi.check(_capi.lib.icnn_bundle_init(C.byref(st.c), nIter, stream))
    evs, stats = [], []
    for t in range(nIter):
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        _capi.check(_capi.lib.icnn_picnn_fg(net._h, C.byref(fg.c_gates), st.y32.data_ptr(), st.f.data_ptr(), st.G.data_ptr(), 0,
                                            st.perm.data_ptr(), st.count.data_ptr(), KS, fg.ws.data_ptr(), None, stream))
        e1.record()
        _capi.check(_capi.lib.icnn_bundle_step(C.byref(ccfg), C.byref(st.c), t, stream))
        e2.record()
        evs.append((e0, e1, e2))
        if rep:
            torch.cuda.synchronize()
            cnt = st.count.cpu().numpy(); fin = st.finished.cpu().numpy(); ni = int(st.newton_its.cpu().numpy().sum())
            stats.append((cnt.mean(), cnt.max(), int((fin == 0).sum()), ni - (stats[-1][4] if stats else 0), ni))
    torch.cuda.synchronize()
print("%s B=%d n=%d nIter=%d solver=%s WPS=%s" % (name, B, n, nIter, solver, os.environ.get("ICNN_K2_WPS", "auto")))
k1 = [a.elapsed_time(b) for a, b, _ in evs]; k2 = [b.elapsed_time(c) for _, b, c in evs]
for t in range(nIter):
    if t < 6 or t % 5 == 4 or t == nIter - 1:
        print("  t=%2d  K1 %.3f ms  K2 %.3f ms   k mean %.1f max %d  active %d  inner its/sample %.1f" % (t, k1[t], k2[t], stats[t][0], stats[t][1], stats[t][2], stats[t][3] / max(1, (stats[t - 1][2] if t else B))))
print("  total K1 %.2f ms  K2 %.2f ms" % (sum(k1), sum(k2)))
