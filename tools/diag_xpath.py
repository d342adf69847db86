import os, sys; sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, icnn_b200
from oracle import picnn_np, synth
for B in (5, 40, 64, 130):
    p,x,y0 = synth.make_inputs("C5",B=B)
    net = icnn_b200.PICNN.from_params(p)
    y = np.random.RandomState(11).uniform(0.02,0.98,size=y0.shape).astype(np.float32).astype(np.float64)
    fo,go = picnn_np.make_fg(p,x)(y)
    ocz,ocy,od = picnn_np.gates(p,x)
    for xp in (True, False):
        net._xpath = xp and True
        fg = net.bind(x)
        f,g = fg(y)
        gerr = max(np.abs(fg.cy[i].cpu().numpy()-ocy[i]).max()/np.abs(ocy[i]).max() for i in range(p.L+1))
        derr = max(np.abs(fg.d[i].cpu().numpy()-od[i]).max()/max(1,np.abs(od[i]).max()) for i in range(p.L+1))
        print("B=%d xpath=%s  f relerr %.2e  g relerr %.2e  cy relerr %.2e d relerr %.2e"%(B,xp,np.abs(f-fo).max()/np.abs(fo).max(), np.abs(g-go).max()/np.abs(go).max(), gerr, derr))
