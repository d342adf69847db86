"""wgmma / TMA 3xTF32 GEMM self test: C = A B^T vs float64, several shapes."""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from icnn_b200 import _capi

torch.manual_seed(0)
dev = torch.device("cuda")
stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
shapes = [(128, 64, 32), (128, 128, 64), (256, 192, 96), (400, 512, 2048), (77, 40, 8), (4096, 1024, 1536), (130, 600, 612)]
if len(sys.argv) > 1:
    shapes = [tuple(int(v) for v in a.split("x")) for a in sys.argv[1:]]
for (M, N, K) in shapes:
    A = torch.randn(M, K, device=dev)
    B = torch.randn(N, K, device=dev)
    Cc = torch.full((M, N), float("nan"), device=dev)
    scratch = torch.empty((2 * M + 2 * N) * ((K + 3) & ~3), device=dev)   # split operands, rows padded to 4 floats
    _capi.check(_capi.lib.icnn_tc_gemm_selftest(A.data_ptr(), B.data_ptr(), Cc.data_ptr(), M, N, K, scratch.data_ptr(), stream))
    torch.cuda.synchronize()
    ref = A.double() @ B.double().T
    err = (Cc.double() - ref).abs().max().item() / ref.abs().max().item()
    tf = (A @ B.T)
    err32 = (tf.double() - ref).abs().max().item() / ref.abs().max().item()
    # timing
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        _capi.lib.icnn_tc_gemm_selftest(A.data_ptr(), B.data_ptr(), Cc.data_ptr(), M, N, K, scratch.data_ptr(), stream)
    e0.record()
    for _ in range(10):
        _capi.lib.icnn_tc_gemm_selftest(A.data_ptr(), B.data_ptr(), Cc.data_ptr(), M, N, K, scratch.data_ptr(), stream)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    print("M=%d N=%d K=%d  rel err 3xTF32 %.2e (cuBLAS fp32 %.2e)  nan %d  %.3f ms  %.1f TFLOP/s (incl. split kernels)" % (
        M, N, K, err, err32, int(torch.isnan(Cc).sum()), ms, 2.0 * M * N * K / ms / 1e9), flush=True)
