"""Signed error of the wgmma 3xTF32 GEMM (C = A B^T) vs float64: is the systematic bias a function of the
accumulation LENGTH (then slicing K helps) or intrinsic to every MMA (then it does not)?"""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from icnn_b200 import _capi

torch.manual_seed(0)
dev = torch.device("cuda")
stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)


def gemm(A, B):
    M, K = A.shape
    N = B.shape[0]
    Cc = torch.empty(M, N, device=dev)
    scratch = torch.empty((2 * M + 2 * N) * ((K + 3) & ~3), device=dev)   # split operands, rows padded to 4 floats
    Ac, Bc = A.contiguous(), B.contiguous()      # keep the copies alive across the launch
    _capi.check(_capi.lib.icnn_tc_gemm_selftest(Ac.data_ptr(), Bc.data_ptr(), Cc.data_ptr(), M, N, K,
                                                scratch.data_ptr(), stream))
    torch.cuda.synchronize()
    return Cc


for dist_name in ("uniform(0,1) x uniform(0,1)  (all products positive)", "relu(randn) x |randn|  (PICNN-like)", "randn x randn"):
    for K in (512, 2048, 5120):
        M, N = 256, 256
        if dist_name.startswith("uniform"):
            A, B = torch.rand(M, K, device=dev), torch.rand(N, K, device=dev)
        elif dist_name.startswith("relu"):
            A, B = torch.relu(torch.randn(M, K, device=dev)), torch.randn(N, K, device=dev).abs()
        else:
            A, B = torch.randn(M, K, device=dev), torch.randn(N, K, device=dev)
        ref = A.double() @ B.double().T
        scale = ref.abs().mean()
        one = gemm(A, B).double()
        parts = sum(gemm(A[:, k0:k0 + 640], B[:, k0:k0 + 640]) for k0 in range(0, K, 640)).double() if K > 640 else one
        parts128 = sum(gemm(A[:, k0:k0 + 128], B[:, k0:k0 + 128]) for k0 in range(0, K, 128)).double()
        cub = (A @ B.T).double()
        print("%-52s K=%-5d signed mean err / mean|C|: one launch %+.2e | 640-slices summed in fp32 %+.2e | 128-slices %+.2e | cuBLAS fp32 %+.2e ; max |err| one launch %.2e"
              % (dist_name, K, ((one - ref).mean() / scale).item(), ((parts - ref).mean() / scale).item(),
                 ((parts128 - ref).mean() / scale).item(), ((cub - ref).mean() / scale).item(), ((one - ref).abs().max() / scale).item()), flush=True)
