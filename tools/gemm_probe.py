"""Throughput of nmb_tr_gemm (hand-written SGEMM of the training path) vs torch.matmul (cuBLAS fp32)."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import torch
from neumesh_b200 import train_ops
dev = torch.device("cuda:0")
P = train_ops.CudaPrims(dev)
torch.backends.cuda.matmul.allow_tf32 = False
def timeit(fn, n=10):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n
M = 130560
for (name, m, n, k, akc, bkc) in [("forward  X[M,256] . W[256,256]^T", M, 256, 256, True, True),
                                  ("forward  X[M,177] . W[256,177]^T", M, 256, 177, True, True),
                                  ("bwd data dZ[M,256] . W[256,256]", M, 256, 256, True, False),
                                  ("bwd wgt  dZ^T[256,M] . X[M,256]", 256, 256, M, False, False)]:
    if name.startswith("bwd wgt"):
        A = torch.randn(M, 256, device=dev); B = torch.randn(M, 256, device=dev); C = torch.empty(256, 256, device=dev)
        f1 = lambda: P.gemm(A, 256, False, B, 256, False, C, 256, 256, 256, M)
        f2 = lambda: torch.matmul(A.t(), B)
    elif akc and bkc:
        A = torch.randn(m, k, device=dev); B = torch.randn(n, k, device=dev); C = torch.empty(m, n, device=dev)
        f1 = lambda: P.gemm(A, k, True, B, k, True, C, n, m, n, k)
        f2 = lambda: torch.matmul(A, B.t())
    else:
        A = torch.randn(m, k, device=dev); B = torch.randn(k, n, device=dev); C = torch.empty(m, n, device=dev)
        f1 = lambda: P.gemm(A, k, True, B, n, False, C, n, m, n, k)
        f2 = lambda: torch.matmul(A, B)
    t1, t2 = timeit(f1), timeit(f2)
    fl = 2.0 * m * n * k
    print(f"{name:36s}: nmb_tr_gemm {t1:7.3f} ms ({fl / t1 / 1e9:6.1f} TFLOP/s)   cuBLAS fp32 {t2:7.3f} ms ({fl / t2 / 1e9:6.1f} TFLOP/s)")
