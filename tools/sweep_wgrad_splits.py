"""Sweep split-K factors of the wgrad GEMMs (both operands MN-major, fp32 atomics) at cfg-2 shapes."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from transformerscandobayesianinference_b200 import _lib as L
dev = torch.device("cuda:0"); N = 512000
def t(fn, reps=10):
    for _ in range(2): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps
for (M, Nn, name) in [(1536, 512, "qkv"), (1024, 512, "mlp1"), (512, 1024, "mlp2"), (512, 512, "out")]:
    A = torch.randn(N, M, device=dev).to(torch.bfloat16); Bm = torch.randn(N, Nn, device=dev).to(torch.bfloat16)
    C = torch.zeros(M, Nn, device=dev)
    res = []
    for ks in (2, 3, 4, 5, 6, 8, 9, 11, 12, 16, 18, 24, 33, 37, 74):
        ms = t(lambda: L.gemm(A, Bm, C, a_mn_major=True, b_mn_major=True, M=M, N=Nn, K=N, accumulate=True, k_splits=ks, use_tc=True))
        res.append(f"{ks}:{ms:.3f}")
    print(f"{name} wgrad {M}x{Nn}: " + "  ".join(res), flush=True)
