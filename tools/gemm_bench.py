"""Time r2d2_gemm_f32 on the learner's shapes (dev tool): us and fp32-equivalent TFLOP/s, wgmma vs mma.sync."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200")]
import torch
from r2d2_b200 import native as nv
lib = nv.lib()
SHAPES = [  # layout, M, N, K, split, label
    (0, 32000, 1024, 256, 1, "z*Wih^T (NT)"),
    (0, 32000, 256, 17, 1, "obs*W1^T (NT, K=17)"),
    (0, 20480, 6, 256, 1, "head (NT, N=6)"),
    (1, 30720, 256, 1024, 1, "dgin*Wih (NN)"),
    (2, 1024, 256, 30720, 0, "dWhh (TN, split-K)"),
    (2, 256, 17, 30720, 0, "dW1 (TN, N=17)"),
    (0, 8192, 8192, 1024, 1, "square-ish 8192x8192x1024"),
]
def run(layout, M, N, K, split):
    if layout == 0: A, B = torch.randn(M, K, device="cuda"), torch.randn(N, K, device="cuda"); lda, ldb = K, K
    elif layout == 1: A, B = torch.randn(M, K, device="cuda"), torch.randn(K, N, device="cuda"); lda, ldb = K, N
    else: A, B = torch.randn(K, M, device="cuda"), torch.randn(K, N, device="cuda"); lda, ldb = M, N
    C = torch.zeros(M, N, device="cuda")
    def call():
        nv.check(lib.r2d2_gemm_f32(layout, M, N, K, nv.dptr(A), lda, nv.dptr(B), ldb, None, 0, None, 0, 0, nv.dptr(C), N,
                                   None, None, 0, 0, split, nv.current_stream()))
    for _ in range(3): call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10): call()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 10 * 1e3
for layout, M, N, K, split, label in SHAPES:
    res = []
    for impl in (1, 0):
        lib.r2d2_set_gemm_impl(impl)
        sk = split if split else (max(1, min(64, (K // 32) // 8)))
        us = run(layout, M, N, K, sk)
        res.append(f"{'tc ' if impl else 'mma'} {us:8.1f} us {2.0 * M * N * K / us / 1e6:7.1f} TF/s")
    print(f"{label:28s} M={M:6d} N={N:5d} K={K:6d} | " + " | ".join(res))
lib.r2d2_set_gemm_impl(1)
