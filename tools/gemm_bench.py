"""Time r2d2_gemm_f32 on the learner's wgmma shapes (dev tool, needs a GPU).

For every cfg-3 and cfg-2 product that takes the wgmma path it prints
  - the whole call (operand packing, GEMM, split-K sum) in us, from CUDA events around 20 calls,
  - the gemm_packed_kernel alone in us, from torch.profiler over 20 calls of its own,
  - algorithmic TFLOP/s (2 M N K over the kernel time) and bf16-MMA TFLOP/s (3 passes: x3), each also as a fraction of
    the 989 TFLOP/s dense-BF16 data-sheet rate of the H100 SXM,
  - the L2 -> SM operand feed the kernel needs (32 KB of tile images per 128 x 128 x 32 k tile), computed from the
    shape over the kernel time.
The card name, power limit and SM clock are printed first.

  python tools/gemm_bench.py [OUT_DIR]      # OUT_DIR/gemm_bench.json as well
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "pytorch-r2d2-dpg_b200")]
import ctypes  # noqa: E402

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from r2d2_b200 import native as nv  # noqa: E402

PEAK_BF16 = 989e12   # dense BF16, H100 SXM data sheet (700 W)
NT, NN, TN = 0, 1, 2
SHAPES = [  # label, layout, M, N, K   (split-K as the learner picks it: gemm_tc_suggest_split_k)
    ("cfg3 gin T*B=64000", NT, 64000, 2048, 512),
    ("cfg3 gin T*B=61440", NT, 61440, 2048, 512),
    ("cfg3 gin T*B=40960", NT, 40960, 2048, 512),
    ("cfg3 l1 actor", NT, 64000, 512, 376),
    ("cfg3 l1 critic", NT, 64000, 512, 393),
    ("cfg3 dW_hh S*B=61440", TN, 2048, 512, 61440),
    ("cfg3 dW_hh S*B=81920", TN, 2048, 512, 81920),
    ("cfg3 dW_ih T*B=61440", TN, 2048, 512, 61440),
    ("cfg3 dW_ih T*B=40960", TN, 2048, 512, 40960),
    ("cfg3 dgin T*B=61440", NN, 61440, 512, 2048),
    ("cfg3 dgin T*B=40960", NN, 40960, 512, 2048),
    ("cfg3 dW1 T*B=61440", TN, 512, 376, 61440),
    ("cfg3 dW1 T*B=40960", TN, 512, 376, 40960),
    ("cfg2 gin T*B=32000", NT, 32000, 1024, 256),
    ("cfg2 gin T*B=30720", NT, 30720, 1024, 256),
    ("cfg2 gin T*B=20480", NT, 20480, 1024, 256),
    ("cfg2 dW_hh S*B=30720", TN, 1024, 256, 30720),
    ("cfg2 dW_hh S*B=40960", TN, 1024, 256, 40960),
    ("cfg2 dW_ih T*B=20480", TN, 1024, 256, 20480),
    ("cfg2 dgin T*B=30720", NN, 30720, 256, 1024),
    ("cfg2 dgin T*B=20480", NN, 20480, 256, 1024),
]


def cdiv(a, b):
    return -(-a // b)


def suggest_split_k(M, N, K, sms):
    """gemm_tc.cu gemm_tc_suggest_split_k"""
    tiles, k_tiles = cdiv(M, 128) * cdiv(N, 128), cdiv(K, 32)
    if tiles >= sms or k_tiles < 16:
        return 1
    return max(1, min(cdiv(2 * sms, tiles), k_tiles // 8, 256))


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), (v.strip() for v in out.split(","))))
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name()}


def bench(lib, layout, M, N, K, split, reps=20):
    shape_a = (K, M) if layout == TN else (M, K)
    shape_b = (N, K) if layout == NT else (K, N)
    A, B = torch.randn(shape_a, device="cuda"), torch.randn(shape_b, device="cuda")
    C = torch.empty(M, N, device="cuda")

    def call():
        nv.check(lib.r2d2_gemm_f32(layout, M, N, K, nv.dptr(A), shape_a[1], nv.dptr(B), shape_b[1], None, 0, None, 0, 0,
                                   nv.dptr(C), N, None, None, 0, 0, split, nv.current_stream()))
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    call_us = e0.elapsed_time(e1) / reps * 1e3
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
    kern_us = sum(float(getattr(ev, "self_device_time_total", 0.0) or getattr(ev, "self_cuda_time_total", 0.0))
                  for ev in prof.key_averages() if "gemm_packed_kernel" in ev.key) / reps
    return call_us, kern_us


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else None
    lib = nv.lib()
    lib.r2d2_set_gemm_impl(1)
    sms = ctypes.c_int(0)
    nv.check(lib.r2d2_device_sm_count(ctypes.byref(sms)))
    info = gpu_info()
    print(f"{info.get('name')}  power limit {info.get('power.limit', '?')}  SM clock {info.get('clocks.sm', '?')} "
          f"(max {info.get('clocks.max.sm', '?')})  {sms.value} SMs")
    print(f"{'product':22s} {'M':>6s} {'N':>5s} {'K':>6s} {'split':>5s} | {'call us':>8s} {'kernel us':>9s} | "
          f"{'alg TF/s':>8s} {'of peak':>7s} | {'MMA TF/s':>8s} {'of peak':>7s} | {'L2->SM TB/s':>11s}")
    rows = []
    for label, layout, M, N, K in SHAPES:
        split = suggest_split_k(M, N, K, sms.value) if layout == TN else 1
        call_us, kern_us = bench(lib, layout, M, N, K, split)
        alg = 2.0 * M * N * K / (kern_us * 1e-6)
        feed = cdiv(M, 128) * cdiv(N, 128) * cdiv(K, 32) * 32768 / (kern_us * 1e-6)
        rows.append(dict(product=label, layout=layout, M=M, N=N, K=K, split_k=split, call_us=call_us,
                         kernel_us=kern_us, alg_tflops=alg / 1e12, alg_of_peak=alg / PEAK_BF16,
                         mma_tflops=3 * alg / 1e12, mma_of_peak=3 * alg / PEAK_BF16, l2_feed_tbs=feed / 1e12))
        print(f"{label:22s} {M:6d} {N:5d} {K:6d} {split:5d} | {call_us:8.1f} {kern_us:9.1f} | {alg / 1e12:8.1f} "
              f"{alg / PEAK_BF16:7.1%} | {3 * alg / 1e12:8.1f} {3 * alg / PEAK_BF16:7.1%} | {feed / 1e12:11.2f}")
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "gemm_bench.json"), "w") as f:
            json.dump({"gpu": info, "sms": sms.value, "peak_bf16_dense": PEAK_BF16, "shapes": rows}, f, indent=1)


if __name__ == "__main__":
    main()
