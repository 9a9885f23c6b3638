"""Fixed cost vs per-k-block cost of the wgmma GEMMs at the encoder's shapes: M = 8032 rows, N in {512, 2048}, K swept from one
k-block (64) upward, fp16 / fp32 outputs.  Event-timed over back-to-back launches (after warm-up); prints one line per shape and
a least-squares (intercept, slope per 64-wide k-block)."""
import ctypes
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from speechbrain_b200._lib import lib, check, ptr  # noqa: E402

M = int(sys.argv[1]) if len(sys.argv) > 1 else 8032
dev = torch.device("cuda:0")
st = torch.cuda.current_stream().cuda_stream
for N in (512, 1024, 2048):
    for f32 in (0, 1):
        pts = []
        for K in (64, 128, 256, 512, 1024, 2048):
            A = (torch.randn(M, K, device=dev) * 0.1).half()
            W = (torch.randn(N, K, device=dev) * 0.1).half()
            bias = torch.zeros(N, device=dev)
            out = torch.empty(M, N, device=dev, dtype=torch.float32 if f32 else torch.float16)
            def run():
                check(lib().sbk_gemm_f16_test(ptr(A), ptr(W), ptr(bias), ptr(out), f32, 0, M, N, K, ctypes.c_void_p(st)), "gemm")
            for _ in range(10):
                run()
            torch.cuda.synchronize()
            reps = 200
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                run()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / reps
            pts.append((K // 64, us))
            print(f"M={M} N={N} K={K} out={'f32' if f32 else 'f16'}: {us:7.2f} us  {2.0 * M * N * K / us / 1e6:7.1f} TFLOP/s", flush=True)
        n = len(pts)
        sx = sum(p[0] for p in pts); sy = sum(p[1] for p in pts)
        sxx = sum(p[0] ** 2 for p in pts); sxy = sum(p[0] * p[1] for p in pts)
        slope = (n * sxy - sx * sy) / (n * sxx - sx * sx)
        icpt = (sy - slope * sx) / n
        print(f"  -> N={N} out={'f32' if f32 else 'f16'}: fixed {icpt:.2f} us + {slope:.3f} us per k-block (128 x 256 tiles per SM: {((M + 127) // 128) * (N // 256) / 132:.2f})", flush=True)

# The encoder's own conditions for the N = 512 residual GEMMs: residual epilogue, operands not L2-hot (rotate over buffer sets
# larger than the 50 MB L2), and one CUDA-event pair per launch (what bench.py's roofline pass does) vs pipelined launches.
print("--- residual epilogue (x += A W^T + b), M=%d N=512" % M, flush=True)
for K in (512, 2048):
    for nset in (1, 12):
        As = [(torch.randn(M, K, device=dev) * 0.1).half() for _ in range(nset)]
        Ws = [(torch.randn(512, K, device=dev) * 0.1).half() for _ in range(nset)]
        xs = [torch.zeros(M, 512, device=dev) for _ in range(nset)]
        bias = torch.zeros(512, device=dev)
        def run(i):
            j = i % nset
            check(lib().sbk_gemm_f16_resid_test(ptr(As[j]), ptr(Ws[j]), ptr(bias), ptr(xs[j]), ctypes.c_float(0.5), M, 512, K,
                                                ctypes.c_void_p(st)), "gemm resid")
        for i in range(2 * nset + 4):
            run(i)
        torch.cuda.synchronize()
        reps = 240
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(reps):
            run(i)
        e1.record()
        torch.cuda.synchronize()
        piped = e0.elapsed_time(e1) * 1e3 / reps
        evs = []
        for i in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); run(i); b.record()
            evs.append((a, b))
        torch.cuda.synchronize()
        per = sorted(a.elapsed_time(b) * 1e3 for a, b in evs)
        print(f"resid K={K} buffer sets={nset:2d} ({'L2-hot' if nset == 1 else 'rotating, > L2'}): pipelined {piped:6.2f} us / launch; "
              f"event pair per launch: median {per[len(per) // 2]:6.2f} us (min {per[0]:.2f})", flush=True)
