"""Kernel micro-benchmarks on the GPU: wgmma GEMM TFLOP/s at the encoder shapes, weight-streaming GB/s at
the decoder shapes.  python tools/kbench.py"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from whisperlive_b200 import _lib
from whisperlive_b200.config import dims_for
from whisperlive_b200.engine import B200Whisper
from whisperlive_b200.weights import random_init

dims = dims_for("micro.en")
eng = B200Whisper(dims, random_init(dims, seed=0), max_streams=1, max_beam=1)


def run(M, N, K, batch=1, iters=20, tr=0):
    ms = C.c_float()
    rc = eng.lib.wl_bench_gemm(eng.ctx, M, N, K, batch, iters, tr, C.byref(ms))
    _lib.check(eng.lib, eng.ctx, rc, "wl_bench_gemm")
    fl = 2.0 * M * N * K * batch
    by = 2.0 * batch * (M * K + N * K + M * N)
    print(f"M={M:6d} N={N:5d} K={K:5d} Z={batch:3d} tr={tr} BN={os.environ.get('WLB200_BN', 'auto'):>4s}: {ms.value * 1000:9.1f} us  "
          f"{fl / ms.value / 1e9:8.1f} TFLOP/s  {by / ms.value / 1e6:8.1f} GB/s", flush=True)


print("# encoder shapes (large-v3, 8 streams: M = 12000)")
for (M, N, K) in [(12000, 2560, 1280), (12000, 1280, 1280), (12000, 5120, 1280), (12000, 1280, 5120), (8192, 8192, 8192)]:
    run(M, N, K)
print("# encoder epilogue variants at M=12000: flags 2=bias 4=gelu 8=f32+residual")
for (N, K, fl) in [(2560, 1280, 2), (1280, 1280, 8 | 2), (5120, 1280, 2 | 4), (1280, 5120, 8 | 2)]:
    run(12000, N, K, tr=fl)
print("# attention shapes (per head batches)")
run(1500, 1500, 64, batch=40)
run(1500, 64, 1536, batch=40)
print("# decoder swap-AB shapes (weights stream once; R = 16 / 128 rows)")
for R in (16, 128):
    for (Mo, K) in [(3840, 1280), (1280, 1280), (5120, 1280), (1280, 5120), (51866, 1280)]:
        run(Mo, R, K, tr=1, iters=50)
