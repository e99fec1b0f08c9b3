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


def run(M, N, K, batch=1, iters=20, tr=0, what=""):
    ms = C.c_float()
    rc = eng.lib.wl_bench_gemm(eng.ctx, M, N, K, batch, iters, tr, C.byref(ms))
    _lib.check(eng.lib, eng.ctx, rc, "wl_bench_gemm")
    fl = 2.0 * M * N * K * batch
    by = 2.0 * batch * (M * K + N * K + M * N)
    print(f"M={M:6d} N={N:5d} K={K:5d} Z={batch:3d} tr={tr:2d} BN={os.environ.get('WLB200_BN', 'auto'):>4s}: {ms.value * 1000:9.1f} us  "
          f"{fl / ms.value / 1e9:8.1f} TFLOP/s  {by / ms.value / 1e6:8.1f} GB/s  {what}", flush=True)


# One encoder pass takes WLB200_ENC_BATCH = 16 streams: M = 16 x 1500 rows, each GEMM with the epilogue the engine
# gives it (engine.cu encoder_pass).  flags: 2 bias, 4 GELU, 8 fp32 output + fp32 residual in place, 16 bias on m,
# 32 A shared by the batch, 64 output rows padded to a multiple of 64 (V^T rows are S_PAD = 1536 apart).
print("# encoder pass of large-v3 at 16 streams (M = 24000), engine epilogues")
run(24000, 2560, 1280, tr=2, what="QK: fp16 + bias")
run(1280, 1500, 1280, batch=16, tr=2 | 16 | 32 | 64, what="V^T (swap-AB): fp16 + bias on m, W shared")
run(24000, 1280, 1280, tr=8 | 2, what="O: fp32 + bias + residual")
run(24000, 5120, 1280, tr=2 | 4, what="FC1: fp16 + bias + GELU")
run(24000, 1280, 5120, tr=8 | 2, what="FC2: fp32 + bias + residual")
run(24000, 1280, 1280, tr=2, what="cross-KV shape: fp16 + bias (row store in place of the head-split layout)")
print("# plain fp32 store")
for (M, N, K) in [(24000, 2560, 1280), (24000, 1280, 1280), (24000, 5120, 1280), (24000, 1280, 5120), (8192, 8192, 8192)]:
    run(M, N, K)
print("# attention shapes (per head batches)")
run(1500, 1500, 64, batch=40)
run(1500, 64, 1536, batch=40)
print("# decoder swap-AB shapes (weights stream once; R = 16 / 128 rows)")
for R in (16, 128):
    for (Mo, K) in [(3840, 1280), (1280, 1280), (5120, 1280), (1280, 5120), (51866, 1280)]:
        run(Mo, R, K, tr=1, iters=50)
