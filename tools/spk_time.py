"""Device time of wl_spk_embed (speaker embeddings) at 1 / 8 / 32 / 64 segments of 2, 10 and 30 s, with random
weights of the real shapes.  Prints one line per shape: the fbank + CMN and network device times (CUDA events on the
library stream, the median of --iters calls after a warm-up call), the host time of the whole call (upload, launches,
download), and the achieved FLOP/s of the network from the shape-counted operations (tests/spk_oracle.flops) against the
989 TFLOP/s dense FP16 data-sheet figure of the H100 SXM.  The card name and power limit are read in the same run.

    python tools/spk_time.py [--iters 10] [--out spk_time.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

from tests.spk_oracle import flops  # noqa: E402
from whisperlive_b200 import speaker as S, synth  # noqa: E402
from whisperlive_b200.config import dims_for  # noqa: E402
from whisperlive_b200.engine import B200Whisper  # noqa: E402
from whisperlive_b200.weights import random_init  # noqa: E402

PEAK_FP16 = 989e12


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    dims = dims_for("micro.en")
    eng = B200Whisper(dims, random_init(dims, seed=0), max_streams=64, max_beam=1)
    eng.spk_load(S.random_weights(0))
    rows = []
    print("card:", card())
    print(f"{'B':>3} {'s':>4} {'fbank ms':>9} {'net ms':>8} {'host ms':>8} {'TFLOP/s':>8} {'of peak':>8}")
    for seconds in (2, 10, 30):
        for B in (1, 8, 32, 64):
            waves = [synth.speech_like(float(seconds), seed=i) for i in range(B)]
            eng.spk_embeddings(waves)
            fb, net, host = [], [], []
            for _ in range(a.iters):
                t0 = time.perf_counter()
                eng.spk_embeddings(waves)
                host.append((time.perf_counter() - t0) * 1e3)
                fb.append(eng.last_device_ms(8))
                net.append(eng.last_device_ms(9))
            f, n, h = float(np.median(fb)), float(np.median(net)), float(np.median(host))
            rate = B * flops(seconds * 16000) / (n * 1e-3)
            rows.append(dict(B=B, seconds=seconds, fbank_ms=f, network_ms=n, host_ms=h, tflops=rate / 1e12,
                             share_of_fp16_peak=rate / PEAK_FP16))
            print(f"{B:>3} {seconds:>4} {f:>9.3f} {n:>8.3f} {h:>8.3f} {rate / 1e12:>8.1f} {rate / PEAK_FP16:>8.1%}")
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(dict(card=card(), rows=rows), fh, indent=1)
    eng.destroy()


if __name__ == "__main__":
    main()
