"""Silero VAD on the device: device ms of wl_vad (front end and recurrence, CUDA events) for 1, 8 and 32 streams x 30 s,
and the time of add_streams for 32 VAD-gated streams with vad="device" against the float64 oracle standing in for the
CPU model (not onnxruntime: the reference's CPU Silero time is not measured here).
    python tools/vad_time.py --reps 5"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--seconds", type=float, default=30.0)
a = ap.parse_args()

from tests import vad_oracle
from whisperlive_b200 import synth
from whisperlive_b200.transcriber import B200WhisperModel
from whisperlive_b200.vad import DeviceVad, VadOptions, random_weights

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip().splitlines()
print(f"card: {card[0] if card else 'unknown'}", flush=True)

m = B200WhisperModel("tiny.en", weights="random", seed=0, hf_tokenizer="synthetic", max_streams=32, vad="device")
eng = m.model
waves = [synth.speech_like(a.seconds, seed=500 + i) for i in range(32)]
for B in (1, 8, 32):
    eng.vad_probs(waves[:B])        # warm-up (first-use workspace growth, module load)
    front, recur, wall = [], [], []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        eng.vad_probs(waves[:B])    # returns after the device-to-host copy has completed
        wall.append((time.perf_counter() - t0) * 1e3)
        front.append(eng.last_device_ms(6))
        recur.append(eng.last_device_ms(7))
    print(f"wl_vad {B:2d} x {a.seconds:.0f} s: front end {np.median(front):.3f} ms, recurrence {np.median(recur):.3f} ms "
          f"(device, median of {a.reps}); host call {np.median(wall):.2f} ms incl. upload and download", flush=True)

kws = [dict(language="en", vad_filter=True, vad_parameters={"threshold": 0.5}) for _ in waves]


def add_streams_ms(vad):
    m._vad = vad
    best = []
    for _ in range(2):
        sess = m.open_session()
        t0 = time.perf_counter()
        sess.add_streams(waves, [dict(k) for k in kws])
        best.append((time.perf_counter() - t0) * 1e3)
        sess.close()
    return min(best)


dv = m._vad
t_dev = add_streams_ms(dv)
t_orc = add_streams_ms(DeviceVad(vad_oracle.OracleVadEngine(), weights=random_weights(0)))
print(f"add_streams, 32 VAD-gated streams x {a.seconds:.0f} s: vad='device' {t_dev:.1f} ms; "
      f"float64 oracle stand-in (not onnxruntime) {t_orc:.1f} ms", flush=True)
m.destroy()
