"""Short hot-path pass for a profiler: large-v3-shaped engine, S streams, a few decode steps.
    python tools/profile_step.py [--model large-v3] [--streams 8] [--tokens 6] [--beam 4]
The profiled region (cudaProfilerStart/Stop) is one mel + encode + generate pass after a warm-up pass."""
import argparse
import ctypes
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap = argparse.ArgumentParser()
ap.add_argument("--model", default="large-v3")
ap.add_argument("--streams", type=int, default=8)
ap.add_argument("--tokens", type=int, default=6)
ap.add_argument("--beam", type=int, default=4)
ap.add_argument("--no-graph", action="store_true")
a = ap.parse_args()

from whisperlive_b200 import synth
from whisperlive_b200.config import dims_for
from whisperlive_b200.engine import B200Whisper
from whisperlive_b200.weights import random_init

dims = dims_for(a.model)
eng = B200Whisper(dims, random_init(dims, seed=0), max_streams=a.streams, max_beam=max(a.beam, 1), enc_slots=a.streams + 1,
                  alignment_heads=[(dims.dec_layers - 1, 0)], use_cuda_graph=not a.no_graph)
waves = [synth.speech_like(30.0, seed=1234 + i) for i in range(a.streams)]
sot = [eng.sot] if not dims.multilingual else [eng.sot, eng.sot + 1, eng.sot + 1 + dims.num_languages + 1]


def one_pass():
    feats = eng.mel(waves)
    f3 = np.stack([f[:, :3000] for f in feats])
    enc = eng.encode(f3)
    out = eng.generate(enc, [sot] * a.streams, beam_size=a.beam, suppress_tokens=[eng.eot], suppress_blank=False,
                       max_length=2 * a.tokens)
    return out


one_pass()
rt = ctypes.CDLL("libcudart.so")
rt.cudaProfilerStart()
out = one_pass()
rt.cudaProfilerStop()
print("steps", [o.steps for o in out], "mel ms", eng.last_device_ms(0), "enc ms (last pass)", eng.last_device_ms(1), "gen ms",
      eng.last_device_ms(2))
