"""Batched long-file transcription: audio-seconds per second of ``BatchedInferencePipeline`` on large-v3 (random
weights, synthetic tokenizer) over about 10 minutes of gapped synthetic speech, at batch_size 1 / 8 / 16 / max_streams,
against ``B200WhisperModel.transcribe`` (one window after another, each prompted with the previous text) on the same
audio.  Chunks come from the deterministic energy-gate detector of tests/stub_vad.py on both paths (random Silero
weights would find no speech).  ``max_new_tokens`` bounds every decode: random weights would otherwise run every chunk
to 448 tokens.  Per group it prints the mean and the longest chunk's token steps -- how long the group's one
``generate`` call waits for its slowest chunk.
    python tools/batched_time.py --minutes 10 --max-new-tokens 48 --reps 2"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ap = argparse.ArgumentParser()
ap.add_argument("--model", default="large-v3")
ap.add_argument("--minutes", type=float, default=10.0)
ap.add_argument("--max-streams", type=int, default=32)
ap.add_argument("--max-new-tokens", type=int, default=48)
ap.add_argument("--beam", type=int, default=5)
ap.add_argument("--reps", type=int, default=2)
a = ap.parse_args()

from tests import stub_vad
from whisperlive_b200 import synth
from whisperlive_b200.transcriber import B200WhisperModel, BatchedInferencePipeline

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip().splitlines()
print(f"card: {card[0] if card else 'unknown'}", flush=True)

rng = np.random.default_rng(7)
parts, total, i = [], 0.0, 0
while total < a.minutes * 60:
    speech, pause = float(rng.uniform(4.0, 20.0)), float(rng.uniform(0.8, 4.0))
    parts += [synth.speech_like(speech, seed=900 + i), synth.silence(pause)]
    total += speech + pause
    i += 1
audio = np.concatenate(parts).astype(np.float32)
duration = len(audio) / 16000

m = B200WhisperModel(a.model, weights="random", seed=0, hf_tokenizer="synthetic", max_streams=a.max_streams,
                     max_beam=max(a.beam, 1), vad=stub_vad)
pipe = BatchedInferencePipeline(m)
common = dict(beam_size=a.beam, max_new_tokens=a.max_new_tokens, language="en")


def timed(fn):
    best, out = None, None
    for _ in range(a.reps):
        t0 = time.perf_counter()
        out = fn()
        dt = time.perf_counter() - t0          # every call ends in a device-to-host copy of its results
        best = dt if best is None else min(best, dt)
    return best, out


list(pipe.transcribe(audio, batch_size=a.max_streams, **common)[0])          # warm-up: module load, workspaces
results = {"card": card[0] if card else "unknown", "model": a.model, "audio_s": round(duration, 1),
           "max_new_tokens": a.max_new_tokens, "beam": a.beam, "batched": {}}
for bs in sorted({1, 8, 16, a.max_streams}):
    dt, segs = timed(lambda: list(pipe.transcribe(audio, batch_size=bs, **common)[0]))
    groups = [dict(chunks=len(g), mean_steps=round(float(np.mean(g)), 1), max_steps=int(max(g))) for g in pipe.group_steps]
    results["batched"][bs] = dict(seconds=round(dt, 3), audio_s_per_s=round(duration / dt, 1), segments=len(segs),
                                  groups=groups)
    print(f"batch_size {bs:2d}: {dt:.2f} s, {duration / dt:.1f} audio-s/s, {sum(x['chunks'] for x in groups)} chunks in "
          f"{len(groups)} groups; per group mean / longest token steps "
          f"{[(x['mean_steps'], x['max_steps']) for x in groups]}", flush=True)

seq_kw = dict(common, vad_filter=True, temperature=[0.0], vad_parameters=dict(min_silence_duration_ms=160))
dt, (segs, _info) = timed(lambda: m.transcribe(audio, **seq_kw))
results["transcribe"] = dict(seconds=round(dt, 3), audio_s_per_s=round(duration / dt, 1), segments=len(segs))
print(f"B200WhisperModel.transcribe (window after window, temperature 0 only): {dt:.2f} s, {duration / dt:.1f} audio-s/s",
      flush=True)
print(json.dumps(results), flush=True)
m.destroy()
