#!/usr/bin/env python
"""Capture the reference's own Silero VAD behaviour (faster-whisper 1.2.0 + onnxruntime), the pin of the frame protocol
that whisperlive_b200/vad.py recalls (frame 512, context 64, the STFT reflection pad, the extra frame at aligned
lengths, the gate order) and of its gating restatement.  Run it ONCE on a machine with

    pip install faster-whisper==1.2.0 onnxruntime

and commit what it writes; tests/test_vad_capture.py consumes it (and skips, loudly, without it):

    tests/golden/silero_vad_capture.npz   per-frame probabilities of every recorded input
    tests/golden/silero_vad_capture.json  the bundled model's tensor table (file, name, shape, dtype, consuming nodes),
                                          get_speech_timestamps for the default VadOptions, {"threshold": 0.5} (the
                                          backend's) and a neg_threshold / max_speech_duration_s case, versions

    python tests/golden/capture_silero_vad.py
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))


def inputs():
    from whisperlive_b200 import synth
    jfk = np.load(os.path.join(HERE, "jfk_16k_i16.npy")).astype(np.float32) / 32768.0
    out = {"jfk": jfk}
    for n in (511, 512, 513, 30 * 16000):
        out[f"speech_{n}"] = synth.speech_like(n / 16000, seed=n)
        out[f"noise_{n}"] = synth.white_noise(n / 16000, seed=n, sigma=0.05)
        out[f"silence_{n}"] = synth.silence(n / 16000)
    return out


OPTIONS = {"default": {}, "backend": {"threshold": 0.5},
           "hysteresis_max": {"threshold": 0.6, "neg_threshold": 0.3, "max_speech_duration_s": 3.0,
                              "min_silence_duration_ms": 300, "speech_pad_ms": 100}}


def tensor_table(paths):
    import onnx   # the capture machine has it through onnxruntime's tooling; the product reads ONNX by hand
    rows = []
    for p in paths:
        m = onnx.load(p)

        def walk(g, scope):
            consumers = {}
            for n in g.node:
                for i in n.input:
                    consumers.setdefault(i, []).append(f"{n.op_type}:{n.name}")
                for a in n.attribute:
                    if a.type == onnx.AttributeProto.GRAPH:
                        walk(a.g, scope + "/" + n.name + "." + a.name)
                    if a.type == onnx.AttributeProto.TENSOR:
                        rows.append(dict(file=os.path.basename(p), scope=scope, name=n.output[0], shape=list(a.t.dims),
                                         dtype=int(a.t.data_type), consumers=[]))
            for t in g.initializer:
                rows.append(dict(file=os.path.basename(p), scope=scope, name=t.name, shape=list(t.dims),
                                 dtype=int(t.data_type), consumers=consumers.get(t.name, [])))
            for r in rows:
                if r["scope"] == scope and not r["consumers"]:
                    r["consumers"] = consumers.get(r["name"], [])
        walk(m.graph, "")
    return rows


def main():
    import faster_whisper
    from faster_whisper import vad
    from whisperlive_b200.vad import _bundled_model_files
    model = vad.get_vad_model()
    probs, stamps = {}, {}
    for name, audio in inputs().items():
        pad = 512 - audio.shape[0] % 512
        probs[name] = np.asarray(model(np.pad(audio, (0, pad)))).reshape(-1).astype(np.float32)
        stamps[name] = {k: vad.get_speech_timestamps(audio, vad.VadOptions(**o)) for k, o in OPTIONS.items()}
    files = _bundled_model_files()
    np.savez_compressed(os.path.join(HERE, "silero_vad_capture.npz"), **probs)
    with open(os.path.join(HERE, "silero_vad_capture.json"), "w") as f:
        json.dump(dict(versions={"faster_whisper": faster_whisper.__version__}, model_files=[os.path.basename(p) for p in files],
                       tensors=tensor_table(files), options=OPTIONS, timestamps=stamps,
                       lengths={k: int(v.shape[0]) for k, v in inputs().items()}), f, indent=1)
    print("wrote tests/golden/silero_vad_capture.{npz,json}")


if __name__ == "__main__":
    main()
