"""Generate tests/golden/rest_reference.json by running the reference's own REST route
(whisper_live/server.py ``TranscriptionServer.run(enable_rest=True)``, :693-867 and the SSE variant :490-537) in
process, with Starlette's ``TestClient``:

* ``WhisperModel`` is the reference's vendored ``transcriber_faster_whisper.WhisperModel`` over the CPU oracle engine
  (micro, seeded random weights, synthetic vocabulary), with the sys.modules stubs of make_golden_transcribe.py; the
  upload is read as 16-bit WAV here, since the stubbed ``decode_audio`` has no decoder;
* ``SpeakerDiarizer`` is the reference's class with its pyannote model replaced by tests/spk_oracle.py (seeded random
  wespeaker weights), and ``load_audio`` reads the WAV the same way.

What this pins is the route's answers -- response shapes, SSE events, speaker labels, the 400 cases -- given identical
engine outputs.  Reproducible byte for byte; runs only in the build container.

    python tests/golden/make_golden_rest.py
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)

from tests import rest_app  # noqa: E402
from tests.golden.make_golden_transcribe import install_stubs, reference_model  # noqa: E402

MODEL, SEED, SPK_SEED = "micro", 5, 0


def main():
    torch.set_num_threads(8)
    install_stubs()
    sys.path.insert(0, rest_app.REF)
    from whisper_live.transcriber import transcriber_faster_whisper as ref
    import whisper_live.diarization as diarization
    from oracle.engine import OracleWhisper
    from starlette.testclient import TestClient
    from tests import spk_oracle
    from whisperlive_b200 import speaker
    from whisperlive_b200.config import dims_for
    from whisperlive_b200.weights import random_init

    dims = dims_for(MODEL)
    engine = OracleWhisper(random_init(dims, seed=SEED), dims)
    spk_weights = speaker.random_weights(SPK_SEED)

    class OracleFileModel:
        """The vendored WhisperModel; the route passes a file path, which is read here."""

        def __init__(self, *a, **k):
            self.m = reference_model(ref, engine, dims)

        def transcribe(self, audio, **kw):
            return self.m.transcribe(rest_app.read_wav(audio) if isinstance(audio, str) else audio, **kw)

    class OracleDiarizer(diarization.SpeakerDiarizer):
        def _load_model(self):
            self._model = lambda wf: spk_oracle.embed(wf["waveform"][0].numpy(), spk_weights)

    server = rest_app.server_module()
    server.WhisperModel = OracleFileModel
    diarization.SpeakerDiarizer = OracleDiarizer
    diarization.load_audio = lambda path, sample_rate=16000: rest_app.read_wav(path)
    client = TestClient(rest_app.build_app(server))
    out = {}
    for name in rest_app.cases():
        out[name] = rest_app.post(client, name)
        print(name, out[name]["status"], out[name]["body"][:160].replace("\n", " | "))
    with open(os.path.join(HERE, "rest_reference.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
