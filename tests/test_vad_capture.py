"""Consumes tests/golden/silero_vad_capture.{npz,json}, recorded from faster-whisper 1.2.0's own Silero model by
tests/golden/capture_silero_vad.py.  Neither faster-whisper nor onnxruntime nor the model file is available where this
project is built, so without the recording every test here SKIPS with that reason and the recalled frame protocol of
whisperlive_b200/vad.py stays unpinned.

What the recording pins once committed:
  * the gating restatement: get_speech_timestamps of the real module on the real probabilities, per option set;
  * the frame protocol and the network: the float64 oracle (tests/vad_oracle.py) on the bundled weights, read by the
    project's ONNX reader, against the recorded probabilities (needs the model: WLB200_VAD_MODEL or faster-whisper);
  * the frame counts at 511, 512 and 513 samples (the extra frame at an aligned length).
"""
import json
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
NPZ = os.path.join(HERE, "golden", "silero_vad_capture.npz")
JSN = os.path.join(HERE, "golden", "silero_vad_capture.json")
HAVE = os.path.exists(NPZ) and os.path.exists(JSN)
needs_capture = pytest.mark.skipif(not HAVE, reason="no Silero VAD capture committed: run tests/golden/capture_silero_vad.py "
                                   "on a machine with faster-whisper 1.2.0 and onnxruntime (the VAD frame protocol stays "
                                   "unpinned until then)")


def _load():
    with open(JSN) as f:
        return np.load(NPZ), json.load(f)


def _audio(name):
    from tests.golden.capture_silero_vad import inputs
    return inputs()[name]


@needs_capture
def test_frame_counts_match_the_recording():
    from whisperlive_b200.vad import n_frames
    probs, meta = _load()
    for name, n in meta["lengths"].items():
        assert probs[name].shape == (n_frames(n),), name


@needs_capture
def test_gating_restatement_matches_the_recording():
    from whisperlive_b200.vad import VadOptions, speech_timestamps_from_probs
    probs, meta = _load()
    for name, by_opt in meta["timestamps"].items():
        for key, want in by_opt.items():
            got = speech_timestamps_from_probs(probs[name], meta["lengths"][name], VadOptions(**meta["options"][key]))
            assert got == want, (name, key)


@needs_capture
def test_oracle_on_the_bundled_weights_matches_the_recording():
    from tests import vad_oracle
    from whisperlive_b200.vad import resolve_weights
    try:
        w = resolve_weights(None)
    except RuntimeError as e:
        pytest.skip(f"the bundled Silero model is not available here: {e}")
    probs, meta = _load()
    for name in meta["lengths"]:
        np.testing.assert_allclose(vad_oracle.probs(_audio(name), w), probs[name], rtol=0, atol=1e-4, err_msg=name)
