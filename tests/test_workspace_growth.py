"""Workspaces that grow with the calls they serve (``wl_mel``, ``wl_vad``) replace the buffer before them: after the
calls grow twice, ``device_bytes`` has gained exactly the last size, computed here from the engine's sizing rules, and
a fixed input gives the same output bit for bit before and after the growth."""
import numpy as np
import pytest

from whisperlive_b200 import synth

SR = 16000


def _engine(max_streams):
    from whisperlive_b200.config import dims_for
    from whisperlive_b200.engine import B200Whisper
    from whisperlive_b200.weights import random_init
    dims = dims_for("micro.en")
    return B200Whisper(dims, random_init(dims, seed=0), max_streams=max_streams, max_beam=1)


def _slack(n):
    """wl_mel's workspaces: the request plus a quarter"""
    return n + n // 4


@pytest.mark.gpu
def test_mel_workspaces_replace_the_smaller_ones():
    eng = _engine(max_streams=2)
    try:
        before = eng.device_bytes
        fixed = synth.speech_like(5.0, seed=1)
        first = eng.mel([fixed])[0].copy()
        for sec in (10, 20):
            eng.mel([synth.speech_like(float(sec), seed=sec)])
        n = 20 * SR
        last = 4 * (_slack(n) + _slack((n // 160 + 1) * eng.n_mels))   # float32 PCM and log-mel
        assert eng.device_bytes - before == last
        np.testing.assert_array_equal(eng.mel([fixed])[0], first)
    finally:
        eng.destroy()


@pytest.mark.gpu
def test_vad_workspaces_replace_the_smaller_ones():
    from whisperlive_b200.vad import random_weights
    eng = _engine(max_streams=2)
    try:
        eng.vad_load(random_weights(seed=3))
        before = eng.device_bytes
        fixed = [synth.speech_like(30.0, seed=4), synth.white_noise(30.0, seed=5, sigma=0.05)]
        first = eng.vad_probs(fixed)
        for sec in (60, 120):
            eng.vad_probs([synth.speech_like(float(sec), seed=sec), synth.speech_like(float(sec), seed=sec + 1)])
        n = 120 * SR
        frames = 2 * (n // 512 + 1)
        last = 4 * 2 * n + 4 * frames * 512 + 4 * frames + 8 * 2 * (2 + 1)   # PCM, gate inputs, probabilities, offsets
        assert eng.device_bytes - before == last
        for g, f in zip(eng.vad_probs(fixed), first):
            np.testing.assert_array_equal(g, f)
    finally:
        eng.destroy()
