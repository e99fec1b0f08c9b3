"""Consumes tests/golden/wespeaker_capture.{npz,json}, recorded from pyannote's own wespeaker-voxceleb-resnet34-LM by
tests/golden/capture_wespeaker.py.  Neither pyannote.audio nor the checkpoint is available where this project is built,
so without the recording every test here SKIPS with that reason and the protocol whisperlive_b200/speaker.py recalls
stays unpinned (the fbank alone is pinned against torchaudio by tests/test_speaker_embedding.py).

What the recording pins once committed:
  * the checkpoint's tensor names and shapes: the ones the reader expects;
  * input scaling, fbank options and CMN: the float64 oracle's features against pyannote's;
  * the network and pooling: the oracle on the real weights (WLB200_SPK_MODEL) against pyannote's embeddings;
  * fp16 headroom: every stage's activation maximum well inside the fp16 range.
"""
import json
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
NPZ = os.path.join(HERE, "golden", "wespeaker_capture.npz")
JSN = os.path.join(HERE, "golden", "wespeaker_capture.json")
HAVE = os.path.exists(NPZ) and os.path.exists(JSN)
needs_capture = pytest.mark.skipif(not HAVE, reason="no wespeaker capture committed: run tests/golden/capture_wespeaker.py "
                                   "on a machine with pyannote.audio and the checkpoint (the speaker-embedding protocol "
                                   "stays unpinned until then)")


def _load():
    with open(JSN) as f:
        return np.load(NPZ), json.load(f)


def _inputs():
    import importlib.util
    spec = importlib.util.spec_from_file_location("capture_wespeaker", os.path.join(HERE, "golden", "capture_wespeaker.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.inputs()


@needs_capture
def test_checkpoint_tensor_table():
    from whisperlive_b200.speaker import checkpoint_shapes
    _, meta = _load()
    for name, shape in checkpoint_shapes().items():
        assert name in meta["tensors"], name
        assert tuple(meta["tensors"][name][0]) == shape, name


@needs_capture
def test_fbank_after_cmn_matches():
    from tests import spk_oracle as O
    data, _ = _load()
    for key, wave in _inputs().items():
        want = data["fbank_cmn_" + key]
        got = O.features(wave).T
        assert got.shape == want.shape, key
        assert np.abs(got - want).max() < 1e-3, key


@needs_capture
def test_fp16_headroom_on_the_real_weights():
    _, meta = _load()
    for key, stages in meta["stages"].items():
        assert all(mx < 6e3 for mx, _rms in stages), (key, stages)


@needs_capture
def test_oracle_embeddings_on_the_real_weights():
    if not os.environ.get("WLB200_SPK_MODEL"):
        pytest.skip("WLB200_SPK_MODEL (the wespeaker checkpoint) is not set")
    from tests import spk_oracle as O
    from whisperlive_b200.speaker import resolve_weights
    w = resolve_weights(None)
    data, _ = _load()
    for key, wave in _inputs().items():
        if wave.shape[0] < 8 * 160 + 400:
            continue
        want = data["embedding_" + key]
        got = O.embed(wave, w)
        cos = float(np.dot(got, want) / (np.linalg.norm(got) * np.linalg.norm(want)))
        assert cos > 0.9999, (key, cos)
