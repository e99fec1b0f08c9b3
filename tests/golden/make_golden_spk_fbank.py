"""Writes tests/golden/spk_fbank_reference.npz: ``torchaudio.compliance.kaldi.fbank`` -- the function pyannote's
wespeaker wrapper calls -- with the parameters whisperlive_b200/speaker.py names, over the jfk fixture and seeded
noise / tone / impulse waveforms of 400, 401, 559, 560, 4800 samples and 30 s.

For each float32 waveform in [-1, 1] that ``waveforms()`` regenerates from its seed (the tests import it, so the
waveforms are not stored): ``frames_<name>`` is the frame count torchaudio gives, ``index_<name>`` the frames kept and
``fbank_<name>`` the float32 [kept, 80] fbank of ``wave * 32768`` at those frames, before CMN.  Every frame is kept up to
64 frames; a longer waveform keeps its first and last 8 frames and 48 spread between them, which keeps the fixture small
(each frame is computed on its own, so the kept ones check the arithmetic and the count checks the framing).
Run from the repository root: ``python tests/golden/make_golden_spk_fbank.py``."""
import os
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)
from whisperlive_b200 import speaker as S  # noqa: E402


def waveforms():
    jfk = np.load(os.path.join(ROOT, "tests", "golden", "jfk_16k_i16.npy")).astype(np.float32) / 32768.0
    out = {"jfk": jfk}
    for n in (400, 401, 559, 560, 4800, 30 * 16000):
        rng = np.random.default_rng(n)
        t = np.arange(n) / 16000.0
        out[f"noise_{n}"] = (0.1 * rng.standard_normal(n)).astype(np.float32)
        out[f"tone_{n}"] = (0.3 * np.sin(2 * np.pi * rng.uniform(100, 4000) * t)
                            + 1e-3 * rng.standard_normal(n)).astype(np.float32)
        imp = np.zeros(n, np.float32)
        imp[rng.integers(0, n, size=max(1, n // 4000))] = 0.8
        out[f"impulse_{n}"] = imp
    return out


def kept_frames(n: int) -> np.ndarray:
    if n <= 64:
        return np.arange(n, dtype=np.int32)
    mid = np.linspace(8, n - 9, 48).round().astype(np.int64)
    return np.unique(np.concatenate([np.arange(8), mid, np.arange(n - 8, n)])).astype(np.int32)


def main():
    import torch
    import torchaudio
    data = {}
    for name, w in waveforms().items():
        f = torchaudio.compliance.kaldi.fbank(torch.from_numpy(w)[None] * S.INPUT_SCALE, **S.FBANK)
        idx = kept_frames(f.shape[0])
        data["frames_" + name] = np.asarray(f.shape[0], np.int32)
        data["index_" + name] = idx
        data["fbank_" + name] = f.numpy()[idx].astype(np.float32)
    data["torchaudio_version"] = np.asarray(torchaudio.__version__)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "spk_fbank_reference.npz"), **data)


if __name__ == "__main__":
    main()
