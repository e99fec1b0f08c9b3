"""GPU feature extractor with the ``faster_whisper.feature_extractor.FeatureExtractor`` surface
(constructed at whisper_live/transcriber/transcriber_faster_whisper.py:655, called at :862, :1759 and
whisper_live/batch_inference.py:258; attributes read at :657-665, :1057-1058, :1115-1126).
The arithmetic is kernel K1 in libwlb200 (csrc/mel.cu); only the Slaney filterbank table is built
here (host, float64 -> float32) and uploaded once."""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np


def mel_filters(n_mels: int, sr: int = 16000, n_fft: int = 400) -> np.ndarray:
    """[n_mels, n_fft//2+1] float32 Slaney mel filterbank (area-normalised triangles)."""
    hz = np.fft.rfftfreq(n_fft, 1.0 / sr)
    mel = np.linspace(0.0, 45.245640471924965, n_mels + 2)
    edges = np.where(mel >= 15.0, 1000.0 * np.exp((np.log(6.4) / 27.0) * (mel - 15.0)), (200.0 / 3.0) * mel)
    up = (hz[None, :] - edges[:-2, None]) / (edges[1:-1] - edges[:-2])[:, None]
    down = (edges[2:, None] - hz[None, :]) / (edges[2:] - edges[1:-1])[:, None]
    fb = np.clip(np.minimum(up, down), 0.0, None) * (2.0 / (edges[2:] - edges[:-2]))[:, None]
    return fb.astype(np.float32)


class ResidentFeatures:
    """The log-mel of one stream, resident in HBM (engine.mel_device).  Quacks like the ``float32 [n_mels, frames]``
    array the reference's FeatureExtractor returns as far as the transcriber needs it: ``shape`` and slicing along the
    frame axis (``f[:, a:b]`` / ``f[..., a:]``), which yields views the engine encodes with ``encode_windows``.
    ``np.asarray(f)`` is deliberately not supported -- a consumer that needs host values calls the host-returning
    ``FeatureExtractor.__call__``."""

    ndim = 2

    def __init__(self, engine, stream: int, n_mels: int, start: int, stop: int, epoch: int):
        self.engine, self.stream, self.n_mels, self.start, self.stop, self.epoch = engine, stream, n_mels, start, stop, epoch

    @property
    def shape(self):
        return (self.n_mels, self.stop - self.start)

    def __getitem__(self, key) -> "ResidentFeatures":
        if not isinstance(key, tuple):
            key = (key,)
        sl = key[-1]
        lead = key[:-1]
        ok_lead = all(k is Ellipsis or (isinstance(k, slice) and k == slice(None)) for k in lead)
        if not (isinstance(sl, slice) and sl.step in (None, 1) and ok_lead and len(lead) <= 1):
            raise TypeError("ResidentFeatures supports slicing along the frame axis only")
        a, b, _ = sl.indices(self.stop - self.start)
        return ResidentFeatures(self.engine, self.stream, self.n_mels, self.start + a, self.start + max(a, b), self.epoch)

    @property
    def resident(self) -> bool:
        """False once a later mel_device call on the engine has replaced these features."""
        return getattr(self.engine, "_resident_epoch", None) == self.epoch

    def window(self, max_frames: int = 3000):
        """(stream, seek, length) for engine.encode_windows."""
        if not self.resident:
            raise RuntimeError("these features are no longer resident: a later mel_device call replaced them")
        return (self.stream, self.start, min(self.stop - self.start, max_frames))


class FeatureExtractor:
    def __init__(self, engine, feature_size: int = 80, sampling_rate: int = 16000, hop_length: int = 160,
                 chunk_length: int = 30, n_fft: int = 400):
        if (sampling_rate, hop_length, n_fft) != (16000, 160, 400):
            raise ValueError("the CUDA mel kernel is specialised for 16 kHz / hop 160 / n_fft 400 (every Whisper checkpoint)")
        if feature_size != engine.n_mels:
            raise ValueError(f"feature_size {feature_size} does not match the model's n_mels {engine.n_mels}")
        self.engine = engine
        self.n_fft = n_fft
        self.hop_length = hop_length
        self.chunk_length = chunk_length
        self.n_samples = chunk_length * sampling_rate
        self.nb_max_frames = self.n_samples // hop_length
        self.time_per_frame = hop_length / sampling_rate
        self.sampling_rate = sampling_rate
        self.feature_size = feature_size
        self.mel_filters = mel_filters(feature_size)

    def _set_chunk(self, chunk_length: Optional[int]) -> None:
        if chunk_length is not None:
            self.n_samples = chunk_length * self.sampling_rate
            self.nb_max_frames = self.n_samples // self.hop_length

    def __call__(self, waveform: np.ndarray, padding: int = 160, chunk_length: Optional[int] = None) -> np.ndarray:
        return self.batch([waveform], padding, chunk_length)[0]

    def batch_resident(self, waveforms: Sequence[np.ndarray], chunk_length: Optional[int] = None) -> List[ResidentFeatures]:
        """Like ``batch`` but the features stay in HBM (at most ``engine.max_streams`` waveforms per call, valid until
        the next call): what ``B200WhisperModel.transcribe_batch`` uses between its own mel and encode steps."""
        self._set_chunk(chunk_length)
        frames = self.engine.mel_device(waveforms)
        ep = self.engine._resident_epoch
        return [ResidentFeatures(self.engine, i, self.feature_size, 0, f, ep) for i, f in enumerate(frames)]

    def batch(self, waveforms: Sequence[np.ndarray], padding: int = 160, chunk_length: Optional[int] = None) -> List[np.ndarray]:
        if padding != 160:
            raise ValueError("padding must be 160 (the reference never passes anything else)")
        self._set_chunk(chunk_length)
        return self.engine.mel(waveforms)
