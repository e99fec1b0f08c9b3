"""Float64 restatement of the Silero VAD network (16 kHz), the yardstick of csrc/vad.cu.

It follows the protocol constants named in whisperlive_b200/vad.py (frame, context, STFT reflection pad, the extra
frame, gate order), so a correction there moves the oracle and the host-side frame count together.  Two entry points:
``probs`` runs a whole stream at once the way faster-whisper does (every frame's input built first, then the
recurrence); ``FrameLoop`` carries h, c and the 64-sample context from call to call, like
whisper_live/vad.py:74-86 feeding 512 samples at a time.  The tests check that the two agree."""
from __future__ import annotations

from typing import Dict, List

import numpy as np

from whisperlive_b200.vad import (CONTEXT_SAMPLES, FRAME_SAMPLES, HIDDEN, STFT_REFLECT_PAD, n_frames)


def _w(weights: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    return {k: np.asarray(v, dtype=np.float64) for k, v in weights.items()}


def _conv1d(x: np.ndarray, w: np.ndarray, b: np.ndarray, stride: int, pad: int) -> np.ndarray:
    """x [N, ci, T], w [co, ci, k] -> [N, co, T_out]"""
    if pad:
        x = np.pad(x, ((0, 0), (0, 0), (pad, pad)))
    k = w.shape[2]
    t_out = (x.shape[2] - k) // stride + 1
    cols = np.stack([x[:, :, t * stride:t * stride + k] for t in range(t_out)], axis=1)   # [N, T, ci, k]
    return np.einsum("ntck,ock->not", cols, w) + b[None, :, None]


def frame_inputs(audio: np.ndarray) -> np.ndarray:
    """[n_frames, 576]: each frame's 64 context samples (zeros for frame 0) then its 512 samples, zero-padded."""
    a = np.asarray(audio, dtype=np.float64).reshape(-1)
    nf = n_frames(a.shape[0])
    padded = np.zeros(nf * FRAME_SAMPLES)
    padded[:a.shape[0]] = a
    frames = padded.reshape(nf, FRAME_SAMPLES)
    ctx = np.zeros((nf, CONTEXT_SAMPLES))
    if nf > 1:
        ctx[1:] = frames[:-1, -CONTEXT_SAMPLES:]
    return np.concatenate([ctx, frames], axis=1)


def encoder(x576: np.ndarray, weights: Dict[str, np.ndarray]) -> np.ndarray:
    """[N, 576] -> the LSTM input [N, 128]"""
    w = _w(weights)
    side, width = STFT_REFLECT_PAD
    pad = (0, width) if side == "right" else (width, 0) if side == "left" else (width, width)
    x = np.pad(x576, ((0, 0), pad), mode="reflect")[:, None, :]
    spec = _conv1d(x, w["vad.stft.basis"], np.zeros(258), stride=128, pad=0)     # [N, 258, 4]
    mag = np.sqrt(spec[:, :129] ** 2 + spec[:, 129:] ** 2)
    h = np.maximum(_conv1d(mag, w["vad.conv0.weight"], w["vad.conv0.bias"], 1, 1), 0)
    h = np.maximum(_conv1d(h, w["vad.conv1.weight"], w["vad.conv1.bias"], 2, 1), 0)
    h = np.maximum(_conv1d(h, w["vad.conv2.weight"], w["vad.conv2.bias"], 2, 1), 0)
    h = np.maximum(_conv1d(h, w["vad.conv3.weight"], w["vad.conv3.bias"], 1, 1), 0)
    assert h.shape[1:] == (128, 1), h.shape
    return h[:, :, 0]


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def decoder_step(x: np.ndarray, h: np.ndarray, c: np.ndarray, w: Dict[str, np.ndarray]):
    """One LSTM cell step (gate order i, f, g, o) and the output head; returns (prob, h, c)."""
    g = w["vad.lstm.weight_ih"] @ x + w["vad.lstm.bias_ih"] + w["vad.lstm.weight_hh"] @ h + w["vad.lstm.bias_hh"]
    i, f, gg, o = np.split(g, 4)
    c = _sigmoid(f) * c + _sigmoid(i) * np.tanh(gg)
    h = _sigmoid(o) * np.tanh(c)
    logit = w["vad.out.weight"][0, :, 0] @ np.maximum(h, 0) + w["vad.out.bias"][0]
    return float(_sigmoid(logit)), h, c


def probs(audio: np.ndarray, weights: Dict[str, np.ndarray]) -> np.ndarray:
    """Per-frame speech probabilities of one whole stream (float64)."""
    x = frame_inputs(audio)
    if x.shape[0] == 0:
        return np.zeros(0)
    enc = encoder(x, weights)
    w = _w(weights)
    h, c = np.zeros(HIDDEN), np.zeros(HIDDEN)
    out = np.empty(enc.shape[0])
    for t in range(enc.shape[0]):
        out[t], h, c = decoder_step(enc[t], h, c, w)
    return out


class FrameLoop:
    """Frame-by-frame use with the state carried by the caller's side: 512 new samples per call."""

    def __init__(self, weights: Dict[str, np.ndarray]):
        self.weights = weights
        self.w = _w(weights)
        self.h, self.c = np.zeros(HIDDEN), np.zeros(HIDDEN)
        self.context = np.zeros(CONTEXT_SAMPLES)

    def __call__(self, chunk512: np.ndarray) -> float:
        x = np.concatenate([self.context, np.asarray(chunk512, dtype=np.float64)])
        self.context = x[-CONTEXT_SAMPLES:]
        p, self.h, self.c = decoder_step(encoder(x[None], self.weights)[0], self.h, self.c, self.w)
        return p


class OracleVadEngine:
    """Stands in for the CUDA engine under ``DeviceVad``: the oracle's probabilities, counting the calls."""

    def __init__(self):
        self.weights = None
        self.calls: List[int] = []

    def vad_load(self, tensors):
        self.weights = dict(tensors)

    def vad_probs(self, audios):
        self.calls.append(len(audios))
        return [probs(a, self.weights).astype(np.float32) for a in audios]
