"""Float64 numpy restatement of the speaker-embedding protocol named in whisperlive_b200/speaker.py: Kaldi fbank, CMN,
the wespeaker ResNet34 (folded ``spk.*`` weights, or the pyannote-named state dict with explicit BatchNorm), TSTP pooling
and the embedding layer.  The checker the device kernels (csrc/spk.cu) and the golden torchaudio fixture are compared
with."""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np

from whisperlive_b200 import speaker as S


def _mel(f):
    return 1127.0 * np.log(1.0 + np.asarray(f, np.float64) / 700.0)


def mel_banks() -> np.ndarray:
    """[80, 257] triangular filters on Kaldi's mel scale, 20 Hz .. Nyquist (the Nyquist column is zero)."""
    nb, half = S.MEL_BINS, S.N_FFT // 2
    width = S.SAMPLING_RATE / S.N_FFT
    lo, hi = _mel(S.MEL_LOW_HZ), _mel(S.SAMPLING_RATE / 2)
    delta = (hi - lo) / (nb + 1)
    m = _mel(width * np.arange(half))
    out = np.zeros((nb, half + 1))
    for b in range(nb):
        left, center, right = lo + b * delta, lo + (b + 1) * delta, lo + (b + 2) * delta
        up = (m - left) / (center - left)
        down = (right - m) / (right - center)
        out[b, :half] = np.maximum(0.0, np.minimum(up, down))
    return out


def fbank(wave: np.ndarray) -> np.ndarray:
    """[frames, 80] log mel energies of a waveform in [-1, 1] (scaled by 32768 first), before CMN."""
    x = np.asarray(wave, np.float64).reshape(-1) * S.INPUT_SCALE
    T = S.n_frames(x.shape[0])
    if T == 0:
        return np.zeros((0, S.MEL_BINS))
    idx = np.arange(T)[:, None] * S.FRAME_SHIFT + np.arange(S.FRAME_SAMPLES)[None, :]
    fr = x[idx]
    fr = fr - fr.mean(axis=1, keepdims=True)
    prev = np.concatenate([fr[:, :1], fr[:, :-1]], axis=1)
    fr = fr - S.PREEMPHASIS * prev
    n = np.arange(S.FRAME_SAMPLES)
    win = 0.54 - 0.46 * np.cos(2 * np.pi * n / (S.FRAME_SAMPLES - 1))
    spec = np.fft.rfft(fr * win, n=S.N_FFT, axis=1)
    power = spec.real ** 2 + spec.imag ** 2
    return np.log(np.maximum(power @ mel_banks().T, S.LOG_FLOOR))


def features(wave: np.ndarray) -> np.ndarray:
    """The network input [80, T]: fbank after CMN, frequency as H and time as W."""
    f = fbank(wave)
    return (f - f.mean(axis=0, keepdims=True)).T


def conv2d(x: np.ndarray, w: np.ndarray, b: Optional[np.ndarray], stride: int) -> np.ndarray:
    """x [C_in, H, W], w [C_out, C_in, k, k] (k = 3 with padding 1, or 1 without) -> [C_out, H', W']."""
    ci, H, W = x.shape
    co, _, k, _ = w.shape
    p = k // 2
    Ho, Wo = (H + 2 * p - k) // stride + 1, (W + 2 * p - k) // stride + 1
    xp = np.pad(x, ((0, 0), (p, p), (p, p)))
    cols = np.empty((ci, k, k, Ho, Wo))
    for dh in range(k):
        for dw in range(k):
            cols[:, dh, dw] = xp[:, dh:dh + stride * (Ho - 1) + 1:stride, dw:dw + stride * (Wo - 1) + 1:stride]
    y = w.reshape(co, -1) @ cols.reshape(ci * k * k, Ho * Wo)
    if b is not None:
        y += b[:, None]
    return y.reshape(co, Ho, Wo)


def _relu(x):
    return np.maximum(x, 0.0)


def _folded_conv(w: Dict[str, np.ndarray], name: str):
    W, b = w[name + ".weight"].astype(np.float64), w[name + ".bias"].astype(np.float64)
    return lambda x, stride: conv2d(x, W, b, stride)


def _bn_conv(sd: Dict[str, np.ndarray], conv: str, bn: str):
    W = np.asarray(sd[conv + ".weight"], np.float64)
    g, beta = np.asarray(sd[bn + ".weight"], np.float64), np.asarray(sd[bn + ".bias"], np.float64)
    m, v = np.asarray(sd[bn + ".running_mean"], np.float64), np.asarray(sd[bn + ".running_var"], np.float64)

    def f(x, stride):
        y = conv2d(x, W, None, stride)
        return ((y - m[:, None, None]) / np.sqrt(v[:, None, None] + S.BN_EPS)) * g[:, None, None] + beta[:, None, None]
    return f


def _convs(weights: Dict[str, np.ndarray]):
    """spk prefix -> conv(x, stride) for folded weights, or for a pyannote state dict with explicit BN."""
    sd = weights.get("state_dict", weights)
    if "resnet.conv1.weight" in sd:
        return {name: _bn_conv(sd, conv, bn) for name, conv, bn in S._checkpoint_convs()}, \
            (np.asarray(sd["resnet.seg_1.weight"], np.float64), np.asarray(sd["resnet.seg_1.bias"], np.float64))
    return {name: _folded_conv(weights, name) for name, *_ in S.conv_names()}, \
        (weights["spk.seg_1.weight"].astype(np.float64), weights["spk.seg_1.bias"].astype(np.float64))


def network(x: np.ndarray, weights: Dict[str, np.ndarray], stages: Optional[List[np.ndarray]] = None) -> np.ndarray:
    """x [80, T] -> the embedding [256].  ``stages``: when a list, receives the stem output and each stage's output."""
    conv, (w1, b1) = _convs(weights)
    h = _relu(conv["spk.conv1"](x[None], 1))
    if stages is not None:
        stages.append(h)
    cin = S.STEM_CHANNELS
    for L, (c, nb, stride) in enumerate(S.STAGES, start=1):
        for i in range(nb):
            s = stride if i == 0 else 1
            y = _relu(conv[f"spk.layer{L}.{i}.conv1"](h, s))
            y = conv[f"spk.layer{L}.{i}.conv2"](y, 1)
            short = conv[f"spk.layer{L}.{i}.shortcut"](h, s) if (i == 0 and (s != 1 or cin != c)) else h
            h = _relu(y + short)
            cin = c
        if stages is not None:
            stages.append(h)
    return pooled_embedding(h, w1, b1)


def pooled_embedding(h: np.ndarray, w1: np.ndarray, b1: np.ndarray) -> np.ndarray:
    """TSTP over time of [C * H, T'] then seg_1."""
    C, H, Tp = h.shape
    f = h.reshape(C * H, Tp)
    mean = f.mean(axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        var = ((f - mean[:, None]) ** 2).sum(axis=1) / (Tp - 1)
    pooled = np.concatenate([mean, np.sqrt(var + S.POOL_VAR_EPS)])
    return w1 @ pooled + b1


def embed(wave: np.ndarray, weights: Dict[str, np.ndarray]) -> np.ndarray:
    return network(features(wave), weights)


def flops(n_samples: int) -> int:
    """Multiply-adds x 2 of the convolutions and the embedding layer for one segment."""
    T = S.n_frames(n_samples)
    H, W, total = S.MEL_BINS, T, 2 * S.STEM_CHANNELS * 9 * S.MEL_BINS * T
    cin = S.STEM_CHANNELS
    for c, nb, stride in S.STAGES:
        for i in range(nb):
            s = stride if i == 0 else 1
            Ho, Wo = -(-H // s), -(-W // s)
            total += 2 * c * cin * 9 * Ho * Wo + 2 * c * c * 9 * Ho * Wo
            if i == 0 and (s != 1 or cin != c):
                total += 2 * c * cin * Ho * Wo
            H, W, cin = Ho, Wo, c
    return total + 2 * S.POOL_DIM * S.EMBED_DIM
