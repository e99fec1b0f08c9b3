"""Speaker embeddings on the device behind the reference's ``whisper_live.diarization.SpeakerDiarizer``.

The reference embeds every committed segment with pyannote's ``wespeaker-voxceleb-resnet34-LM`` through PyTorch, one
segment at a time on the client's thread (diarization.py:100-118), and turns diarization off when pyannote.audio is not
installed.  ``wl_spk_embed`` (csrc/spk.cu) computes the same network -- Kaldi fbank, CMN, ResNet34, statistics pooling,
the embedding layer -- for every segment of a round in one CUDA pass; ``DeviceSpeakerDiarizer`` keeps the reference's
clustering and asks the connection's ``RoundScheduler`` for the vectors.

Weights come from a wespeaker checkpoint (``torch.load`` or ``.safetensors``): an explicit file, ``WLB200_SPK_MODEL``,
or a local Hugging Face snapshot of the reference's default ``embedding_model``.  Nothing is downloaded.
``weights="random"`` is the explicit opt-in for tests and tools.

The protocol below is recalled from pyannote.audio / wespeaker; neither is in the reference tree, so nothing here is
read from it.  Each constant is a fact tests/golden/capture_wespeaker.py records on a machine that has the package, and
tests/test_spk_capture.py checks against that record."""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

# ---------------------------------------------------------------------------------------------- the recalled protocol
SAMPLING_RATE = 16000
INPUT_SCALE = 32768.0                # the waveform in [-1, 1] times 2**15 before the fbank
FBANK = dict(num_mel_bins=80, frame_length=25, frame_shift=10, dither=0.0, window_type="hamming", use_energy=False,
             sample_frequency=16000)  # torchaudio.compliance.kaldi.fbank; Kaldi defaults for everything else
FRAME_SAMPLES = 400                  # 25 ms
FRAME_SHIFT = 160                    # 10 ms
N_FFT = 512                          # the frame padded to the next power of two
PREEMPHASIS = 0.97                   # x[i] -= 0.97 x[i - 1], x[0] -= 0.97 x[0]; after the DC offset is removed
MEL_BINS = 80
MEL_LOW_HZ = 20.0                    # mel bins from 20 Hz to Nyquist, Kaldi's mel scale 1127 ln(1 + f / 700)
LOG_FLOOR = float(np.finfo(np.float32).eps)   # log(max(energy, eps))
# CMN: the per-segment mean over frames of each bin is subtracted
STAGES = ((32, 3, 1), (64, 4, 2), (128, 6, 2), (256, 3, 2))   # (channels, BasicBlocks, stride of the first block)
STEM_CHANNELS = 32
BN_EPS = 1e-5
POOL_VAR_EPS = 1e-7                  # TSTP: [mean, sqrt(unbiased var + 1e-7)] over time of [256 * 10, T']
POOL_DIM = 2 * 256 * (MEL_BINS // 8)  # 5120
EMBED_DIM = 256                      # seg_1 (two_emb_layer=False)
DEFAULT_EMBEDDING_MODEL = "pyannote/wespeaker-voxceleb-resnet34-LM"   # SpeakerDiarizer's default (diarization.py:61)


def n_frames(n_samples: int) -> int:
    """Fbank frames of ``n_samples`` (snip_edges): 0 below one frame."""
    return 0 if n_samples < FRAME_SAMPLES else 1 + (n_samples - FRAME_SAMPLES) // FRAME_SHIFT


def conv_names() -> List[Tuple[str, int, int, int]]:
    """``(spk name prefix, C_out, C_in, kernel)`` of every convolution, in network order."""
    out = [("spk.conv1", STEM_CHANNELS, 1, 3)]
    cin = STEM_CHANNELS
    for L, (c, nb, stride) in enumerate(STAGES, start=1):
        for i in range(nb):
            out.append((f"spk.layer{L}.{i}.conv1", c, cin, 3))
            out.append((f"spk.layer{L}.{i}.conv2", c, c, 3))
            if i == 0 and (stride != 1 or cin != c):
                out.append((f"spk.layer{L}.{i}.shortcut", c, cin, 1))
            cin = c
    return out


def tensor_shapes() -> Dict[str, Tuple[int, ...]]:
    """name -> shape of every tensor ``wl_spk_load_tensor`` takes (BN folded into each conv's weight and bias)."""
    shapes: Dict[str, Tuple[int, ...]] = {}
    for name, co, ci, k in conv_names():
        shapes[name + ".weight"] = (co, ci, k, k)
        shapes[name + ".bias"] = (co,)
    shapes["spk.seg_1.weight"] = (EMBED_DIM, POOL_DIM)
    shapes["spk.seg_1.bias"] = (EMBED_DIM,)
    return shapes


TENSOR_SHAPES = tensor_shapes()


def _checkpoint_convs() -> List[Tuple[str, str, str]]:
    """``(spk prefix, checkpoint conv name, checkpoint BN name)`` of every conv."""
    out = []
    for name, _co, _ci, _k in conv_names():
        if name == "spk.conv1":
            out.append((name, "resnet.conv1", "resnet.bn1"))
        elif name.endswith("shortcut"):
            base = "resnet." + name[len("spk."):]
            out.append((name, base + ".0", base + ".1"))
        else:
            base = "resnet." + name[len("spk."):]
            out.append((name, base, base.replace(".conv", ".bn")))
    return out


def checkpoint_shapes() -> Dict[str, Tuple[int, ...]]:
    """name -> shape of every tensor of a pyannote / wespeaker ResNet34 state dict this module reads."""
    shapes: Dict[str, Tuple[int, ...]] = {}
    spk = TENSOR_SHAPES
    for name, conv, bn in _checkpoint_convs():
        shapes[conv + ".weight"] = spk[name + ".weight"]
        for p in ("weight", "bias", "running_mean", "running_var"):
            shapes[f"{bn}.{p}"] = spk[name + ".bias"]
    shapes["resnet.seg_1.weight"] = (EMBED_DIM, POOL_DIM)
    shapes["resnet.seg_1.bias"] = (EMBED_DIM,)
    return shapes


# ---------------------------------------------------------------------------------------------- checkpoints
class CheckpointError(ValueError):
    pass


def fold_checkpoint(state: Dict[str, object]) -> Dict[str, np.ndarray]:
    """A pyannote-named state dict (optionally nested under ``state_dict``) -> the ``spk.*`` tensors, each BN folded into
    its conv in float64: w' = w g / sqrt(v + eps), b' = beta - m g / sqrt(v + eps).  Returns float32 arrays."""
    if "state_dict" in state and isinstance(state["state_dict"], dict):
        state = state["state_dict"]
    arrays: Dict[str, np.ndarray] = {}
    for name, shape in checkpoint_shapes().items():
        if name not in state:
            raise CheckpointError(f"wespeaker checkpoint: tensor {name!r} {list(shape)} is missing")
        t = state[name]
        a = t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
        if a.dtype.kind != "f":
            raise CheckpointError(f"wespeaker checkpoint: tensor {name!r} has dtype {a.dtype}; the weights must be float")
        if tuple(a.shape) != shape:
            raise CheckpointError(f"wespeaker checkpoint: tensor {name!r} has shape {list(a.shape)}, expected {list(shape)}")
        arrays[name] = a.astype(np.float64)
    out: Dict[str, np.ndarray] = {}
    for name, conv, bn in _checkpoint_convs():
        scale = arrays[bn + ".weight"] / np.sqrt(arrays[bn + ".running_var"] + BN_EPS)
        out[name + ".weight"] = (arrays[conv + ".weight"] * scale[:, None, None, None]).astype(np.float32)
        out[name + ".bias"] = (arrays[bn + ".bias"] - arrays[bn + ".running_mean"] * scale).astype(np.float32)
    out["spk.seg_1.weight"] = arrays["resnet.seg_1.weight"].astype(np.float32)
    out["spk.seg_1.bias"] = arrays["resnet.seg_1.bias"].astype(np.float32)
    return out


def read_wespeaker_checkpoint(path) -> Dict[str, np.ndarray]:
    """The ``spk.*`` tensors of a wespeaker ResNet34 checkpoint: ``torch.load(map_location="cpu", weights_only=True)``
    or a ``.safetensors`` file; BN folded (``fold_checkpoint``)."""
    path = os.fspath(path)
    if path.endswith(".safetensors"):
        from safetensors.numpy import load_file
        return fold_checkpoint(load_file(path))
    import torch
    return fold_checkpoint(torch.load(path, map_location="cpu", weights_only=True))


def random_checkpoint(seed: int = 0) -> Dict[str, np.ndarray]:
    """A seeded pyannote-named state dict of the real shapes (tests and tools): He-scaled convs, BN statistics away from
    the identity, and the second conv of each block scaled down so that the residual sums keep every stage's activation
    RMS within [0.1, 10] on speech-like input (tests/test_speaker_embedding.py asserts it)."""
    rng = np.random.default_rng(seed)
    out: Dict[str, np.ndarray] = {}
    for name, conv, bn in _checkpoint_convs():
        co, ci, k, _ = TENSOR_SHAPES[name + ".weight"]
        gain = 0.25 if name.endswith("conv2") else 0.6 if name.endswith("shortcut") else 1.0
        w = rng.standard_normal((co, ci, k, k)) * gain * np.sqrt(2.0 / (ci * k * k))
        out[conv + ".weight"] = w.astype(np.float32)
        out[bn + ".weight"] = rng.uniform(0.6, 1.4, co).astype(np.float32)
        out[bn + ".bias"] = (0.1 * rng.standard_normal(co)).astype(np.float32)
        out[bn + ".running_mean"] = (0.2 * rng.standard_normal(co)).astype(np.float32)
        out[bn + ".running_var"] = rng.uniform(0.5, 2.0, co).astype(np.float32)
        out[bn + ".num_batches_tracked"] = np.asarray(1000, dtype=np.int64)
    out["resnet.seg_1.weight"] = (rng.standard_normal((EMBED_DIM, POOL_DIM)) / np.sqrt(POOL_DIM)).astype(np.float32)
    out["resnet.seg_1.bias"] = (0.01 * rng.standard_normal(EMBED_DIM)).astype(np.float32)
    return out


def random_weights(seed: int = 0) -> Dict[str, np.ndarray]:
    """The ``spk.*`` tensors of ``random_checkpoint(seed)``."""
    return fold_checkpoint(random_checkpoint(seed))


def _local_snapshot(model_name: str) -> str:
    import huggingface_hub
    return huggingface_hub.snapshot_download(model_name, local_files_only=True)


def _checkpoint_in(directory: str) -> str:
    for f in ("pytorch_model.bin", "model.safetensors", "pytorch_model.safetensors"):
        p = os.path.join(directory, f)
        if os.path.isfile(p):
            return p
    raise FileNotFoundError(f"no pytorch_model.bin / model.safetensors in {directory}")


def resolve_weights(weights=None, seed: int = 0, model_name: str = DEFAULT_EMBEDDING_MODEL) -> Dict[str, np.ndarray]:
    """A ``spk.*`` tensor dict, ``"random"`` (seeded), a checkpoint file, or None: ``WLB200_SPK_MODEL``, else a local
    Hugging Face snapshot of ``model_name`` (never downloaded).  Raises when none of these gives the weights."""
    if isinstance(weights, dict):
        return dict(weights)
    if isinstance(weights, str) and weights == "random":
        return random_weights(seed)
    if weights is not None:
        return read_wespeaker_checkpoint(weights)
    env = os.environ.get("WLB200_SPK_MODEL")
    if env:
        return read_wespeaker_checkpoint(_checkpoint_in(env) if os.path.isdir(env) else env)
    try:
        path = _checkpoint_in(_local_snapshot(model_name))
    except Exception as e:
        raise RuntimeError(f"the device speaker embedding needs the wespeaker weights: set WLB200_SPK_MODEL=<checkpoint> "
                           f"or place a local snapshot of {model_name!r} in the Hugging Face cache ({e})") from e
    return read_wespeaker_checkpoint(path)


# ---------------------------------------------------------------------------------------------- the diarizer
try:  # the reference package: DeviceSpeakerDiarizer is its SpeakerDiarizer with the embedding moved to the device
    from whisper_live.diarization import SpeakerDiarizer as _RefDiarizer
except Exception as _e:  # pragma: no cover
    _RefDiarizer = None
    _IMPORT_ERROR = _e


if _RefDiarizer is not None:

    class DeviceSpeakerDiarizer(_RefDiarizer):
        """The reference's ``SpeakerDiarizer`` whose embeddings come from ``scheduler.embed`` (``wl_spk_embed`` on the
        scheduler's engine, batched with every other segment of the round).  ``identify_speaker``, ``enroll_speaker``,
        ``reset`` and the clustering are the reference's own methods."""

        def __init__(self, scheduler, similarity_threshold=0.55, max_speakers=10,
                     embedding_model=DEFAULT_EMBEDDING_MODEL, hf_token=None, speaker_names=None):
            super().__init__(similarity_threshold=similarity_threshold, max_speakers=max_speakers,
                             embedding_model=embedding_model, hf_token=hf_token, speaker_names=speaker_names)
            self.scheduler = scheduler

        @classmethod
        def replacing(cls, diarizer, scheduler) -> "DeviceSpeakerDiarizer":
            """A device diarizer with ``diarizer``'s settings and state (threshold, ``max_speakers``, names, enrolled
            and running speakers)."""
            new = cls(scheduler, similarity_threshold=diarizer.similarity_threshold, max_speakers=diarizer.max_speakers,
                      embedding_model=getattr(diarizer, "_embedding_model_name", DEFAULT_EMBEDDING_MODEL),
                      hf_token=getattr(diarizer, "_hf_token", None), speaker_names=diarizer.speaker_names)
            new.speakers = dict(diarizer.speakers)
            new._speaker_count = diarizer._speaker_count
            return new

        def _load_model(self):
            pass

        def _compute_embedding(self, audio_np, sample_rate=16000):
            if len(audio_np) < sample_rate * 0.3:
                return None
            if sample_rate != SAMPLING_RATE:
                raise ValueError(f"the speaker embedding runs at {SAMPLING_RATE} Hz, not {sample_rate}")
            request = self.scheduler.embed(np.asarray(audio_np, dtype=np.float32).reshape(-1))
            embedding = request.wait()
            return embedding / np.linalg.norm(embedding)

else:

    class DeviceSpeakerDiarizer:  # type: ignore
        def __init__(self, *a, **k):
            raise ImportError("whisper_live (the reference package) is not importable: DeviceSpeakerDiarizer subclasses "
                              f"whisper_live.diarization.SpeakerDiarizer ({_IMPORT_ERROR})")
