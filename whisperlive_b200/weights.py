"""Weight containers for the engine: HF ``WhisperForConditionalGeneration`` tensor
names are the canonical key space (so openai/whisper-* safetensors load without
renaming; CT2 ``model.bin`` needs a name map -- SURVEY.md §8(f) N1).

There are no checkpoints in the build container, so tests and bench.py use
``random_init`` (seeded, fp16-representable values) of the named architecture.
"""
from __future__ import annotations

import math
import os
from typing import Dict

import numpy as np
import torch

from .config import WhisperDims


def sinusoids(length: int, channels: int, max_timescale: float = 10000.0) -> torch.Tensor:
    """Whisper encoder positional table (stored as a weight in released checkpoints)."""
    log_inc = math.log(max_timescale) / (channels // 2 - 1)
    inv = torch.exp(-log_inc * torch.arange(channels // 2, dtype=torch.float32))
    t = torch.arange(length, dtype=torch.float32)[:, None] * inv[None, :]
    return torch.cat([t.sin(), t.cos()], dim=1)


def _special_ids(dims: WhisperDims):
    """(eot, timestamp_begin) from the vocabulary size (SURVEY.md A.2)."""
    if not dims.multilingual:
        return 50256, 50363
    n_lang = dims.num_languages
    eot = 50257
    ts_begin = 50258 + 1 + n_lang + 6  # sot, langs, translate, transcribe, sot_lm, sot_prev, nospeech, notimestamps
    return eot, ts_begin


def random_init(dims: WhisperDims, seed: int = 0, eot_scale: float = 2.5, ts_scale: float = 1.25,
                logit_std: float = 3.0, qk_gain: float = 2.5) -> Dict[str, torch.Tensor]:
    """Seeded random weights, values rounded through fp16 so an fp32 oracle and the
    fp16 engine see identical parameters.  Scales are chosen so that activations
    stay O(1), next-token distributions are peaked (logit std ~3) and EOT /
    timestamp tokens occur (their embedding rows are scaled up)."""
    g = torch.Generator().manual_seed(seed)
    d, ff = dims.d_model, dims.d_ff
    w: Dict[str, torch.Tensor] = {}

    def normal(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    def linear(prefix, out_f, in_f, bias=True, gain=1.0):
        w[prefix + ".weight"] = normal(out_f, in_f, std=gain / math.sqrt(in_f))
        if bias:
            w[prefix + ".bias"] = normal(out_f, std=0.02)

    def lnorm(prefix):
        w[prefix + ".weight"] = 1.0 + normal(d, std=0.1)
        w[prefix + ".bias"] = normal(d, std=0.02)

    def attn(prefix):
        linear(prefix + ".q_proj", d, d, gain=qk_gain)   # peaked attention -> audio/position dependent outputs
        linear(prefix + ".k_proj", d, d, bias=False, gain=qk_gain)
        linear(prefix + ".v_proj", d, d)
        linear(prefix + ".out_proj", d, d)

    enc = "model.encoder"
    w[enc + ".conv1.weight"] = normal(d, dims.n_mels, 3, std=1.0 / math.sqrt(3 * dims.n_mels))
    w[enc + ".conv1.bias"] = normal(d, std=0.02)
    w[enc + ".conv2.weight"] = normal(d, d, 3, std=1.0 / math.sqrt(3 * d))
    w[enc + ".conv2.bias"] = normal(d, std=0.02)
    w[enc + ".embed_positions.weight"] = sinusoids(dims.n_audio_ctx, d)
    for i in range(dims.enc_layers):
        p = f"{enc}.layers.{i}"
        attn(p + ".self_attn")
        lnorm(p + ".self_attn_layer_norm")
        linear(p + ".fc1", ff, d)
        linear(p + ".fc2", d, ff)
        lnorm(p + ".final_layer_norm")
    lnorm(enc + ".layer_norm")

    dec = "model.decoder"
    emb = normal(dims.vocab, d, std=logit_std / math.sqrt(d))
    eot, ts_begin = _special_ids(dims)
    emb[eot] *= eot_scale
    emb[ts_begin:] *= ts_scale
    w[dec + ".embed_tokens.weight"] = emb
    w[dec + ".embed_positions.weight"] = normal(dims.n_text_ctx, d, std=1.5 * logit_std / math.sqrt(d))
    for i in range(dims.dec_layers):
        p = f"{dec}.layers.{i}"
        attn(p + ".self_attn")
        lnorm(p + ".self_attn_layer_norm")
        attn(p + ".encoder_attn")
        lnorm(p + ".encoder_attn_layer_norm")
        linear(p + ".fc1", ff, d)
        linear(p + ".fc2", d, ff)
        lnorm(p + ".final_layer_norm")
    lnorm(dec + ".layer_norm")
    return {k: v.half().float().contiguous() for k, v in w.items()}


def load_safetensors(path: str) -> Dict[str, torch.Tensor]:
    """Read an HF ``model.safetensors`` (openai/whisper-*) into the canonical dict."""
    from safetensors.torch import load_file

    if os.path.isdir(path):
        path = os.path.join(path, "model.safetensors")
    sd = load_file(path)
    out = {}
    for k, v in sd.items():
        if k == "proj_out.weight":
            continue  # tied to model.decoder.embed_tokens.weight
        out[k if k.startswith("model.") else "model." + k] = v.float().contiguous()
    return out


def load_model_dir(path: str) -> Dict[str, torch.Tensor]:
    """A model directory in either format the reference's users have on disk: HF ``model.safetensors``
    (openai/whisper-*) or CTranslate2 ``model.bin`` (Systran/faster-whisper-*; ct2_format.py)."""
    if os.path.exists(os.path.join(path, "model.safetensors")):
        return load_safetensors(path)
    if os.path.exists(os.path.join(path, "model.bin")):
        from .ct2_format import load_ct2_model_bin
        return load_ct2_model_bin(path)
    raise FileNotFoundError(f"{path}: neither model.safetensors nor model.bin")


# Size name -> hub repository of its CTranslate2 conversion, for the sizes whose repository is not
# ``Systran/faster-whisper-<size>``.  Like faster-whisper's ``utils._MODELS``, which this table is recalled from:
# faster-whisper is not a dependency of this project, so the table was not read from it.
HUB_REPOS = {
    "distil-small.en": "Systran/faster-distil-whisper-small.en",
    "distil-medium.en": "Systran/faster-distil-whisper-medium.en",
    "distil-large-v2": "Systran/faster-distil-whisper-large-v2",
    "distil-large-v3": "Systran/faster-distil-whisper-large-v3",
    "large-v3-turbo": "mobiuslabsgmbh/faster-whisper-large-v3-turbo",
    "turbo": "mobiuslabsgmbh/faster-whisper-large-v3-turbo",
}


def hub_repo(name: str) -> str:
    """Hub repository a size name or hub id resolves to: a hub id (``owner/repo``) as given, a size in ``HUB_REPOS``
    through the table, any other size as ``Systran/faster-whisper-<size>``."""
    name = str(name)
    if "/" in name:
        return name
    return HUB_REPOS.get(name, f"Systran/faster-whisper-{name}")


def resolve_model_dir(model_size_or_path: str, download_root=None, local_files_only: bool = False) -> str:
    """Directory holding the checkpoint + tokenizer.json for a path, a size name or a hub id.
    Mirrors the reference's resolution order (faster_whisper_backend.py:133-178): local directory first,
    then the hub snapshot of ``hub_repo(size)`` (CT2 format, what ``download_model`` fetches).
    Raises FileNotFoundError with the reason instead of falling back to anything."""
    if isinstance(model_size_or_path, str) and os.path.isdir(model_size_or_path):
        return model_size_or_path
    name = str(model_size_or_path)
    repo = hub_repo(name)
    try:
        import huggingface_hub
    except Exception as e:
        raise FileNotFoundError(f"{name!r} is not a model directory and huggingface_hub is not importable ({e})") from e
    allow = ["config.json", "preprocessor_config.json", "model.bin", "model.safetensors", "tokenizer.json", "vocabulary.*"]
    try:
        return huggingface_hub.snapshot_download(repo, cache_dir=download_root, local_files_only=local_files_only,
                                                 allow_patterns=allow)
    except Exception as first:
        try:   # offline / no network: a previously downloaded snapshot still resolves
            return huggingface_hub.snapshot_download(repo, cache_dir=download_root, local_files_only=True, allow_patterns=allow)
        except Exception:
            raise FileNotFoundError(
                f"no checkpoint for {name!r}: not a local directory and the hub snapshot {repo!r} is unavailable "
                f"({type(first).__name__}: {first}).  Pass a model directory (model.safetensors or model.bin + "
                f"tokenizer.json), or weights='random' for a seeded random-init engine (bench/tests only).") from first


def infer_dims(weights: Dict[str, torch.Tensor], name: str = "custom") -> WhisperDims:
    d = weights["model.encoder.conv1.weight"].shape[0]
    n_mels = weights["model.encoder.conv1.weight"].shape[1]
    vocab = weights["model.decoder.embed_tokens.weight"].shape[0]
    enc_layers = 1 + max(int(k.split(".")[3]) for k in weights if k.startswith("model.encoder.layers."))
    dec_layers = 1 + max(int(k.split(".")[3]) for k in weights if k.startswith("model.decoder.layers."))
    return WhisperDims(name, d, d // 64, enc_layers, dec_layers, n_mels, vocab)


def to_numpy_f16(weights: Dict[str, torch.Tensor]) -> Dict[str, np.ndarray]:
    return {k: v.half().numpy() for k, v in weights.items()}
