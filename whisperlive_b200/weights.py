"""Weight containers for the engine: HF ``WhisperForConditionalGeneration`` tensor
names are the canonical key space (so openai/whisper-* safetensors load without
renaming; CT2 ``model.bin`` needs a name map -- SURVEY.md §8(f) N1).

There are no checkpoints in the build container, so tests and bench.py use
``random_init`` (seeded, fp16-representable values) of the named architecture.
"""
from __future__ import annotations

import json
import math
import os
import pickle
import re
import struct
from typing import Dict, Iterator, List, Optional, Tuple

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


# ------------------------------------------------------------------------------------------ checkpoints on disk
# A reader yields ``(canonical name, array as stored, scale or None)`` one tensor at a time, so a load never holds
# more than the tensor being uploaded: float32 / float16 arrays, bfloat16 as its uint16 bit patterns (numpy has no
# bfloat16, and no checkpoint stores uint16 weights), int8 with one scale per leading-dimension row.
BF16 = np.dtype(np.uint16)


def to_float32(a: np.ndarray, scale: Optional[np.ndarray] = None) -> np.ndarray:
    """The fp32 value of a stored array (a new array): what wl_load_tensor_typed converts on the device before it
    rounds to fp16.  int8 is ``q / scale[row]`` in fp32."""
    if a.dtype == BF16:
        return (a.astype(np.uint32) << 16).view(np.float32)
    if a.dtype == np.int8:
        s = np.asarray(scale).reshape(-1)
        s = to_float32(s) if s.dtype == BF16 else s.astype(np.float32)
        return a.astype(np.float32) / s.reshape((-1,) + (1,) * (a.ndim - 1))
    return np.array(a, dtype=np.float32, copy=True)


def _canonical(key: str) -> str:
    return key if key.startswith("model.") else "model." + key


def _st_header(path: str) -> Dict[str, dict]:
    """The JSON header of a .safetensors file (name -> dtype, shape, offsets), read without touching the payload."""
    with open(path, "rb") as f:
        (n,) = struct.unpack("<Q", f.read(8))
        head = json.loads(f.read(n))
    head.pop("__metadata__", None)
    return head


def _torch_np(t: torch.Tensor, name: str) -> np.ndarray:
    if t.dtype == torch.bfloat16:
        return t.view(torch.int16).numpy().view(BF16)
    if t.dtype in (torch.float32, torch.float16):
        return t.numpy()
    raise ValueError(f"{name}: dtype {t.dtype} is not float32, float16 or bfloat16")


class HFCheckpoint:
    """A Hugging Face Whisper checkpoint: ``model.safetensors``, its sharded index (``model.safetensors.index.json`` +
    shards), ``pytorch_model.bin`` or its sharded index, in fp32 / fp16 / bf16, keys with or without ``model.``.
    Safetensors wins when both formats are present, as in transformers.  Shapes come from the headers; tensors are
    memory-mapped (``safe_open`` / ``torch.load(mmap=True)``) and yielded one at a time, never inflated."""

    def __init__(self, path: str):
        self.path = path
        files = {}
        for index, single, kind in (("model.safetensors.index.json", "model.safetensors", "safetensors"),
                                    ("pytorch_model.bin.index.json", "pytorch_model.bin", "bin")):
            if os.path.exists(os.path.join(path, index)):
                with open(os.path.join(path, index), "r", encoding="utf-8") as f:
                    weight_map = json.load(f)["weight_map"]
                for shard in sorted(set(weight_map.values())):
                    if not os.path.exists(os.path.join(path, shard)):
                        raise FileNotFoundError(f"{path}: shard {shard!r} listed in {index} is missing")
                files = dict(weight_map)
                self.layout = kind + "-sharded"
                break
            if os.path.exists(os.path.join(path, single)):
                files = None
                self.layout = kind
                self._single = single
                break
        else:
            raise FileNotFoundError(f"{path}: no model.safetensors, pytorch_model.bin or sharded index")
        self.kind = self.layout.split("-")[0]
        shards = sorted(set(files.values())) if files is not None else [self._single]
        self._stored: Dict[str, Tuple[str, Tuple[int, ...], str]] = {}   # stored key -> (shard, shape, dtype)
        for shard in shards:
            p = os.path.join(path, shard)
            if self.kind == "safetensors":
                for k, v in _st_header(p).items():
                    self._stored[k] = (shard, tuple(v["shape"]), v["dtype"])
            else:
                sd = torch.load(p, map_location="cpu", weights_only=True, mmap=True)
                for k, v in sd.items():
                    self._stored[k] = (shard, tuple(v.shape), str(v.dtype).replace("torch.", ""))
        if files is not None:
            missing = sorted(k for k in files if k not in self._stored)
            if missing:
                raise ValueError(f"{path}: {missing[0]!r} is listed in the index but not in shard {files[missing[0]]!r}")
        ok = {"F32", "F16", "BF16", "float32", "float16", "bfloat16"}
        for k, (shard, _, dt) in self._stored.items():
            if dt not in ok:
                raise ValueError(f"{path}/{shard}: {k!r} has dtype {dt}, not float32, float16 or bfloat16")
        self.shapes = {_canonical(k): v[1] for k, v in self._stored.items() if k != "proj_out.weight"}

    def _open(self, shard: str):
        p = os.path.join(self.path, shard)
        if self.kind == "safetensors":
            from safetensors import safe_open
            return safe_open(p, framework="pt")
        return torch.load(p, map_location="cpu", weights_only=True, mmap=True)

    def _get(self, handle, key: str) -> torch.Tensor:
        # a .bin shard is one dict of mapped tensors: each leaves it as it is handed on, so none outlives its upload
        return handle.get_tensor(key) if self.kind == "safetensors" else handle.pop(key)

    def _check_tied_head(self) -> None:
        """``proj_out.weight`` is dropped only when it equals the embedding: the engine ties the two."""
        if "proj_out.weight" not in self._stored:
            return
        emb_key = next(k for k in self._stored if _canonical(k) == "model.decoder.embed_tokens.weight")
        head = self._get(self._open(self._stored["proj_out.weight"][0]), "proj_out.weight")
        emb = self._get(self._open(self._stored[emb_key][0]), emb_key)
        if head.shape != emb.shape or not torch.equal(head, emb):
            raise ValueError(f"{self.path}: proj_out.weight differs from model.decoder.embed_tokens.weight; the engine "
                             f"ties the output head to the embedding and cannot load an untied head")

    def tensors(self) -> Iterator[Tuple[str, np.ndarray, None]]:
        self._check_tied_head()
        by_shard: Dict[str, List[str]] = {}
        for k, (shard, _, _) in self._stored.items():
            if k != "proj_out.weight":
                by_shard.setdefault(shard, []).append(k)
        for shard in sorted(by_shard):
            handle = self._open(shard)
            for k in by_shard[shard]:
                yield _canonical(k), _torch_np(self._get(handle, k), k), None
            del handle


def _read_json(path: str) -> dict:
    if not os.path.isfile(path):
        return {}
    with open(path, "r", encoding="utf-8") as f:
        return json.load(f)


def open_checkpoint(path: str):
    """The checkpoint of a model directory, checked before anything is read past the headers: a Hugging Face layout
    (``HFCheckpoint``) or a CTranslate2 ``model.bin`` (``ct2_format.Ct2Checkpoint``).  Raises ValueError naming what
    the engine cannot run: positions other than 1500 / 448, a head dimension other than 64."""
    names = ("model.safetensors.index.json", "model.safetensors", "pytorch_model.bin.index.json", "pytorch_model.bin")
    if any(os.path.exists(os.path.join(path, n)) for n in names):
        ckpt = HFCheckpoint(path)
        cfg = _read_json(os.path.join(path, "config.json"))
        for key, want in (("max_source_positions", 1500), ("max_target_positions", 448)):
            if key in cfg and int(cfg[key]) != want:
                raise ValueError(f"{path}: config.json {key} = {cfg[key]}; the engine runs {want} only")
        for key in ("encoder_attention_heads", "decoder_attention_heads"):
            if key in cfg and "d_model" in cfg and int(cfg["d_model"]) != 64 * int(cfg[key]):
                raise ValueError(f"{path}: config.json d_model {cfg['d_model']} / {key} {cfg[key]} is a head dimension "
                                 f"other than 64; the engine runs 64 only")
    elif os.path.exists(os.path.join(path, "model.bin")):
        from .ct2_format import Ct2Checkpoint
        ckpt = Ct2Checkpoint(path)
    else:
        raise FileNotFoundError(f"{path}: no model.safetensors, pytorch_model.bin (single or sharded) or model.bin")
    for name, want in (("model.encoder.embed_positions.weight", 1500), ("model.decoder.embed_positions.weight", 448)):
        got = ckpt.shapes.get(name)
        if got is None:
            raise ValueError(f"{path}: {name} is missing")
        if got[0] != want:
            raise ValueError(f"{path}: {name} has {got[0]} positions; the engine runs {want} only")
    return ckpt


def checkpoint_dims(path: str, name: str = "custom") -> Optional[WhisperDims]:
    """The shapes of a model directory from its headers alone, or None when it has no readable header."""
    try:
        return infer_dims(open_checkpoint(path).shapes, name)
    except (OSError, ValueError, KeyError, RuntimeError, EOFError, struct.error, pickle.UnpicklingError):
        return None   # what a malformed file raises (torch.load of a legacy or broken pytorch_model.bin included)


def model_metadata(path: str) -> Dict[str, object]:
    """What the engine's callers read from a CTranslate2 ``config.json``, for any model directory: the file itself
    next to a CT2 ``model.bin``; for a Hugging Face directory what ``TransformersConverter`` writes into it.  That is a
    recalled upstream rule (ctranslate2 ``converters/transformers.py``, the Whisper loader's ``set_config``, restated
    from memory; tests/golden/capture_ct2_convert.py records real conversions, one with a generation config that lacks
    some keys): the keys come from ``generation_config.json`` when it exists, else from ``config.json`` --
    ``alignment_heads`` as given, ``suppress_ids`` = ``suppress_tokens``, ``suppress_ids_begin`` =
    ``begin_suppress_tokens``, ``lang_ids`` = the sorted values of ``lang_to_id``.  Keys the chosen file does not give
    are omitted (the converter's default heads, the upper half of the layers, are the engine's default)."""
    from .ct2_format import read_ct2_config
    hf = ("model.safetensors.index.json", "model.safetensors", "pytorch_model.bin.index.json", "pytorch_model.bin")
    if not any(os.path.exists(os.path.join(path, n)) for n in hf):
        return read_ct2_config(path)
    src = _read_json(os.path.join(path, "generation_config.json")) or _read_json(os.path.join(path, "config.json"))
    out: Dict[str, object] = {}
    if src.get("alignment_heads"):
        out["alignment_heads"] = [(int(a), int(b)) for a, b in src["alignment_heads"]]
    for dst, key in (("suppress_ids", "suppress_tokens"), ("suppress_ids_begin", "begin_suppress_tokens")):
        if src.get(key) is not None:
            out[dst] = [int(x) for x in src[key]]
    if src.get("lang_to_id"):
        out["lang_ids"] = sorted(int(x) for x in src["lang_to_id"].values())
    return out


def load_model_dir(path: str) -> Dict[str, torch.Tensor]:
    """Every tensor of a model directory (any layout ``open_checkpoint`` reads) as the canonical fp32 dict."""
    return {name: torch.from_numpy(to_float32(a, scale)) for name, a, scale in open_checkpoint(path).tensors()}


_HF_WEIGHTS = re.compile(r"^(model(-\d+-of-\d+)?\.safetensors|model\.safetensors\.index\.json)$")
_BIN_WEIGHTS = re.compile(r"^(pytorch_model(-\d+-of-\d+)?\.bin|pytorch_model\.bin\.index\.json)$")
_HUB_META = ["config.json", "generation_config.json", "preprocessor_config.json", "tokenizer.json", "vocabulary.*"]


def hub_allow_patterns(files: Optional[List[str]]) -> List[str]:
    """The files of a hub repository to fetch, given its file list: the metadata, and ONE copy of the weights --
    safetensors (single or sharded) before ``pytorch_model*.bin`` before a CTranslate2 ``model.bin``, the order
    ``open_checkpoint`` reads them in.  ``files=None`` (the list is unknown, e.g. offline): every pattern, which only
    matters for finding a snapshot already on disk."""
    if files is None:
        return _HUB_META + ["model.bin", "model*.safetensors", "model.safetensors.index.json", "pytorch_model*.bin",
                            "pytorch_model.bin.index.json"]
    for pattern in (_HF_WEIGHTS, _BIN_WEIGHTS):
        weights = sorted(f for f in files if pattern.match(f))
        if weights:
            return _HUB_META + weights
    return _HUB_META + (["model.bin"] if "model.bin" in files else [])


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
    # Downloads go by the repository's file list, so only one copy of the weights is fetched.  Without the list
    # (local_files_only, or listing failed: offline) nothing is downloaded; a snapshot already on disk still resolves.
    first: Optional[BaseException] = None
    if not local_files_only:
        try:
            files = huggingface_hub.list_repo_files(repo)
            return huggingface_hub.snapshot_download(repo, cache_dir=download_root, allow_patterns=hub_allow_patterns(files))
        except Exception as e:
            first = e
    try:
        return huggingface_hub.snapshot_download(repo, cache_dir=download_root, local_files_only=True,
                                                 allow_patterns=hub_allow_patterns(None))
    except Exception as e:
        first = first or e
        raise FileNotFoundError(
            f"no checkpoint for {name!r}: not a local directory and the hub snapshot {repo!r} is unavailable "
            f"({type(first).__name__}: {first}).  Pass a model directory (model.safetensors or model.bin + "
            f"tokenizer.json), or weights='random' for a seeded random-init engine (bench/tests only).") from first


def infer_dims(weights, name: str = "custom") -> WhisperDims:
    """Shapes of a tensor dict, or of a ``{name: shape}`` table (a checkpoint's ``shapes``)."""
    shapes = {k: (v if isinstance(v, tuple) else tuple(v.shape)) for k, v in weights.items()}
    d, n_mels = shapes["model.encoder.conv1.weight"][:2]
    vocab = shapes["model.decoder.embed_tokens.weight"][0]
    enc_layers = 1 + max(int(k.split(".")[3]) for k in shapes if k.startswith("model.encoder.layers."))
    dec_layers = 1 + max(int(k.split(".")[3]) for k in shapes if k.startswith("model.decoder.layers."))
    return WhisperDims(name, d, d // 64, enc_layers, dec_layers, n_mels, vocab)


def to_numpy_f16(weights: Dict[str, torch.Tensor]) -> Dict[str, np.ndarray]:
    return {k: v.half().numpy() for k, v in weights.items()}
