"""Translation on the device: the M2M100 (SMaLL-100) model behind WhisperLive's ``ServeClientTranslation``.

The reference builds one ``ServeClientTranslation`` per connection that enables translation; each loads its own
``M2M100ForConditionalGeneration`` and runs ``generate()`` for one committed segment at a time.  Here one process-wide
``TranslationWorker`` owns one device context (``wl_mt_*``) and answers every pending segment of every connection with
one ``wl_mt_translate`` call.  ``DeviceTranslationClient`` keeps the reference client's behaviour and protocol.

Recalled facts (transformers 5.5.0 ``models/m2m_100``, ``generation/utils.py``; ``tokenization_small100.py``):
  * shared embedding x sqrt(d) when ``scale_embedding``; sinusoidal positions ``[sin | cos]`` with log(10000)/(half-1),
    the pad row zero, real tokens from padding_idx + 1 (the decoder: 2 + past length);
  * pre-LN encoder / decoder layers, biased q/k/v/out projections, scaling head_dim^-0.5, ReLU FFN, a final LayerNorm on
    both sides; ``lm_head`` tied to ``shared``, no bias;
  * the source is ``[target-language id] + pieces + [</s>]``; the decoder starts from ``decoder_start_token_id``.

Selected with ``WLB200_TRANSLATE=device`` (default ``cpu``: the reference's own object).
"""
from __future__ import annotations

import ctypes as C
import json
import logging
import math
import os
import queue
import threading
from dataclasses import dataclass

import numpy as np

T_MAX = 448                 # decoder positions of the engine (decoder start token included)
MAX_BEAMS = 8
DEFAULT_MODEL = "alirezamsh/small100"

FAIRSEQ_LANGUAGE_CODES = [
    "af", "am", "ar", "ast", "az", "ba", "be", "bg", "bn", "br", "bs", "ca", "ceb", "cs", "cy", "da", "de", "el", "en",
    "es", "et", "fa", "ff", "fi", "fr", "fy", "ga", "gd", "gl", "gu", "ha", "he", "hi", "hr", "ht", "hu", "hy", "id", "ig",
    "ilo", "is", "it", "ja", "jv", "ka", "kk", "km", "kn", "ko", "lb", "lg", "ln", "lo", "lt", "lv", "mg", "mk", "ml",
    "mn", "mr", "ms", "my", "ne", "nl", "no", "ns", "oc", "or", "pa", "pl", "ps", "pt", "ro", "ru", "sd", "si", "sk", "sl",
    "so", "sq", "sr", "ss", "su", "sv", "sw", "ta", "th", "tl", "tn", "tr", "uk", "ur", "uz", "vi", "wo", "xh", "yi", "yo",
    "zh", "zu"]


def translate_mode() -> str:
    mode = os.environ.get("WLB200_TRANSLATE", "cpu")
    if mode not in ("cpu", "device"):
        raise ValueError(f"WLB200_TRANSLATE={mode!r}: expected 'cpu' or 'device'")
    return mode


# ------------------------------------------------------------------------------------------------ model settings
@dataclass(frozen=True)
class MtConfig:
    d_model: int
    n_heads: int
    enc_layers: int
    dec_layers: int
    ffn: int
    vocab: int
    max_positions: int
    pad_id: int = 1
    scale_embedding: bool = True

    @property
    def embed_scale(self) -> float:
        return math.sqrt(self.d_model) if self.scale_embedding else 1.0


SMALL100_SHAPE = dict(d_model=1024, n_heads=16, enc_layers=12, dec_layers=3, ffn=4096, vocab=128112, max_positions=1024)


def config_from_json(cfg: dict) -> MtConfig:
    """MtConfig from a Hugging Face M2M100 ``config.json``; anything the engine does not implement raises by name."""
    def get(k, default=None):
        if k not in cfg and default is None:
            raise ValueError(f"config.json: missing '{k}'")
        return cfg.get(k, default)
    if get("encoder_attention_heads") != get("decoder_attention_heads"):
        raise ValueError("config.json: encoder_attention_heads != decoder_attention_heads is not supported")
    if get("encoder_ffn_dim") != get("decoder_ffn_dim"):
        raise ValueError("config.json: encoder_ffn_dim != decoder_ffn_dim is not supported")
    act = cfg.get("activation_function", "relu")
    if act != "relu":
        raise ValueError(f"config.json: activation_function={act!r} is not supported (relu)")
    c = MtConfig(d_model=int(get("d_model")), n_heads=int(get("encoder_attention_heads")), enc_layers=int(get("encoder_layers")),
                 dec_layers=int(get("decoder_layers")), ffn=int(get("encoder_ffn_dim")), vocab=int(get("vocab_size")),
                 max_positions=int(get("max_position_embeddings")), pad_id=int(cfg.get("pad_token_id", 1)),
                 scale_embedding=bool(cfg.get("scale_embedding", False)))
    if c.d_model != 64 * c.n_heads:
        raise ValueError(f"config.json: head dim {c.d_model // max(c.n_heads, 1)} is not supported (64)")
    return c


@dataclass(frozen=True)
class GenSettings:
    num_beams: int = 1
    max_length: int = 20            # decoder start token included
    length_penalty: float = 1.0
    early_stopping: object = False  # True / False / "never"
    decoder_start_token_id: int = 2
    bos_token_id: int = 0
    eos_token_id: int = 2
    pad_token_id: int = 1
    forced_bos_token_id: int | None = None
    forced_eos_token_id: int | None = None

    @property
    def early_stopping_code(self) -> int:
        return {False: 0, True: 1, "never": 2}[self.early_stopping]


# GenerationConfig attributes the engine does not implement, at their Hugging Face defaults
_UNSUPPORTED_DEFAULTS = {
    "do_sample": False, "temperature": 1.0, "top_k": 50, "top_p": 1.0, "typical_p": 1.0, "epsilon_cutoff": 0.0,
    "eta_cutoff": 0.0, "min_p": None, "repetition_penalty": 1.0, "encoder_repetition_penalty": 1.0,
    "no_repeat_ngram_size": 0, "encoder_no_repeat_ngram_size": 0, "bad_words_ids": None, "force_words_ids": None,
    "min_length": 0, "min_new_tokens": None, "num_beam_groups": 1, "diversity_penalty": 0.0, "constraints": None,
    "renormalize_logits": False, "suppress_tokens": None, "begin_suppress_tokens": None, "sequence_bias": None,
    "exponential_decay_length_penalty": None, "guidance_scale": None, "num_return_sequences": 1, "penalty_alpha": None,
    "max_time": None, "stop_strings": None, "low_memory": None, "remove_invalid_values": False,
}
_SUPPORTED = ("num_beams", "max_length", "max_new_tokens", "length_penalty", "early_stopping", "decoder_start_token_id",
              "bos_token_id", "eos_token_id", "pad_token_id", "forced_bos_token_id", "forced_eos_token_id")


def generation_settings(gen: dict, cfg: dict | None = None, max_positions: int | None = None) -> GenSettings:
    """Settings from ``generation_config.json`` (``gen``), else from ``config.json`` the way GenerationConfig derives
    them; any other setting away from its default raises and names it.  ``max_positions``: the decoder's positions
    must stay inside the model's position table (max_length <= max_positions + 1)."""
    src = dict(gen) if gen else {k: v for k, v in (cfg or {}).items() if k in _SUPPORTED or k in _UNSUPPORTED_DEFAULTS}
    for k, dflt in _UNSUPPORTED_DEFAULTS.items():
        if k in src and src[k] != dflt and not (k == "num_return_sequences" and src[k] in (None, 1)):
            raise ValueError(f"generation setting '{k}' = {src[k]!r} is not supported by the device translator")
    eos = src.get("eos_token_id", 2)
    if isinstance(eos, list):
        if len(eos) != 1:
            raise ValueError("generation setting 'eos_token_id': one EOS token is supported")
        eos = eos[0]
    num_beams = int(src.get("num_beams", 1) or 1)
    if not 1 <= num_beams <= MAX_BEAMS:
        raise ValueError(f"generation setting 'num_beams' = {num_beams}: supported up to {MAX_BEAMS}")
    max_length = int(src.get("max_length", 20) or 20)
    if src.get("max_new_tokens") is not None:
        max_length = int(src["max_new_tokens"]) + 1           # generate counts the decoder start token
    if max_length > T_MAX:
        raise ValueError(f"generation setting 'max_length' = {max_length} exceeds the decoder limit of {T_MAX} positions")
    if max_positions is not None and max_length > max_positions + 1:
        raise ValueError(f"generation setting 'max_length' = {max_length} exceeds the position table "
                         f"(max_position_embeddings {max_positions} + 1)")
    es = src.get("early_stopping", False)
    if es not in (True, False, "never"):
        raise ValueError(f"generation setting 'early_stopping' = {es!r} is not supported")
    start = src.get("decoder_start_token_id")
    start = eos if start is None else start
    return GenSettings(num_beams=num_beams, max_length=max_length, length_penalty=float(src.get("length_penalty", 1.0)),
                       early_stopping=es, decoder_start_token_id=int(start), bos_token_id=int(src.get("bos_token_id", 0) or 0),
                       eos_token_id=int(eos), pad_token_id=int(src.get("pad_token_id", 1) if src.get("pad_token_id") is not None else 1),
                       forced_bos_token_id=src.get("forced_bos_token_id"), forced_eos_token_id=src.get("forced_eos_token_id"))


# ------------------------------------------------------------------------------------------------ checkpoint
def checkpoint_shapes(cfg: MtConfig) -> dict:
    """Hugging Face names and shapes of every tensor the engine reads."""
    d, f = cfg.d_model, cfg.ffn
    out = {"model.shared.weight": (cfg.vocab, d)}
    att = ("q_proj", "k_proj", "v_proj", "out_proj")
    for side, n, attns, lns in (("encoder", cfg.enc_layers, ("self_attn",), ("self_attn_layer_norm", "final_layer_norm")),
                                ("decoder", cfg.dec_layers, ("self_attn", "encoder_attn"),
                                 ("self_attn_layer_norm", "encoder_attn_layer_norm", "final_layer_norm"))):
        for l in range(n):
            p = f"model.{side}.layers.{l}."
            for a in attns:
                for proj in att:
                    out[p + f"{a}.{proj}.weight"] = (d, d)
                    out[p + f"{a}.{proj}.bias"] = (d,)
            for ln in lns:
                out[p + f"{ln}.weight"] = (d,)
                out[p + f"{ln}.bias"] = (d,)
            out[p + "fc1.weight"] = (f, d)
            out[p + "fc1.bias"] = (f,)
            out[p + "fc2.weight"] = (d, f)
            out[p + "fc2.bias"] = (d,)
        out[f"model.{side}.layer_norm.weight"] = (d,)
        out[f"model.{side}.layer_norm.bias"] = (d,)
    return out


def read_checkpoint(path: str, cfg: MtConfig) -> dict:
    """float32 numpy arrays by Hugging Face name from ``pytorch_model.bin`` (torch.load, weights_only) or
    ``model.safetensors`` (a file or a snapshot directory).  The tied ``lm_head`` may be absent or equal to ``shared``;
    the embeddings may be stored under encoder / decoder ``embed_tokens``.  A missing tensor, a wrong shape or a
    non-float dtype raises by name."""
    import torch
    if os.path.isdir(path):
        for fn in ("model.safetensors", "pytorch_model.bin"):
            if os.path.exists(os.path.join(path, fn)):
                path = os.path.join(path, fn)
                break
        else:
            raise FileNotFoundError(f"{path}: no model.safetensors or pytorch_model.bin")
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        sd = load_file(path)
    else:
        sd = torch.load(path, map_location="cpu", weights_only=True)
    sd = {k[len("module."):] if k.startswith("module.") else k: v for k, v in sd.items()}
    if "model.shared.weight" not in sd:
        for alt in ("model.encoder.embed_tokens.weight", "model.decoder.embed_tokens.weight", "lm_head.weight"):
            if alt in sd:
                sd["model.shared.weight"] = sd[alt]
                break
    out = {}
    for name, shape in checkpoint_shapes(cfg).items():
        if name not in sd:
            raise ValueError(f"checkpoint: missing tensor '{name}'")
        t = sd[name]
        if not t.is_floating_point():
            raise ValueError(f"checkpoint: tensor '{name}' has non-float dtype {t.dtype}")
        if tuple(t.shape) != shape:
            raise ValueError(f"checkpoint: tensor '{name}' has shape {tuple(t.shape)}, expected {shape}")
        out[name] = t.detach().to(torch.float32).numpy()
    if "lm_head.weight" in sd and not torch.equal(sd["lm_head.weight"].float(), sd["model.shared.weight"].float()):
        raise ValueError("checkpoint: 'lm_head.weight' differs from 'model.shared.weight' (the head must be tied)")
    return out


def random_checkpoint(cfg: MtConfig, seed: int) -> dict:
    """Random weights at ``cfg``'s shapes (tests and tools only): N(0, 0.02) matrices and embeddings like Hugging
    Face's init, zero pad row, small random biases, LayerNorms near identity."""
    rng = np.random.default_rng(seed)
    out = {}
    for name, shape in checkpoint_shapes(cfg).items():
        if "layer_norm" in name:
            base = 1.0 if name.endswith("weight") else 0.0
            out[name] = (base + 0.05 * rng.standard_normal(shape)).astype(np.float32)
        elif name.endswith("bias"):
            out[name] = (0.02 * rng.standard_normal(shape)).astype(np.float32)
        else:
            out[name] = (0.02 * rng.standard_normal(shape)).astype(np.float32)
    out["model.shared.weight"][cfg.pad_id] = 0.0
    return out


def position_table(cfg: MtConfig) -> np.ndarray:
    """The sinusoidal table [max_positions + 2][d] as M2M100SinusoidalPositionalEmbedding builds it (float32)."""
    import torch
    n, dim, half = cfg.max_positions + 2, cfg.d_model, cfg.d_model // 2
    emb = math.log(10000) / (half - 1)
    emb = torch.exp(torch.arange(half, dtype=torch.int64).float() * -emb)
    emb = torch.arange(n, dtype=torch.int64).float().unsqueeze(1) * emb.unsqueeze(0)
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=1).view(n, -1)
    if dim % 2 == 1:
        emb = torch.cat([emb, torch.zeros(n, 1)], dim=1)
    emb[cfg.pad_id, :] = 0
    return emb.numpy().astype(np.float32)


def engine_tensors(ck: dict, cfg: MtConfig) -> dict:
    """The engine's tensor names (include/wlb200.h): q/k/v fused, the decoder's cross K/V of every layer in one matrix."""
    out = {"shared": ck["model.shared.weight"], "positions": position_table(cfg)}
    cat = np.concatenate
    for side, tag, n in (("encoder", "enc", cfg.enc_layers), ("decoder", "dec", cfg.dec_layers)):
        for l in range(n):
            p, e = f"model.{side}.layers.{l}.", f"{tag}.{l}."
            sa = p + "self_attn."
            out[e + "qkv.w"] = cat([ck[sa + f"{x}_proj.weight"] for x in "qkv"])
            out[e + "qkv.b"] = cat([ck[sa + f"{x}_proj.bias"] for x in "qkv"])
            out[e + "out.w"], out[e + "out.b"] = ck[sa + "out_proj.weight"], ck[sa + "out_proj.bias"]
            lns = ("self_attn_layer_norm", "final_layer_norm") if tag == "enc" else \
                ("self_attn_layer_norm", "encoder_attn_layer_norm", "final_layer_norm")
            for i, ln in enumerate(lns):
                out[e + f"ln{i + 1}.w"], out[e + f"ln{i + 1}.b"] = ck[p + ln + ".weight"], ck[p + ln + ".bias"]
            for fc in ("fc1", "fc2"):
                out[e + fc + ".w"], out[e + fc + ".b"] = ck[p + fc + ".weight"], ck[p + fc + ".bias"]
            if tag == "dec":
                xa = p + "encoder_attn."
                out[e + "xq.w"], out[e + "xq.b"] = ck[xa + "q_proj.weight"], ck[xa + "q_proj.bias"]
                out[e + "xout.w"], out[e + "xout.b"] = ck[xa + "out_proj.weight"], ck[xa + "out_proj.bias"]
        out[f"{tag}.ln.w"], out[f"{tag}.ln.b"] = ck[f"model.{side}.layer_norm.weight"], ck[f"model.{side}.layer_norm.bias"]
    xa = [f"model.decoder.layers.{l}.encoder_attn." for l in range(cfg.dec_layers)]
    out["dec.xkv.w"] = cat([ck[p + f"{x}_proj.weight"] for p in xa for x in "kv"])
    out["dec.xkv.b"] = cat([ck[p + f"{x}_proj.bias"] for p in xa for x in "kv"])
    return out


def resolve_snapshot(path: str | None = None, model_name: str = DEFAULT_MODEL) -> str:
    """An explicit directory, then ``WLB200_MT_MODEL``, then a local Hugging Face snapshot of ``model_name``.  Never
    downloads and never substitutes another model."""
    for cand in (path, os.environ.get("WLB200_MT_MODEL")):
        if cand:
            if not os.path.isdir(cand):
                raise FileNotFoundError(f"translation model directory {cand!r} does not exist")
            return cand
    try:
        from huggingface_hub import snapshot_download
        return snapshot_download(model_name, local_files_only=True)
    except Exception as e:   # no hub package or no local snapshot
        raise FileNotFoundError(f"no local snapshot of {model_name!r}; set WLB200_MT_MODEL to a model directory ({e})") from e


def load_snapshot_settings(path: str) -> tuple[MtConfig, GenSettings]:
    with open(os.path.join(path, "config.json")) as f:
        cfg_json = json.load(f)
    gen_json = None
    gp = os.path.join(path, "generation_config.json")
    if os.path.exists(gp):
        with open(gp) as f:
            gen_json = json.load(f)
    cfg = config_from_json(cfg_json)
    return cfg, generation_settings(gen_json, cfg_json, cfg.max_positions)


def check_source_length(n: int, cfg: MtConfig) -> None:
    if n > cfg.max_positions - 2:
        raise ValueError(f"source of {n} tokens exceeds the limit of {cfg.max_positions - 2} (max_position_embeddings - 2)")


# ------------------------------------------------------------------------------------------------ tokenizer
class Small100Tokenizer:
    """SMaLL-100's tokenizer restated on ``sentencepiece`` + ``vocab.json``: pieces map through the vocabulary (an
    unknown piece to ``<unk>``); the 100 language tokens ``__xx__`` follow the vocabulary, then 8 made-up words; the
    source is ``[target-language id] + pieces + [</s>]``; decoding skips the special tokens and joins the pieces with
    ``sp_model.decode``."""

    def __init__(self, vocab_file: str, spm_file: str):
        import sentencepiece
        with open(vocab_file) as f:
            self.encoder = json.load(f)
        self.decoder = {v: k for k, v in self.encoder.items()}
        self.sp = sentencepiece.SentencePieceProcessor()
        self.sp.Load(spm_file)
        n = len(self.encoder)
        self.lang_id = {c: n + i for i, c in enumerate(FAIRSEQ_LANGUAGE_CODES)}
        self.id_lang = {v: f"__{k}__" for k, v in self.lang_id.items()}
        self.unk_id, self.eos_id = self.encoder["<unk>"], self.encoder["</s>"]
        # what skip_special_tokens drops under transformers 5 (pinned in tests/golden/translate_reference.json): BOS, EOS,
        # PAD, the language tokens, and the last made-up word, the id transformers registers for "<unk>" as an added
        # token; vocabulary <unk> (3) and the other made-up words stay and decode as sentencepiece's unknown piece
        self.special = {self.encoder[t] for t in ("<s>", "</s>", "<pad>") if t in self.encoder} | set(self.lang_id.values())
        self.special.add(n + len(FAIRSEQ_LANGUAGE_CODES) + 7)

    @classmethod
    def from_dir(cls, path: str) -> "Small100Tokenizer":
        return cls(os.path.join(path, "vocab.json"), os.path.join(path, "sentencepiece.bpe.model"))

    def encode(self, text: str, target_language: str) -> list[int]:
        if target_language not in self.lang_id:
            raise KeyError(target_language)
        pieces = self.sp.encode(text, out_type=str)
        return [self.lang_id[target_language]] + [self.encoder.get(p, self.unk_id) for p in pieces] + [self.eos_id]

    def decode(self, ids) -> str:
        toks = [self.id_lang.get(i, self.decoder.get(i, "<unk>")) for i in ids if i not in self.special]
        return self.sp.decode(toks)


# ------------------------------------------------------------------------------------------------ device engine
def mt_footprint(cfg: MtConfig, capacity: int, beams: int, max_src_tokens: int) -> int:
    """Device bytes a DeviceTranslator allocates (what wl_mt_init and the weights take), counted like wl_mt_init."""
    d, f, Le, Ld, V = cfg.d_model, cfg.ffn, cfg.enc_layers, cfg.dec_layers, cfg.vocab
    Ns, R, B = max_src_tokens, capacity * beams, capacity
    vld = (V + 7) // 8 * 8
    b = 0
    b += Ns * d * 4 + Ns * d * 2 + Ns * 3 * d * 2 + Ns * d * 2 + Ns * f * 2 + Ns * 2 * d * Ld * 2 + 2 * Ns * 4
    b += (B + 1) * 4 + (Ns // 64 + B) * 8
    b += R * d * 4 + R * 3 * d * 4 + R * d * 4 + R * vld * 4 + R * d * 2 * 2 + R * f * 2 + 2 * Ld * R * d * T_MAX * 2
    b += R * 4 * 3 + R * T_MAX * 2 + R * T_MAX * 4 + R * 4 * 2 + R * 16 * 8 + R * 4 * 3 + B * 8 * T_MAX * 4 + B * 4 * 3 + 8
    # weights
    lin = lambda o, i: o * i * 2 + o * 4
    w = V * d * 2 + (cfg.max_positions + 2) * d * 4
    w += Le * (2 * 2 * d * 4 + lin(3 * d, d) + lin(d, d) + lin(f, d) + lin(d, f)) + 2 * d * 4
    w += Ld * (3 * 2 * d * 4 + lin(3 * d, d) + 3 * lin(d, d) + lin(f, d) + lin(d, f)) + 2 * d * 4 + lin(2 * d * Ld, d)
    return b + w


class DeviceTranslator:
    """One wl_mt context: the model's weights and the buffers for ``capacity`` segments of up to ``beams`` beams."""

    def __init__(self, cfg: MtConfig, gen: GenSettings, weights: dict, tokenizer: Small100Tokenizer | None = None,
                 device: int = 0, capacity: int = 32, max_src_tokens: int | None = None, use_cuda_graph: bool = True):
        from . import _lib
        self._lib = lib = _lib.load()
        self.cfg, self.gen, self.tok, self.capacity = cfg, gen, tokenizer, capacity
        self.beams = gen.num_beams
        self.max_src_tokens = max_src_tokens or capacity * 128
        self.use_cuda_graph = use_cuda_graph
        mc = _lib.WlMtConfig(abi_version=_lib.ABI_VERSION, d_model=cfg.d_model, n_heads=cfg.n_heads, enc_layers=cfg.enc_layers,
                             dec_layers=cfg.dec_layers, ffn=cfg.ffn, vocab=cfg.vocab, max_positions=cfg.max_positions,
                             pad_id=cfg.pad_id, embed_scale=cfg.embed_scale, max_src_tokens=self.max_src_tokens)
        ctx = C.c_void_p()
        rc = lib.wl_mt_init(C.byref(mc), device, capacity, self.beams, C.byref(ctx))
        if rc != 0:
            raise _lib.WlError(f"wl_mt_init failed ({rc}): {lib.wl_mt_last_error(None).decode()}")
        self.ctx = ctx
        for name, arr in engine_tensors(weights, cfg).items():
            a = np.ascontiguousarray(arr, dtype=np.float32)
            shape = np.asarray(a.shape, dtype=np.int64)
            self._check(lib.wl_mt_load_tensor(ctx, name.encode(), _lib.ptr(a, C.c_float), _lib.ptr(shape, C.c_int64), a.ndim),
                        "wl_mt_load_tensor")
        self._check(lib.wl_mt_finalize(ctx), "wl_mt_finalize")

    def _check(self, rc, what):
        if rc != 0:
            from ._lib import WlError
            raise WlError(f"{what} failed ({rc}): {self._lib.wl_mt_last_error(self.ctx).decode()}")

    def close(self):
        if getattr(self, "ctx", None):
            self._lib.wl_mt_destroy(self.ctx)
            self.ctx = None

    def device_bytes(self) -> int:
        v = C.c_int64()
        self._check(self._lib.wl_mt_device_bytes(self.ctx, C.byref(v)), "wl_mt_device_bytes")
        return v.value

    def _opts(self, gen: GenSettings):
        from . import _lib
        return _lib.WlMtOpts(num_beams=gen.num_beams, max_length=gen.max_length, length_penalty=gen.length_penalty,
                             early_stopping=gen.early_stopping_code, decoder_start=gen.decoder_start_token_id,
                             eos=gen.eos_token_id,
                             forced_bos=-1 if gen.forced_bos_token_id is None else gen.forced_bos_token_id,
                             forced_eos=-1 if gen.forced_eos_token_id is None else gen.forced_eos_token_id,
                             use_cuda_graph=1 if self.use_cuda_graph else 0)

    def translate_ids(self, sources: list, gen: GenSettings | None = None) -> tuple[list, list]:
        """Token ids of each source -> (generated ids without the decoder start token, scores); one wl_mt_translate."""
        from . import _lib
        gen = gen or self.gen
        for s in sources:
            check_source_length(len(s), self.cfg)
        B = len(sources)
        off = np.zeros(B + 1, dtype=np.int32)
        off[1:] = np.cumsum([len(s) for s in sources])
        ids = np.ascontiguousarray(np.concatenate([np.asarray(s, dtype=np.int32) for s in sources]) if B else np.zeros(0, np.int32))
        out = np.full((B, gen.max_length), -1, dtype=np.int32)
        n = np.zeros(B, dtype=np.int32)
        score = np.zeros(B, dtype=np.float32)
        self._check(self._lib.wl_mt_translate(self.ctx, _lib.ptr(ids, C.c_int32), _lib.ptr(off, C.c_int32), B,
                                              C.byref(self._opts(gen)), _lib.ptr(out, C.c_int32), _lib.ptr(n, C.c_int32),
                                              _lib.ptr(score, C.c_float)), "wl_mt_translate")
        return [out[b, :n[b]].tolist() for b in range(B)], score.tolist()

    def decoder_logits(self, sources: list, prefixes) -> np.ndarray:
        """Teacher-forced logits [B][P][vocab] of the decoder fed ``prefixes`` [B][P] over the encoded ``sources``
        (the wl_test_mt_logits hook: the engine's encoder and decoder without the search)."""
        from . import _lib
        B = len(sources)
        off = np.zeros(B + 1, dtype=np.int32)
        off[1:] = np.cumsum([len(s) for s in sources])
        ids = np.ascontiguousarray(np.concatenate([np.asarray(s, dtype=np.int32) for s in sources]))
        pre = np.ascontiguousarray(np.asarray(prefixes, dtype=np.int32))
        P = pre.shape[1]
        out = np.zeros((B, P, self.cfg.vocab), dtype=np.float32)
        self._check(self._lib.wl_test_mt_logits(self.ctx, _lib.ptr(ids, C.c_int32), _lib.ptr(off, C.c_int32), B,
                                                _lib.ptr(pre, C.c_int32), P, _lib.ptr(out, C.c_float)), "wl_test_mt_logits")
        return out

    def translate_batch(self, texts: list, target_languages: list) -> list:
        """The translation of every text: whitespace-only text comes back unchanged; a text that cannot be translated
        (unknown language, source too long) gets its exception in its place, and the others are unaffected.  The rest
        go to wl_mt_translate in as few calls as the capacity and the source-token budget allow."""
        out = list(texts)
        todo = []
        for i, (t, lang) in enumerate(zip(texts, target_languages)):
            if not t.strip():
                continue
            try:
                ids = self.tok.encode(t, lang)
                check_source_length(len(ids), self.cfg)
                if len(ids) > self.max_src_tokens:
                    raise ValueError(f"source of {len(ids)} tokens exceeds the call budget of {self.max_src_tokens}")
                todo.append((i, ids))
            except Exception as e:
                out[i] = e
        for chunk in _chunks(todo, self.capacity, self.max_src_tokens):
            try:
                ids, _ = self.translate_ids([src for _, src in chunk])
                for (i, _), seq in zip(chunk, ids):
                    out[i] = self.tok.decode(seq)
            except Exception as e:
                for i, _ in chunk:
                    out[i] = e
        return out

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _chunks(items: list, capacity: int, token_budget: int) -> list:
    """Consecutive groups of (index, ids) with at most ``capacity`` sources and ``token_budget`` tokens each."""
    groups, cur, n = [], [], 0
    for it in items:
        if cur and (len(cur) == capacity or n + len(it[1]) > token_budget):
            groups.append(cur)
            cur, n = [], 0
        cur.append(it)
        n += len(it[1])
    if cur:
        groups.append(cur)
    return groups


# ------------------------------------------------------------------------------------------------ worker
class TranslationWorker:
    """The process-wide owner of the device translator: one thread, the only one that touches the context.  It takes
    every request pending from every connection and answers them with one call (up to the translator's capacity); a
    failing call fails only its own requests."""

    _shared = None
    _shared_lock = threading.Lock()

    @property
    def loaded(self) -> bool:
        return self._engine is not None

    def __init__(self, factory):
        self._factory = factory     # () -> object with translate_batch(texts, langs) and capacity
        self._q: queue.Queue = queue.Queue()
        self._engine = None
        self._error = None
        self.calls = 0
        self._thread = threading.Thread(target=self._run, name="wlb200-translate", daemon=True)
        self._thread.start()

    @classmethod
    def shared(cls, factory=None) -> "TranslationWorker":
        with cls._shared_lock:
            if cls._shared is None:
                cls._shared = cls(factory or default_translator)
            return cls._shared

    def submit(self, text: str, target_language: str, timeout: float | None = None) -> str:
        done = threading.Event()
        slot = {}
        self._q.put((text, target_language, done, slot))
        if not done.wait(timeout):
            raise TimeoutError("translation request timed out")
        if "error" in slot:
            raise slot["error"]
        return slot["text"]

    def _run(self):
        while True:
            batch = [self._q.get()]
            if self._engine is None and self._error is None:
                try:
                    self._engine = self._factory()
                except Exception as e:   # every request fails with the load error
                    self._error = e
            cap = getattr(self._engine, "capacity", 1 << 30)
            while len(batch) < cap:
                try:
                    batch.append(self._q.get_nowait())
                except queue.Empty:
                    break
            try:
                if self._error is not None:
                    raise self._error
                self.calls += 1
                res = self._engine.translate_batch([b[0] for b in batch], [b[1] for b in batch])
                for (_, _, done, slot), r in zip(batch, res):
                    if isinstance(r, BaseException):   # this request's own failure
                        slot["error"] = r
                    else:
                        slot["text"] = r
                    done.set()
            except Exception as e:
                for _, _, done, slot in batch:
                    slot["error"] = e
                    done.set()


DEFAULT_CAPACITY = 32          # segments per wl_mt_translate call of the process-wide translator
SRC_TOKENS_PER_SEGMENT = 128    # its packed source-token budget per segment


def translator_device() -> int:
    return int(os.environ.get("WLB200_DEVICES", "0").split(",")[0])


def default_translator() -> DeviceTranslator:
    path = resolve_snapshot()
    cfg, gen = load_snapshot_settings(path)
    tok = Small100Tokenizer.from_dir(path)
    return DeviceTranslator(cfg, gen, read_checkpoint(path, cfg), tok, device=translator_device(), capacity=DEFAULT_CAPACITY,
                            max_src_tokens=DEFAULT_CAPACITY * SRC_TOKENS_PER_SEGMENT)


def default_footprint() -> int | None:
    """Device bytes default_translator() will allocate (None when no snapshot can be found: it cannot load either)."""
    try:
        cfg, gen = load_snapshot_settings(resolve_snapshot())
    except Exception:
        return None
    return mt_footprint(cfg, DEFAULT_CAPACITY, gen.num_beams, DEFAULT_CAPACITY * SRC_TOKENS_PER_SEGMENT)


_footprint_cache: dict = {}


def pending_translator_bytes(device: int, footprint=default_footprint) -> int:
    """What the process-wide translator will still allocate on ``device``: its footprint while ``WLB200_TRANSLATE=device``
    and it is not loaded yet (ModelRegistry counts it as spoken for), else 0."""
    if translate_mode() != "device" or int(device) != translator_device():
        return 0
    w = TranslationWorker._shared
    if w is not None and w.loaded:
        return 0
    if footprint not in _footprint_cache:
        _footprint_cache[footprint] = footprint()
    return int(_footprint_cache[footprint] or 0)


# ------------------------------------------------------------------------------------------------ client
def _client_base():
    try:
        from whisper_live.backend.base import ServeClientBase
        return ServeClientBase
    except ImportError:      # the reference package is not installed: the same constructor contract
        class ServeClientBase:
            def __init__(self, client_uid, websocket, send_last_n_segments=10):
                self.client_uid, self.websocket, self.send_last_n_segments = client_uid, websocket, send_last_n_segments
                self.exit = False
        return ServeClientBase


class DeviceTranslationClient(_client_base()):
    """The reference's ``ServeClientTranslation`` on the shared device translator: same constructor, queue loop,
    messages and fall-backs (text echoed when the model or the language is unavailable or a call fails); the model is
    never loaded per connection and ``cleanup`` never frees it."""

    def __init__(self, client_uid, websocket, translation_queue, target_language="fr", send_last_n_segments=10,
                 model_name=DEFAULT_MODEL, worker: TranslationWorker | None = None):
        super().__init__(client_uid, websocket, send_last_n_segments)
        self.translation_queue = translation_queue
        self.target_language = target_language
        self.model_name = model_name
        self.translated_segments = []
        self.worker = worker
        self.model_loaded = False
        self.load_translation_model()

    def load_translation_model(self):
        try:
            if self.worker is None:
                self.worker = TranslationWorker.shared()
            self.model_loaded = self.target_language in FAIRSEQ_LANGUAGE_CODES
            if not self.model_loaded:
                logging.error(f"Failed to load translation model: unknown target language {self.target_language!r}")
        except Exception as e:
            logging.error(f"Failed to load translation model: {e}")
            self.model_loaded = False

    def translate_text(self, text: str) -> str:
        if not self.model_loaded or not text.strip():
            return text
        try:
            return self.worker.submit(text, self.target_language)
        except Exception as e:
            logging.error(f"Translation failed for text '{text}': {e}")
            return text

    def process_translation_queue(self):
        while not self.exit:
            try:
                segment = self.translation_queue.get(timeout=1.0)
                if segment is None:
                    break
                if not segment.get("completed", False):
                    self.translation_queue.task_done()
                    continue
                translated = self.translate_text(segment.get("text", ""))
                self.translated_segments.append({
                    "start": segment["start"], "end": segment["end"], "text": translated,
                    "completed": segment.get("completed", False), "target_language": self.target_language,
                })
                self.send_translation_to_client(self.prepare_translated_segments())
                self.translation_queue.task_done()
            except queue.Empty:
                continue
            except Exception as e:
                logging.error(f"Error processing translation queue: {e}")
                continue

    def prepare_translated_segments(self):
        if len(self.translated_segments) >= self.send_last_n_segments:
            return self.translated_segments[-self.send_last_n_segments:]
        return self.translated_segments[:]

    def send_translation_to_client(self, translated_segments):
        try:
            self.websocket.send(json.dumps({"uid": self.client_uid, "translated_segments": translated_segments}))
        except Exception as e:
            logging.error(f"[ERROR]: Sending translation data to client: {e}")

    def speech_to_text(self):
        self.process_translation_queue()

    def set_target_language(self, language: str):
        # as the reference: the new language is kept, then its tokenizer raises on an unknown one
        self.target_language = language
        if self.model_loaded and language not in FAIRSEQ_LANGUAGE_CODES:
            raise KeyError(language)

    def cleanup(self):
        self.exit = True
        try:
            self.translation_queue.put(None, timeout=1.0)
        except Exception:
            pass
        self.translated_segments.clear()
