"""CTranslate2 ``model.bin`` reader / writer for Whisper checkpoints (SURVEY.md §8f N1).

The reference loads ``<model_dir>/model.bin`` + ``config.json`` through ``ctranslate2.models.Whisper(model_path, ...)``
(/root/reference/whisper_live/transcriber/transcriber_faster_whisper.py:634-643; the directory comes from
``download_model`` / a local path, backend/faster_whisper_backend.py:133-178).  CTranslate2 is not vendored in the
reference tree and not installed here, so the container format below is RESTATED FROM THE PUBLISHED SOURCE FROM MEMORY
(ctranslate2 4.x ``python/ctranslate2/specs/model_spec.py::ModelSpec._serialize``, binary version 6, and the variable
names produced by ``specs/whisper_spec.py`` + ``transformer_spec.py`` + ``attention_spec.py``).  It is exercised by a
write -> read round trip only (tests/test_transcriber_host.py); it has NOT been checked against a real converted model.
Anything unexpected in a file makes the reader fail loudly instead of guessing.

Layout (little endian):
    u32 binary_version (6) | str spec_name ("WhisperSpec") | u32 spec_revision | u32 n_variables
    n_variables x { str name | u8 rank | rank x u32 dim | u8 dtype_id | u32 n_bytes | bytes }
    u32 n_aliases | n_aliases x { str alias | str variable_name }
    str = u16 (len + 1) | utf-8 bytes | NUL
dtype ids (ctranslate2 ``DataType``): 0 float32, 1 int8, 2 int16, 3 int32, 4 float16, 5 bfloat16.
"""
from __future__ import annotations

import json
import os
import struct
from typing import Dict, Iterator, List, NamedTuple, Optional, Tuple

import numpy as np
import torch

BINARY_VERSION = 6
_DTYPES = {0: np.float32, 1: np.int8, 2: np.int16, 3: np.int32, 4: np.float16}
_DTYPE_IDS = {np.dtype(np.float32): 0, np.dtype(np.int8): 1, np.dtype(np.int16): 2, np.dtype(np.int32): 3,
              np.dtype(np.float16): 4}
_BF16 = 5


def _read_str(f) -> str:
    (n,) = struct.unpack("<H", f.read(2))
    raw = f.read(n)
    if len(raw) != n or n == 0 or raw[-1] != 0:
        raise ValueError("model.bin: malformed string field")
    return raw[:-1].decode("utf-8")


def _write_str(f, s: str) -> None:
    b = s.encode("utf-8")
    f.write(struct.pack("<H", len(b) + 1))
    f.write(b)
    f.write(b"\0")


class VarInfo(NamedTuple):
    """A variable of a model.bin as its header describes it: where its payload lies in the file."""
    shape: Tuple[int, ...]
    dtype_id: int
    offset: int
    n_bytes: int


_ITEMSIZE = {0: 4, 1: 1, 2: 2, 3: 4, 4: 2, 5: 2}


def read_variables(path: str, header_only: bool = False):
    """Return (variables, aliases, header) of a CTranslate2 model.bin.  bfloat16 payloads come back as float32.
    ``header_only``: the variables are ``VarInfo`` records and the payloads are skipped with a seek, so the table of a
    multi-gigabyte file is read in a few kilobytes."""
    variables: Dict[str, object] = {}
    with open(path, "rb") as f:
        (version,) = struct.unpack("<I", f.read(4))
        if version != BINARY_VERSION:
            raise ValueError(f"model.bin: binary version {version}, this reader understands {BINARY_VERSION} only")
        spec = _read_str(f)
        revision, n_var = struct.unpack("<II", f.read(8))
        size = os.fstat(f.fileno()).st_size
        for _ in range(n_var):
            name = _read_str(f)
            (rank,) = struct.unpack("<B", f.read(1))
            shape = struct.unpack(f"<{rank}I", f.read(4 * rank)) if rank else ()
            dtype_id, n_bytes = struct.unpack("<BI", f.read(5))
            if dtype_id not in _ITEMSIZE:
                raise ValueError(f"model.bin: variable {name!r} has unknown dtype id {dtype_id}")
            count = int(np.prod(shape)) if rank else 1
            if n_bytes != _ITEMSIZE[dtype_id] * count:
                raise ValueError(f"model.bin: variable {name!r}: {n_bytes} bytes for {count} values of dtype id {dtype_id}")
            if header_only:
                offset = f.tell()
                if offset + n_bytes > size:
                    raise ValueError(f"model.bin: variable {name!r} truncated")
                f.seek(n_bytes, os.SEEK_CUR)
                variables[name] = VarInfo(tuple(shape), dtype_id, offset, n_bytes)
                continue
            raw = f.read(n_bytes)
            if len(raw) != n_bytes:
                raise ValueError(f"model.bin: variable {name!r} truncated")
            if dtype_id == _BF16:
                u = np.frombuffer(raw, dtype=np.uint16).astype(np.uint32) << 16
                arr = u.view(np.float32).reshape(shape)
            else:
                arr = np.frombuffer(raw, dtype=np.dtype(_DTYPES[dtype_id])).reshape(shape).copy()
            variables[name] = arr
        aliases: Dict[str, str] = {}
        tail = f.read(4)
        if tail:
            (n_alias,) = struct.unpack("<I", tail)
            for _ in range(n_alias):
                alias = _read_str(f)
                aliases[alias] = _read_str(f)
        if f.read(1):
            raise ValueError("model.bin: trailing bytes after the alias table")
    for alias, target in aliases.items():
        if target not in variables:
            raise ValueError(f"model.bin: alias {alias!r} points at missing variable {target!r}")
    return variables, aliases, {"spec": spec, "revision": revision, "version": version}


def write_variables(path: str, variables: Dict[str, np.ndarray], aliases: Optional[Dict[str, str]] = None,
                    spec: str = "WhisperSpec", revision: int = 3) -> None:
    with open(path, "wb") as f:
        f.write(struct.pack("<I", BINARY_VERSION))
        _write_str(f, spec)
        f.write(struct.pack("<II", revision, len(variables)))
        for name in sorted(variables):
            arr = np.ascontiguousarray(variables[name])
            if arr.dtype not in _DTYPE_IDS and arr.dtype != np.uint16:
                raise ValueError(f"cannot serialise {name!r} of dtype {arr.dtype}")
            _write_str(f, name)
            f.write(struct.pack("<B", arr.ndim))
            for d in arr.shape:
                f.write(struct.pack("<I", d))
            # bfloat16 variables are handed over as their uint16 bit patterns (numpy has no bfloat16)
            f.write(struct.pack("<BI", _BF16 if arr.dtype == np.uint16 else _DTYPE_IDS[arr.dtype], arr.nbytes))
            f.write(arr.tobytes())
        aliases = aliases or {}
        f.write(struct.pack("<I", len(aliases)))
        for alias in sorted(aliases):
            _write_str(f, alias)
            _write_str(f, aliases[alias])


# ------------------------------------------------------------------------------------------ name mapping
# Dequantization, a recalled upstream rule (ctranslate2 4.x ``specs/model_spec.py``, the ``int8*`` branch of the
# quantization step, restated from memory; tests/golden/capture_ct2_convert.py records real conversions to check it):
# a ``.../weight`` matrix W is stored as int8 ``q = round(W[r] * scale[r])`` with ``scale[r] = 127 / amax(|W[r]|)``
# (an all-zero row gets ``amax = 127``) and its scales as the sibling variable ``.../weight_scale``, one per row.
# CTranslate2 computes with ``W[r] = q / scale[r]``; loading at compute_type float16 rounds that value to fp16.
# ``int16`` files (``scale`` a single 2^k) are not read: the engine has no use for them and they are rare.

# Each canonical tensor is rows [r0, r1) of one CT2 variable (None: all rows): CT2 fuses the attention projections --
# self-attention linear_0 = [q; k; v], linear_1 = out; cross-attention linear_0 = q, linear_1 = [k; v],
# linear_2 = out.  Whisper's k_proj has no bias (CT2 stores zeros in its slice).
Plan = List[Tuple[str, str, Optional[Tuple[int, int]]]]


def ct2_plan(shapes: Dict[str, Tuple[int, ...]], aliases: Optional[Dict[str, str]] = None) -> Plan:
    """(canonical HF name, CT2 variable, row range) for every tensor the engine reads, from the variable table alone."""
    aliases = aliases or {}
    plan: Plan = []

    def var(name):
        key = aliases.get(name, name)
        if key not in shapes:
            raise KeyError(f"model.bin: variable {name!r} is missing")
        return key

    def whole(dst, src):
        plan.append((dst, var(src), None))

    def norm(src, dst):
        whole(f"{dst}.weight", f"{src}/gamma")
        whole(f"{dst}.bias", f"{src}/beta")

    def attention(src, dst, cross):
        if cross:
            d = shapes[var(f"{src}/linear_0/weight")][0]
            whole(f"{dst}.q_proj.weight", f"{src}/linear_0/weight")
            whole(f"{dst}.q_proj.bias", f"{src}/linear_0/bias")
            kv, kvb = var(f"{src}/linear_1/weight"), var(f"{src}/linear_1/bias")
            plan.extend([(f"{dst}.k_proj.weight", kv, (0, d)), (f"{dst}.v_proj.weight", kv, (d, 2 * d)),
                         (f"{dst}.v_proj.bias", kvb, (d, 2 * d))])
            out = 2
        else:
            w, b = var(f"{src}/linear_0/weight"), var(f"{src}/linear_0/bias")
            d = shapes[w][0] // 3
            plan.extend([(f"{dst}.q_proj.weight", w, (0, d)), (f"{dst}.q_proj.bias", b, (0, d)),
                         (f"{dst}.k_proj.weight", w, (d, 2 * d)),
                         (f"{dst}.v_proj.weight", w, (2 * d, 3 * d)), (f"{dst}.v_proj.bias", b, (2 * d, 3 * d))])
            out = 1
        whole(f"{dst}.out_proj.weight", f"{src}/linear_{out}/weight")
        whole(f"{dst}.out_proj.bias", f"{src}/linear_{out}/bias")

    def ffn(s, h):
        norm(f"{s}/ffn/layer_norm", f"{h}.final_layer_norm")
        for i, fc in enumerate(("fc1", "fc2")):
            whole(f"{h}.{fc}.weight", f"{s}/ffn/linear_{i}/weight")
            whole(f"{h}.{fc}.bias", f"{s}/ffn/linear_{i}/bias")

    for conv in ("conv1", "conv2"):
        whole(f"model.encoder.{conv}.weight", f"encoder/{conv}/weight")
        whole(f"model.encoder.{conv}.bias", f"encoder/{conv}/bias")
    whole("model.encoder.embed_positions.weight", "encoder/position_encodings/encodings")
    norm("encoder/layer_norm", "model.encoder.layer_norm")
    n_enc = 0
    while f"encoder/layer_{n_enc}/self_attention/linear_0/weight" in shapes:
        s, h = f"encoder/layer_{n_enc}", f"model.encoder.layers.{n_enc}"
        norm(f"{s}/self_attention/layer_norm", f"{h}.self_attn_layer_norm")
        attention(f"{s}/self_attention", f"{h}.self_attn", cross=False)
        ffn(s, h)
        n_enc += 1
    whole("model.decoder.embed_tokens.weight", "decoder/embeddings/weight")
    whole("model.decoder.embed_positions.weight", "decoder/position_encodings/encodings")
    norm("decoder/layer_norm", "model.decoder.layer_norm")
    n_dec = 0
    while f"decoder/layer_{n_dec}/self_attention/linear_0/weight" in shapes:
        s, h = f"decoder/layer_{n_dec}", f"model.decoder.layers.{n_dec}"
        norm(f"{s}/self_attention/layer_norm", f"{h}.self_attn_layer_norm")
        attention(f"{s}/self_attention", f"{h}.self_attn", cross=False)
        norm(f"{s}/attention/layer_norm", f"{h}.encoder_attn_layer_norm")
        attention(f"{s}/attention", f"{h}.encoder_attn", cross=True)
        ffn(s, h)
        n_dec += 1
    if n_enc == 0 or n_dec == 0:
        raise ValueError("model.bin: no encoder / decoder layers found under the expected variable names")
    return plan


class Ct2Checkpoint:
    """A CTranslate2 ``model.bin`` read in place: the variable table from the header, payloads through one read-only
    memory map.  ``tensors()`` yields ``(canonical name, array as stored, scale or None)`` one tensor at a time:
    float32 / float16 arrays, bfloat16 as uint16 bit patterns, int8 with its per-row scales (module comment above)."""
    layout = "ct2"

    def __init__(self, path: str):
        if os.path.isdir(path):
            path = os.path.join(path, "model.bin")
        self.path = path
        variables, aliases, header = read_variables(path, header_only=True)
        if header["spec"] != "WhisperSpec":
            raise ValueError(f"model.bin holds a {header['spec']!r}, not a WhisperSpec")
        self.variables, self.aliases = variables, aliases
        self.plan = ct2_plan({k: v.shape for k, v in variables.items()}, aliases)
        for dst, src, _ in self.plan:
            info = variables[src]
            if info.dtype_id == 2:
                raise ValueError(f"model.bin: {src!r} is int16-quantised; int16 CTranslate2 files are not supported "
                                 f"(convert with --quantization float16, int8_float16 or bfloat16)")
            if info.dtype_id == 1:
                sc = variables.get(src + "_scale")
                if sc is None:
                    raise ValueError(f"model.bin: {src!r} is int8 but its scale {src + '_scale'!r} is missing")
                if sc.dtype_id not in (0, 4, _BF16) or int(np.prod(sc.shape)) != info.shape[0]:
                    raise ValueError(f"model.bin: {src + '_scale'!r} must hold one float per row of {src!r} "
                                     f"({info.shape[0]}), has shape {sc.shape} and dtype id {sc.dtype_id}")
            elif info.dtype_id not in (0, 4, _BF16):
                raise ValueError(f"model.bin: {src!r} has dtype id {info.dtype_id}, not a float or int8 weight")
        self.shapes = {dst: ((r[1] - r[0],) if r else variables[src].shape[:1]) + tuple(variables[src].shape[1:])
                       for dst, src, r in self.plan}
        # the spec stores each stack's head count as an int16 scalar; the engine runs 64-wide heads only
        d = self.shapes["model.encoder.conv1.weight"][0]
        for side in ("encoder", "decoder"):
            info = variables.get(f"{side}/num_heads")
            if info is None:
                continue
            with open(path, "rb") as f:
                f.seek(info.offset)
                raw = f.read(info.n_bytes)
            heads = int(np.frombuffer(raw, dtype=_DTYPES[info.dtype_id])[0])
            if heads <= 0 or d != 64 * heads:
                raise ValueError(f"model.bin: {side}/num_heads = {heads} with d_model {d} is a head dimension other "
                                 f"than 64; the engine runs 64 only")

    def _array(self, mm, name: str) -> np.ndarray:
        info = self.variables[name]
        dt = np.uint16 if info.dtype_id == _BF16 else _DTYPES[info.dtype_id]
        count = int(np.prod(info.shape)) if info.shape else 1
        return np.frombuffer(mm, dtype=dt, count=count, offset=info.offset).reshape(info.shape)

    def tensors(self) -> Iterator[Tuple[str, np.ndarray, Optional[np.ndarray]]]:
        mm = np.memmap(self.path, dtype=np.uint8, mode="r")
        try:
            for dst, src, rows in self.plan:
                a = self._array(mm, src)
                scale = self._array(mm, src + "_scale").reshape(-1) if a.dtype == np.int8 else None
                if rows is not None:
                    a = a[rows[0]:rows[1]]
                    scale = scale[rows[0]:rows[1]] if scale is not None else None
                yield dst, a, scale
        finally:
            del mm


def load_ct2_model_bin(path: str) -> Dict[str, torch.Tensor]:
    """``model.bin`` (or its directory) -> the canonical HF-named fp32 dict (the key space of the Hugging Face
    readers, weights.HFCheckpoint).  int8 weights are dequantized with the rule above; int16 files are refused."""
    from .weights import to_float32
    return {name: torch.from_numpy(to_float32(a, scale)) for name, a, scale in Ct2Checkpoint(path).tensors()}


def expected_ct2_names(n_enc: int, n_dec: int) -> List[str]:
    """Every variable name ``load_ct2_model_bin`` reads for a Whisper with n_enc / n_dec layers -- compared against the
    variable table of a REAL converted model by tests/test_ct2_capture.py (the container layout and these names are
    restated from memory; that test is what validates them)."""
    names = ["encoder/conv1/weight", "encoder/conv1/bias", "encoder/conv2/weight", "encoder/conv2/bias",
             "encoder/position_encodings/encodings", "encoder/layer_norm/gamma", "encoder/layer_norm/beta",
             "decoder/embeddings/weight", "decoder/position_encodings/encodings", "decoder/layer_norm/gamma", "decoder/layer_norm/beta"]

    def norm(p):
        return [f"{p}/gamma", f"{p}/beta"]

    def lin(p, i):
        return [f"{p}/linear_{i}/weight", f"{p}/linear_{i}/bias"]
    for l in range(n_enc):
        s_ = f"encoder/layer_{l}"
        names += norm(f"{s_}/self_attention/layer_norm") + lin(f"{s_}/self_attention", 0) + lin(f"{s_}/self_attention", 1)
        names += norm(f"{s_}/ffn/layer_norm") + lin(f"{s_}/ffn", 0) + lin(f"{s_}/ffn", 1)
    for l in range(n_dec):
        s_ = f"decoder/layer_{l}"
        names += norm(f"{s_}/self_attention/layer_norm") + lin(f"{s_}/self_attention", 0) + lin(f"{s_}/self_attention", 1)
        names += norm(f"{s_}/attention/layer_norm") + lin(f"{s_}/attention", 0) + lin(f"{s_}/attention", 1) + lin(f"{s_}/attention", 2)
        names += norm(f"{s_}/ffn/layer_norm") + lin(f"{s_}/ffn", 0) + lin(f"{s_}/ffn", 1)
    return names


QUANTIZATIONS = {"float32": (np.float32, False), "float16": (np.float16, False), "bfloat16": ("bfloat16", False),
                 "int8": (np.float32, True), "int8_float32": (np.float32, True), "int8_float16": (np.float16, True),
                 "int8_bfloat16": ("bfloat16", True), "int16": (np.float32, "int16")}


def _quantize(w: np.ndarray, bits: int = 8) -> Tuple[np.ndarray, np.ndarray]:
    """The converter's per-row quantization (module comment above); int16 uses one power-of-two scale."""
    w = w.astype(np.float32)
    if bits == 16:
        scale = np.float32(2.0 ** np.floor(np.log2(32767.0 / max(float(np.abs(w).max()), 1e-30))))
        return np.rint(w * scale).astype(np.int16), np.asarray(scale, np.float32)
    amax = np.abs(w).max(axis=1)
    amax[amax == 0] = 127.0
    scale = (127.0 / amax).astype(np.float32)
    return np.rint(w * scale[:, None]).astype(np.int8), scale


def save_ct2_model_bin(weights: Dict[str, torch.Tensor], path: str, dtype=np.float16,
                       quantization: Optional[str] = None) -> None:
    """Inverse of load_ct2_model_bin (tests, and to hand a checkpoint to a CTranslate2 install for cross-checks).
    ``quantization`` names a CTranslate2 conversion ("float16", "bfloat16", "int8_float16", ...): float variables are
    written in its float type, and for int8* / int16 every 2-D ``.../weight`` is quantized with a ``..._scale``
    sibling.  Without it every variable is written as ``dtype``."""
    quant = False
    if quantization is not None:
        if quantization not in QUANTIZATIONS:
            raise ValueError(f"quantization {quantization!r}: one of {sorted(QUANTIZATIONS)}")
        dtype, quant = QUANTIZATIONS[quantization]

    def npy(name):
        a = weights[name].detach().cpu().float()
        if dtype == "bfloat16":
            return a.bfloat16().view(torch.int16).numpy().view(np.uint16)
        return a.numpy().astype(dtype)

    def zeros_like_bias(w):
        return np.zeros((w.shape[0],), dtype=np.uint16 if dtype == "bfloat16" else dtype)

    v: Dict[str, np.ndarray] = {}
    for conv in ("conv1", "conv2"):
        v[f"encoder/{conv}/weight"], v[f"encoder/{conv}/bias"] = npy(f"model.encoder.{conv}.weight"), npy(f"model.encoder.{conv}.bias")
    v["encoder/position_encodings/encodings"] = npy("model.encoder.embed_positions.weight")
    v["encoder/layer_norm/gamma"], v["encoder/layer_norm/beta"] = npy("model.encoder.layer_norm.weight"), npy("model.encoder.layer_norm.bias")

    def norm(src, dst):
        v[f"{dst}/gamma"], v[f"{dst}/beta"] = npy(f"{src}.weight"), npy(f"{src}.bias")

    def ffn(h, s):
        norm(f"{h}.final_layer_norm", f"{s}/ffn/layer_norm")
        for i, fc in enumerate(("fc1", "fc2")):
            v[f"{s}/ffn/linear_{i}/weight"], v[f"{s}/ffn/linear_{i}/bias"] = npy(f"{h}.{fc}.weight"), npy(f"{h}.{fc}.bias")

    def self_attn(h, s):
        wq, wk, wv = npy(f"{h}.q_proj.weight"), npy(f"{h}.k_proj.weight"), npy(f"{h}.v_proj.weight")
        v[f"{s}/linear_0/weight"] = np.concatenate([wq, wk, wv], 0)
        v[f"{s}/linear_0/bias"] = np.concatenate([npy(f"{h}.q_proj.bias"), zeros_like_bias(wk), npy(f"{h}.v_proj.bias")], 0)
        v[f"{s}/linear_1/weight"], v[f"{s}/linear_1/bias"] = npy(f"{h}.out_proj.weight"), npy(f"{h}.out_proj.bias")

    i = 0
    while f"model.encoder.layers.{i}.fc1.weight" in weights:
        h, s = f"model.encoder.layers.{i}", f"encoder/layer_{i}"
        norm(f"{h}.self_attn_layer_norm", f"{s}/self_attention/layer_norm")
        self_attn(f"{h}.self_attn", f"{s}/self_attention")
        ffn(h, s)
        i += 1
    v["decoder/embeddings/weight"] = npy("model.decoder.embed_tokens.weight")
    v["decoder/position_encodings/encodings"] = npy("model.decoder.embed_positions.weight")
    v["decoder/layer_norm/gamma"], v["decoder/layer_norm/beta"] = npy("model.decoder.layer_norm.weight"), npy("model.decoder.layer_norm.bias")
    i = 0
    while f"model.decoder.layers.{i}.fc1.weight" in weights:
        h, s = f"model.decoder.layers.{i}", f"decoder/layer_{i}"
        norm(f"{h}.self_attn_layer_norm", f"{s}/self_attention/layer_norm")
        self_attn(f"{h}.self_attn", f"{s}/self_attention")
        norm(f"{h}.encoder_attn_layer_norm", f"{s}/attention/layer_norm")
        a = f"{h}.encoder_attn"
        wk, wv = npy(f"{a}.k_proj.weight"), npy(f"{a}.v_proj.weight")
        v[f"{s}/attention/linear_0/weight"], v[f"{s}/attention/linear_0/bias"] = npy(f"{a}.q_proj.weight"), npy(f"{a}.q_proj.bias")
        v[f"{s}/attention/linear_1/weight"] = np.concatenate([wk, wv], 0)
        v[f"{s}/attention/linear_1/bias"] = np.concatenate([zeros_like_bias(wk), npy(f"{a}.v_proj.bias")], 0)
        v[f"{s}/attention/linear_2/weight"], v[f"{s}/attention/linear_2/bias"] = npy(f"{a}.out_proj.weight"), npy(f"{a}.out_proj.bias")
        ffn(h, s)
        i += 1
    if quant:
        for name in [k for k in v if k.endswith("/weight") and v[k].ndim == 2]:
            w = v[name].astype(np.uint32) << 16 if v[name].dtype == np.uint16 else v[name]
            w = w.view(np.float32) if w.dtype == np.uint32 else w
            v[name], v[name + "_scale"] = _quantize(w, 16 if quant == "int16" else 8)
    heads = np.int16(v["encoder/conv1/weight"].shape[0] // 64)
    v["encoder/num_heads"] = v["decoder/num_heads"] = np.asarray(heads, dtype=np.int16)
    # the output projection is tied to the embedding: CT2 stores it once and lists the second name as an alias
    write_variables(path, v, aliases={"decoder/projection/weight": "decoder/embeddings/weight"})


def read_ct2_config(model_dir: str) -> Dict[str, object]:
    """``config.json`` next to model.bin: alignment heads and special-token id lists written by the CT2 converter
    (keys ``alignment_heads``, ``lang_ids``, ``suppress_ids``, ``suppress_ids_begin``); absent keys are omitted."""
    p = os.path.join(model_dir, "config.json")
    if not os.path.exists(p):
        return {}
    cfg = json.load(open(p))
    out: Dict[str, object] = {}
    if "alignment_heads" in cfg:
        out["alignment_heads"] = [(int(a), int(b)) for a, b in cfg["alignment_heads"]]
    for k in ("lang_ids", "suppress_ids", "suppress_ids_begin"):
        if k in cfg:
            out[k] = [int(x) for x in cfg[k]]
    return out
