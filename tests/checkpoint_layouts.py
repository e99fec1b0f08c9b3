"""Writers of every checkpoint layout the engine reads, from a canonical tensor dict (``weights.random_init``), and the
values each layout should give the device.  Shared by tests/test_checkpoint_formats.py and its GPU twin."""
from __future__ import annotations

import json
import os
from typing import Dict

import numpy as np
import torch

from whisperlive_b200 import ct2_format

HF_LAYOUTS = ["safetensors", "safetensors-sharded", "bin", "bin-sharded"]
HF_DTYPES = {"float32": torch.float32, "float16": torch.float16, "bfloat16": torch.bfloat16}
CT2_QUANT = ["float16", "bfloat16", "float32", "int8", "int8_float16", "int8_float32", "int8_bfloat16"]


def _shards(keys, n):
    keys = sorted(keys)
    return [keys[i::n] for i in range(n)]


def write_hf(w: Dict[str, torch.Tensor], path: str, layout: str, dtype: str = "float16", prefix: bool = True,
             n_shards: int = 3) -> str:
    """``layout`` in HF_LAYOUTS; keys keep ``model.`` unless ``prefix`` is False."""
    os.makedirs(path, exist_ok=True)
    sd = {(k if prefix else k[len("model."):]): v.to(HF_DTYPES[dtype]).contiguous() for k, v in w.items()}
    st = layout.startswith("safetensors")
    if st:
        from safetensors.torch import save_file

        def save(d, f):
            save_file(d, os.path.join(path, f), metadata={"format": "pt"})
    else:
        def save(d, f):
            torch.save(d, os.path.join(path, f))
    single = "model.safetensors" if st else "pytorch_model.bin"
    if not layout.endswith("sharded"):
        save(sd, single)
        return path
    groups = _shards(sd, n_shards)
    weight_map = {}
    for i, keys in enumerate(groups):
        name = (f"model-{i + 1:05d}-of-{len(groups):05d}.safetensors" if st
                else f"pytorch_model-{i + 1:05d}-of-{len(groups):05d}.bin")
        save({k: sd[k] for k in keys}, name)
        weight_map.update({k: name for k in keys})
    total = sum(v.numel() * v.element_size() for v in sd.values())
    with open(os.path.join(path, single + ".index.json"), "w") as f:
        json.dump({"metadata": {"total_size": total}, "weight_map": weight_map}, f)
    return path


def write_ct2(w: Dict[str, torch.Tensor], path: str, quantization: str) -> str:
    os.makedirs(path, exist_ok=True)
    ct2_format.save_ct2_model_bin(w, os.path.join(path, "model.bin"), quantization=quantization)
    return path


def _float_of(t: torch.Tensor, dtype: str) -> np.ndarray:
    return t.to(HF_DTYPES[dtype]).float().numpy()


def expected_f32(w: Dict[str, torch.Tensor], fmt: str, dtype: str) -> Dict[str, np.ndarray]:
    """The fp32 value of every tensor the engine reads from the layout (before the device rounds matrices to fp16):
    the stored float rounding, and for int8 the host formula ``q.astype(f32) / scale`` on the writer's quantization."""
    if fmt != "ct2":
        return {k: _float_of(v, dtype) for k, v in w.items()}
    ftype, quant = ct2_format.QUANTIZATIONS[dtype]
    ftype = "bfloat16" if ftype == "bfloat16" else {np.float16: "float16", np.float32: "float32"}[ftype]
    out = {}
    for k, v in w.items():
        if k.endswith("k_proj.bias"):
            continue
        f = _float_of(v, ftype)
        # the 2-D weights of attention, FFN and the embedding are quantized; position tables are "encodings"
        if quant and f.ndim == 2 and "embed_positions" not in k:
            q, s = ct2_format._quantize(f)
            f = q.astype(np.float32) / s[:, None]
        out[k] = f
    return out


def device_value(name: str, f32: np.ndarray) -> np.ndarray:
    """What the engine keeps on the device for a tensor of that fp32 value (csrc/engine.cu, wl_load_tensor)."""
    if f32.ndim == 1 or name in ("model.encoder.embed_positions.weight", "mel_filters"):
        return f32.astype(np.float32)
    return f32.astype(np.float16)
