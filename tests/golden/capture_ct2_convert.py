#!/usr/bin/env python
"""Capture what CTranslate2's ``TransformersConverter`` writes for a Whisper model, to pin the rules the loader
recalls (whisperlive_b200/ct2_format.py: int8 dequantization; weights.model_metadata: the config.json keys).

Run it once on a machine with ``pip install ctranslate2 transformers`` and commit what it writes:

    tests/golden/ct2_convert_capture.json   per quantization (float16, int8_float16, int8, bfloat16): the converted
                                            config.json, the variable table (name, dtype id, shape) and, for a few
                                            variables, rows as stored plus their scales

It writes a seeded micro Whisper (WhisperForConditionalGeneration with a generation_config holding alignment heads,
suppress lists and lang_to_id) with transformers and converts it four times, then once more with a generation_config
that lacks the heads and the begin-suppress list (config.json holding both), to show where missing keys come from.
tests/test_ct2_convert_capture.py consumes the fixture and is skipped, with that reason, until it exists.

    python tests/golden/capture_ct2_convert.py
"""
from __future__ import annotations

import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "ct2_convert_capture.json")
QUANTIZATIONS = ["float16", "int8_float16", "int8", "bfloat16"]
ROWS = ["decoder/layer_0/self_attention/linear_0/weight", "decoder/embeddings/weight", "encoder/conv1/weight",
        "encoder/layer_0/ffn/linear_1/weight"]


def main() -> int:
    try:
        import ctranslate2
        import transformers
    except ImportError as e:
        print(f"capture_ct2_convert.py needs ctranslate2 and transformers ({e})", file=sys.stderr)
        return 2
    import numpy as np
    import torch
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from whisperlive_b200 import ct2_format
    from whisperlive_b200.config import dims_for
    from whisperlive_b200.weights import random_init

    dims = dims_for("micro")
    torch.manual_seed(0)
    cfg = transformers.WhisperConfig(vocab_size=dims.vocab, num_mel_bins=dims.n_mels, d_model=dims.d_model,
                                     encoder_layers=dims.enc_layers, decoder_layers=dims.dec_layers,
                                     encoder_attention_heads=dims.n_heads, decoder_attention_heads=dims.n_heads,
                                     encoder_ffn_dim=dims.d_ff, decoder_ffn_dim=dims.d_ff)
    model = transformers.WhisperForConditionalGeneration(cfg)
    sd = dict(random_init(dims, seed=11))
    sd["proj_out.weight"] = sd["model.decoder.embed_tokens.weight"]
    model.load_state_dict(sd, strict=False)
    gen = model.generation_config
    gen.alignment_heads = [[1, 0], [1, 1]]
    gen.suppress_tokens = [1, 2, 7]
    gen.begin_suppress_tokens = [220, 50257]
    gen.lang_to_id = {"<|en|>": 50259, "<|de|>": 50261, "<|fr|>": 50265}
    out = {"versions": {"ctranslate2": ctranslate2.__version__, "transformers": transformers.__version__},
           "conversions": {}}
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "hf")
        model.save_pretrained(src)
        for q in QUANTIZATIONS:
            dst = os.path.join(tmp, q)
            ctranslate2.converters.TransformersConverter(src).convert(dst, quantization=q, force=True)
            info, aliases, header = ct2_format.read_variables(os.path.join(dst, "model.bin"), header_only=True)
            full, _, _ = ct2_format.read_variables(os.path.join(dst, "model.bin"))
            rows = {}
            for name in ROWS:
                if name in full:
                    a = full[name]
                    rows[name] = {"rows": np.asarray(a[:2]).astype(np.float64).tolist()}
                    if name + "_scale" in full:
                        rows[name]["scale"] = np.asarray(full[name + "_scale"]).reshape(-1)[:2].astype(np.float64).tolist()
            out["conversions"][q] = {
                "config": json.load(open(os.path.join(dst, "config.json"))),
                "header": header, "aliases": aliases,
                "variables": {k: {"dtype_id": v.dtype_id, "shape": list(v.shape)} for k, v in info.items()},
                "rows": rows,
                "num_heads": {side: int(np.asarray(full[f"{side}/num_heads"]).reshape(-1)[0])
                              for side in ("encoder", "decoder") if f"{side}/num_heads" in full},
            }
        # A generation config that lacks the heads and the begin-suppress list, with both in config.json: shows
        # whether the converter fills a missing key from config.json or takes generation_config.json alone.
        partial = os.path.join(tmp, "hf-partial")
        model.save_pretrained(partial)
        with open(os.path.join(partial, "generation_config.json")) as f:
            g = json.load(f)
        for k in ("alignment_heads", "begin_suppress_tokens"):
            g.pop(k, None)
        with open(os.path.join(partial, "generation_config.json"), "w") as f:
            json.dump(g, f)
        with open(os.path.join(partial, "config.json")) as f:
            c = json.load(f)
        c["alignment_heads"], c["begin_suppress_tokens"] = [[0, 1]], [220]
        with open(os.path.join(partial, "config.json"), "w") as f:
            json.dump(c, f)
        dst = os.path.join(tmp, "partial")
        ctranslate2.converters.TransformersConverter(partial).convert(dst, quantization="float16", force=True)
        out["partial_generation_config"] = json.load(open(os.path.join(dst, "config.json")))
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1)
    print(f"wrote {OUT}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
