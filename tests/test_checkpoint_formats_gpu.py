"""Checkpoint layouts on the H100: every layout loads through ``B200Whisper.from_model`` into the device weights the
fp32 path makes from the same values; the typed-upload conversion kernels against numpy; the fp16 overflow refusal;
alignment heads from ``generation_config.json``; word-timestamped transcription from a sharded bf16 directory."""
import json
import os

import numpy as np
import pytest
import torch

from tests.checkpoint_layouts import device_value, expected_f32, write_ct2, write_hf
from whisperlive_b200 import _lib, synth
from whisperlive_b200 import weights as W
from whisperlive_b200.config import dims_for
from whisperlive_b200.tokenizer import build_synthetic_tokenizer
from whisperlive_b200.weights import random_init

pytestmark = pytest.mark.gpu

DIMS = dims_for("micro.en")


def _finish_dir(path, dims=DIMS, config=None):
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(config if config is not None else {}, f)
    with open(os.path.join(path, "preprocessor_config.json"), "w") as f:
        json.dump({"feature_size": dims.n_mels, "sampling_rate": 16000, "hop_length": 160, "chunk_length": 30,
                   "n_fft": 400}, f)
    build_synthetic_tokenizer(dims.vocab).save(os.path.join(path, "tokenizer.json"))
    return path


def _feats(dims, seconds, seed):
    from oracle import mel as omel
    return omel.pad_or_trim(omel.log_mel(synth.speech_like(seconds, seed=seed), dims.n_mels)[:, :-1])


LAYOUTS = [("safetensors", "float16"), ("safetensors-sharded", "bfloat16"), ("bin", "float32"),
           ("bin-sharded", "float16"), ("ct2", "float16"), ("ct2", "bfloat16"), ("ct2", "int8_float16"), ("ct2", "int8")]


@pytest.mark.parametrize("fmt,dtype", LAYOUTS)
def test_layout_loads_like_the_same_values_in_memory(tmp_path, fmt, dtype):
    from whisperlive_b200.engine import B200Whisper
    w = random_init(DIMS, seed=4)
    p = str(tmp_path / "m")
    write_ct2(w, p, dtype) if fmt == "ct2" else write_hf(w, p, fmt, dtype)
    _finish_dir(p)
    eng = B200Whisper.from_model(p, max_streams=2, max_beam=5)
    ref = B200Whisper(DIMS, {k: torch.from_numpy(v) for k, v in expected_f32(w, fmt, dtype).items()}, max_streams=2,
                      max_beam=5)
    assert eng.device_bytes == ref.device_bytes      # the staging buffers are gone after finalize
    feats = np.stack([_feats(DIMS, 5.0, 1), _feats(DIMS, 8.0, 2)])
    a, b = eng.encode(feats), ref.encode(feats)
    assert np.array_equal(np.asarray(a), np.asarray(b))
    prompts = [[eng.sot]] * 2
    ga = eng.generate(a, prompts, beam_size=5, max_length=64)
    gb = ref.generate(b, prompts, beam_size=5, max_length=64)
    assert [g.sequences_ids for g in ga] == [g.sequences_ids for g in gb]


class _Unloaded:
    """A context with no weights: tensors go in through wl_load_tensor_typed and come back through
    wl_test_read_weight, and wl_finalize_weights is never called."""

    def __init__(self):
        from whisperlive_b200.engine import B200Whisper

        class NoLoad(B200Whisper):
            def _load_weights(self, weights):
                pass
        self.eng = NoLoad(DIMS, {}, max_streams=1, max_beam=1)

    def read(self, name, shape, f32):
        out = np.empty(shape, np.float32 if f32 else np.uint16)
        _lib.check(self.eng.lib, self.eng.ctx, self.eng.lib.wl_test_read_weight(self.eng.ctx, name.encode(),
                                                                                out.ctypes.data), "read")
        return out


def _source(rng, shape, kind):
    x = rng.standard_normal(shape).astype(np.float32)
    x.reshape(-1)[::7] *= 1e-6        # fp16 subnormals and values that flush to zero
    x.reshape(-1)[::11] *= 3e3        # large but finite in fp16
    if kind == "f32":
        return x, None
    if kind == "f16":
        return x.astype(np.float16), None
    if kind == "bf16":
        return torch.from_numpy(x).bfloat16().view(torch.int16).numpy().view(W.BF16), None
    sdt = kind.split("_")[1]
    q = rng.integers(-127, 128, size=shape).astype(np.int8)
    s = (127.0 / (rng.random(shape[0]) * 3 + 1e-3)).astype(np.float32)
    s = {"f32": s, "f16": s.astype(np.float16),
         "bf16": torch.from_numpy(s).bfloat16().view(torch.int16).numpy().view(W.BF16)}[sdt]
    return q, s


CONVERT_CASES = [((37, 13), "f32"), ((37, 13), "f16"), ((37, 13), "bf16"), ((33, 17), "i8_f32"), ((5, 41), "i8_f16"),
                 ((29, 3), "i8_bf16"), ((1, 7), "f16"), ((129, 257), "bf16"), ((1001,), "f32"), ((1001,), "bf16"),
                 ((7,), "i8_f32"), ((6, 5, 3), "f32"), ((6, 5, 3), "bf16"), ((6, 5, 3), "i8_f16"), ((11, 80, 3), "f16"),
                 ((1500, 9), "f16")]


def test_conversion_kernels_bit_exact_against_numpy():
    ctx = _Unloaded()
    rng = np.random.default_rng(0)
    for i, (shape, kind) in enumerate(CONVERT_CASES):
        name = "model.encoder.embed_positions.weight" if shape == (1500, 9) else f"t{i}"
        a, s = _source(rng, shape, kind)
        ctx.eng._load_typed(name, a, s)
        want = device_value(name, W.to_float32(a, s))
        if want.ndim == 3 and want.dtype == np.float16:
            want = np.ascontiguousarray(want.transpose(0, 2, 1))     # [co][ci][k] -> [co][k][ci]
        got = ctx.read(name, want.shape, want.dtype == np.float32)
        assert np.array_equal(got.view(np.uint32 if want.dtype == np.float32 else np.uint16),
                              want.view(np.uint32 if want.dtype == np.float32 else np.uint16)), (shape, kind)


def test_fp16_overflow_is_refused_by_name():
    ctx = _Unloaded()
    x = np.ones((4, 9), np.float32)
    x[2, 3], x[3, 8] = 70000.0, -1e6
    bf = torch.from_numpy(x).bfloat16().view(torch.int16).numpy().view(W.BF16)
    with pytest.raises(_lib.WlError, match=r"decoder\.layers\.0\.fc1\.weight.*2 finite values"):
        ctx.eng._load_typed("model.decoder.layers.0.fc1.weight", bf, None)
    with pytest.raises(_lib.WlError, match="no weight"):
        ctx.read("model.decoder.layers.0.fc1.weight", (4, 9), False)
    ctx.eng._load_typed("ok", bf[:2], None)       # the context is still usable


def test_alignment_heads_from_generation_config(tmp_path):
    from whisperlive_b200.engine import B200Whisper
    w = random_init(DIMS, seed=5)
    p = _finish_dir(write_hf(w, str(tmp_path / "m"), "safetensors", "float16"))
    with open(os.path.join(p, "generation_config.json"), "w") as f:
        json.dump({"alignment_heads": [[1, 1], [0, 1]], "suppress_tokens": [1, 2], "begin_suppress_tokens": [220]}, f)
    eng = B200Whisper.from_model(p, max_streams=1, max_beam=1)
    assert eng.alignment_heads == [(1, 1), (0, 1)]
    assert eng.model_metadata["suppress_ids_begin"] == [220]


def test_sharded_bf16_transcribes_like_single_fp16(tmp_path):
    from whisperlive_b200.transcriber import B200WhisperModel
    w = random_init(DIMS, seed=6)
    # values both bf16 and fp16 hold exactly: bf16-rounded, nothing below fp16's smallest normal
    both = {k: torch.where(v.abs() < 2.0 ** -14, torch.zeros_like(v), v.bfloat16().float()) for k, v in w.items()}
    a = _finish_dir(write_hf(both, str(tmp_path / "bf16"), "safetensors-sharded", "bfloat16"))
    b = _finish_dir(write_hf(both, str(tmp_path / "f16"), "safetensors", "float16"))
    audio = synth.speech_like(9.0, seed=3)
    out = []
    for p in (a, b):
        model = B200WhisperModel(p, max_streams=2, max_beam=5)
        segs, info = model.transcribe(audio, beam_size=5, temperature=[0.0], word_timestamps=True, log_prob_threshold=None)
        segs = list(segs)
        out.append([(s.text, s.start, s.end, [(x.word, x.start, x.end, x.probability) for x in (s.words or [])])
                    for s in segs])
        del model
    assert out[0] == out[1] and len(out[0]) > 0
