"""Checkpoint layouts on the host: every reader yields, name for name, the values the fp32 path would upload; the
metadata a Hugging Face directory gives; the refusals; the hub file choice; footprints from headers; and the memory a
streamed read needs.  Fixtures are written at test time from ``random_init``."""
import json
import os

import numpy as np
import pytest
import torch

from tests.checkpoint_layouts import CT2_QUANT, HF_LAYOUTS, device_value, expected_f32, write_ct2, write_hf
from whisperlive_b200 import ct2_format
from whisperlive_b200 import weights as W
from whisperlive_b200.config import dims_for
from whisperlive_b200.weights import random_init

DIMS = dims_for("micro")


@pytest.fixture(scope="module")
def w():
    return random_init(DIMS, seed=7)


def _check_reader(path, want):
    ck = W.open_checkpoint(path)
    got = {}
    for name, a, scale in ck.tensors():
        assert name not in got, name
        assert ck.shapes[name] == a.shape, name
        got[name] = W.to_float32(a, scale)
    assert set(got) == set(want)
    for k, v in want.items():
        assert np.array_equal(device_value(k, got[k]), device_value(k, v)), k
    return ck


@pytest.mark.parametrize("layout", HF_LAYOUTS)
@pytest.mark.parametrize("dtype", ["float32", "float16", "bfloat16"])
def test_hf_layouts_give_the_stored_values(tmp_path, w, layout, dtype):
    p = write_hf(w, str(tmp_path / "m"), layout, dtype, prefix=layout != "bin")
    ck = _check_reader(p, expected_f32(w, "hf", dtype))
    assert ck.layout == layout
    # the fp32 dict of the existing path holds the same values
    old = W.load_model_dir(p)
    assert all(np.array_equal(old[k].numpy(), expected_f32(w, "hf", dtype)[k]) for k in w)


@pytest.mark.parametrize("quant", CT2_QUANT)
def test_ct2_quantizations_give_the_stored_values(tmp_path, w, quant):
    p = write_ct2(w, str(tmp_path / "m"), quant)
    ck = _check_reader(p, expected_f32(w, "ct2", quant))
    arrays = {n: (a, s) for n, a, s in ck.tensors()}
    a, s = arrays["model.decoder.layers.0.self_attn.k_proj.weight"]
    if quant.startswith("int8"):
        assert a.dtype == np.int8 and s.shape == (a.shape[0],)
        host = a.astype(np.float32) / W.to_float32(s).reshape(-1, 1)
        assert np.array_equal(host.astype(np.float16), W.to_float32(a, s).astype(np.float16))
    else:
        assert s is None


def test_safetensors_preferred_over_bin(tmp_path, w):
    p = str(tmp_path / "m")
    write_hf(w, p, "bin", "float32")
    write_hf(w, p, "safetensors-sharded", "float16")
    assert W.open_checkpoint(p).layout == "safetensors-sharded"


def test_save_pretrained_layouts_match_hand_written(tmp_path, w):
    transformers = pytest.importorskip("transformers")
    cfg = transformers.WhisperConfig(vocab_size=DIMS.vocab, num_mel_bins=DIMS.n_mels, d_model=DIMS.d_model,
                                     encoder_layers=DIMS.enc_layers, decoder_layers=DIMS.dec_layers,
                                     encoder_attention_heads=DIMS.n_heads, decoder_attention_heads=DIMS.n_heads,
                                     encoder_ffn_dim=DIMS.d_ff, decoder_ffn_dim=DIMS.d_ff, max_source_positions=1500,
                                     max_target_positions=448)
    model = transformers.WhisperForConditionalGeneration(cfg)
    sd = {k: v for k, v in w.items()}
    sd["proj_out.weight"] = w["model.decoder.embed_tokens.weight"]
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    for k in missing:   # Whisper's k_proj has no bias; anything else missing is a fixture error
        assert k.endswith("k_proj.bias") or k == "proj_out.weight", k
    model = model.to(torch.bfloat16)
    out = str(tmp_path / "pretrained")
    model.save_pretrained(out, max_shard_size="300KB")
    ck = W.open_checkpoint(out)
    assert ck.layout in ("safetensors", "safetensors-sharded")
    mine = W.open_checkpoint(write_hf(w, str(tmp_path / "mine"), "safetensors-sharded", "bfloat16"))
    theirs = {n: W.to_float32(a) for n, a, _ in ck.tensors()}
    for n, a, _ in mine.tensors():
        assert np.array_equal(theirs[n], W.to_float32(a)), n


# ------------------------------------------------------------------------------------------ metadata
def test_metadata_from_generation_config(tmp_path, w):
    p = write_hf(w, str(tmp_path / "m"), "safetensors", "float16")
    with open(os.path.join(p, "config.json"), "w") as f:
        json.dump({"suppress_tokens": [1, 2], "begin_suppress_tokens": [220, 50257], "alignment_heads": [[0, 0]]}, f)
    with open(os.path.join(p, "generation_config.json"), "w") as f:
        json.dump({"alignment_heads": [[1, 0], [1, 1]], "suppress_tokens": [3, 4, 5],
                   "lang_to_id": {"<|fr|>": 50265, "<|en|>": 50259}}, f)
    meta = W.model_metadata(p)   # a generation config is read alone: config.json fills none of its gaps
    assert meta == {"alignment_heads": [(1, 0), (1, 1)], "suppress_ids": [3, 4, 5], "lang_ids": [50259, 50265]}
    os.remove(os.path.join(p, "generation_config.json"))
    assert W.model_metadata(p) == {"alignment_heads": [(0, 0)], "suppress_ids": [1, 2], "suppress_ids_begin": [220, 50257]}


def test_metadata_of_a_ct2_directory_is_its_config(tmp_path, w):
    p = write_ct2(w, str(tmp_path / "m"), "int8_float16")
    with open(os.path.join(p, "config.json"), "w") as f:
        json.dump({"alignment_heads": [[1, 1]], "lang_ids": [5], "suppress_ids": [7], "suppress_ids_begin": [8]}, f)
    assert W.model_metadata(p) == {"alignment_heads": [(1, 1)], "lang_ids": [5], "suppress_ids": [7],
                                   "suppress_ids_begin": [8]}


# ------------------------------------------------------------------------------------------ refusals by name
def test_untied_head_is_refused(tmp_path, w):
    from safetensors.torch import save_file
    sd = {k: v.half() for k, v in w.items()}
    sd["proj_out.weight"] = sd["model.decoder.embed_tokens.weight"].clone()
    p = tmp_path / "tied"
    p.mkdir()
    save_file(sd, str(p / "model.safetensors"))
    assert "model.proj_out.weight" not in {n for n, _, _ in W.open_checkpoint(str(p)).tensors()}
    sd["proj_out.weight"][0, 0] += 1
    p = tmp_path / "untied"
    p.mkdir()
    save_file(sd, str(p / "model.safetensors"))
    with pytest.raises(ValueError, match="proj_out.weight"):
        next(W.open_checkpoint(str(p)).tensors())


def test_int16_is_refused(tmp_path, w):
    p = write_ct2(w, str(tmp_path / "m"), "int16")
    with pytest.raises(ValueError, match="int16"):
        W.open_checkpoint(p)


def test_wrong_positions_are_refused(tmp_path, w):
    bad = dict(w)
    bad["model.decoder.embed_positions.weight"] = w["model.decoder.embed_positions.weight"][:400]
    with pytest.raises(ValueError, match="decoder.embed_positions.weight has 400 positions"):
        W.open_checkpoint(write_hf(bad, str(tmp_path / "a"), "safetensors"))
    p = write_hf(w, str(tmp_path / "b"), "safetensors")
    with open(os.path.join(p, "config.json"), "w") as f:
        json.dump({"max_target_positions": 512}, f)
    with pytest.raises(ValueError, match="max_target_positions"):
        W.open_checkpoint(p)
    with open(os.path.join(p, "config.json"), "w") as f:
        json.dump({"d_model": 128, "encoder_attention_heads": 4}, f)
    with pytest.raises(ValueError, match="head dimension"):
        W.open_checkpoint(p)


def test_ct2_head_width_is_refused(tmp_path, w):
    p = write_ct2(w, str(tmp_path / "m"), "float16")
    variables, aliases, _ = ct2_format.read_variables(os.path.join(p, "model.bin"))
    assert int(np.asarray(variables["decoder/num_heads"]).reshape(-1)[0]) == DIMS.n_heads
    variables["decoder/num_heads"] = np.asarray(4, np.int16)      # 32-wide heads at d_model 128
    ct2_format.write_variables(os.path.join(p, "model.bin"), variables, aliases)
    with pytest.raises(ValueError, match="decoder/num_heads = 4"):
        W.open_checkpoint(p)


def test_missing_shard_is_refused(tmp_path, w):
    p = write_hf(w, str(tmp_path / "m"), "safetensors-sharded")
    os.remove(os.path.join(p, "model-00002-of-00003.safetensors"))
    with pytest.raises(FileNotFoundError, match="model-00002-of-00003.safetensors"):
        W.open_checkpoint(p)


def test_missing_scale_is_refused(tmp_path, w):
    p = write_ct2(w, str(tmp_path / "m"), "int8_float16")
    variables, aliases, _ = ct2_format.read_variables(os.path.join(p, "model.bin"))
    del variables["decoder/layer_1/ffn/linear_0/weight_scale"]
    ct2_format.write_variables(os.path.join(p, "model.bin"), variables, aliases)
    with pytest.raises(ValueError, match="decoder/layer_1/ffn/linear_0/weight_scale"):
        W.open_checkpoint(p)


def test_header_only_read_matches_full_read(tmp_path, w):
    p = write_ct2(w, str(tmp_path / "m"), "int8_bfloat16")
    full, aliases, head = ct2_format.read_variables(os.path.join(p, "model.bin"))
    info, aliases2, head2 = ct2_format.read_variables(os.path.join(p, "model.bin"), header_only=True)
    assert aliases == aliases2 and head == head2 and set(full) == set(info)
    assert all(tuple(full[k].shape) == info[k].shape for k in full)


# ------------------------------------------------------------------------------------------ hub file choice
def test_hub_allow_patterns_fetch_one_copy_of_the_weights():
    meta = ["config.json", "generation_config.json", "preprocessor_config.json", "tokenizer.json", "vocabulary.*"]
    both = ["config.json", "model.safetensors", "pytorch_model.bin", "flax_model.msgpack", "tf_model.h5", "README.md"]
    assert W.hub_allow_patterns(both) == meta + ["model.safetensors"]
    sharded = ["model.safetensors.index.json", "model-00001-of-00002.safetensors", "model-00002-of-00002.safetensors",
               "pytorch_model.bin.index.json", "pytorch_model-00001-of-00002.bin", "pytorch_model-00002-of-00002.bin"]
    assert W.hub_allow_patterns(sharded) == meta + sorted(sharded[:3])
    assert W.hub_allow_patterns(["pytorch_model.bin", "config.json"]) == meta + ["pytorch_model.bin"]
    assert W.hub_allow_patterns(sharded[3:]) == meta + sorted(sharded[3:])
    assert W.hub_allow_patterns(["model.bin", "config.json", "vocabulary.json"]) == meta + ["model.bin"]
    assert "model.bin" in W.hub_allow_patterns(None)


def test_hub_resolution_downloads_only_from_the_file_list(monkeypatch):
    """When the repository cannot be listed nothing is downloaded; a snapshot on disk may still resolve."""
    import huggingface_hub
    calls = []

    def snapshot(repo, **kw):
        calls.append(kw)
        raise OSError("not cached")

    def no_list(repo):
        raise OSError("offline")
    monkeypatch.setattr(huggingface_hub, "snapshot_download", snapshot)
    monkeypatch.setattr(huggingface_hub, "list_repo_files", no_list)
    with pytest.raises(FileNotFoundError, match="offline"):
        W.resolve_model_dir("tiny.en")
    assert calls and all(kw.get("local_files_only") for kw in calls)
    calls.clear()
    monkeypatch.setattr(huggingface_hub, "list_repo_files", lambda repo: ["model.safetensors", "pytorch_model.bin"])
    with pytest.raises(FileNotFoundError):
        W.resolve_model_dir("openai/whisper-tiny")
    online = [kw for kw in calls if not kw.get("local_files_only")]
    assert len(online) == 1 and "pytorch_model.bin" not in online[0]["allow_patterns"]


# ------------------------------------------------------------------------------------------ footprint from headers
@pytest.mark.parametrize("fmt", ["safetensors-sharded", "bin", "ct2"])
def test_footprint_from_headers(tmp_path, w, fmt):
    from whisperlive_b200.engine import footprint_estimate
    from whisperlive_b200.models import engine_footprint
    p = write_ct2(w, str(tmp_path / "m"), "int8_float16") if fmt == "ct2" else write_hf(w, str(tmp_path / "m"), fmt)
    assert engine_footprint(p, max_streams=4) == footprint_estimate(DIMS, max_streams=4)
    empty = tmp_path / "empty"
    empty.mkdir()
    assert engine_footprint(str(empty)) is None
    broken = tmp_path / "broken"
    broken.mkdir()
    (broken / "pytorch_model.bin").write_bytes(b"not a torch file")
    assert engine_footprint(str(broken)) is None


# ------------------------------------------------------------------------------------------ streaming bound
class _Live:
    """Bytes of tensors safetensors has materialised that the consumer has not finished with, and their peak."""

    def __init__(self):
        self.bytes = self.peak = 0

    def add(self, n):
        self.bytes += n
        self.peak = max(self.peak, self.bytes)


class _CountingHandle:
    def __init__(self, real, live):
        self._real, self._live = real, live

    def get_tensor(self, key):
        t = self._real.get_tensor(key)
        self._live.add(t.numel() * t.element_size())
        return t

    def __getattr__(self, name):
        return getattr(self._real, name)


def _read_peak(monkeypatch, path, materialise_first):
    import safetensors
    live, real_open = _Live(), safetensors.safe_open
    monkeypatch.setattr(safetensors, "safe_open", lambda *a, **k: _CountingHandle(real_open(*a, **k), live))
    it = W.open_checkpoint(path).tensors()
    if materialise_first:   # what a reader that is not streaming does
        it = list(it)
    for name, a, scale in it:
        np.ascontiguousarray(a)            # what the upload hands to the library
        live.bytes -= a.nbytes             # done with it
    monkeypatch.setattr(safetensors, "safe_open", real_open)
    return live.peak


def test_streamed_read_peaks_below_twice_the_largest_tensor(tmp_path, w, monkeypatch):
    small = dict(w)   # a 1024-token embedding, so that no single tensor is most of the checkpoint
    small["model.decoder.embed_tokens.weight"] = w["model.decoder.embed_tokens.weight"][:1024]
    p = write_hf(small, str(tmp_path / "m"), "safetensors-sharded", "float32", n_shards=4)
    largest = max(v.numel() * 4 for v in small.values())
    total = sum(v.numel() * 4 for v in small.values())
    assert total > 4 * largest
    peak = _read_peak(monkeypatch, p, materialise_first=False)
    assert largest <= peak < 2 * largest, (peak, largest, total)
    # the measure sees a reader that holds the whole checkpoint
    assert _read_peak(monkeypatch, p, materialise_first=True) == total
