"""Host side of the device translator (whisperlive_b200/translation.py) and its float64 oracle; no GPU needed."""
from __future__ import annotations

import json
import os
import queue
import threading
import time

import numpy as np
import pytest
import torch

from tests import mt_oracle as O
from whisperlive_b200 import translation as T

MICRO = T.MtConfig(d_model=128, n_heads=2, enc_layers=2, dec_layers=1, ffn=512, vocab=1000, max_positions=1024)


# ------------------------------------------------------------------------------------------------ settings
@pytest.mark.parametrize("name,value", [("do_sample", True), ("no_repeat_ngram_size", 3), ("repetition_penalty", 1.2),
                                        ("min_length", 5), ("top_k", 10), ("num_beam_groups", 2)])
def test_unsupported_generation_setting_raises_by_name(name, value):
    with pytest.raises(ValueError, match=name):
        T.generation_settings({name: value})


def test_generation_settings_from_generation_config_and_config():
    g = T.generation_settings({"num_beams": 5, "max_length": 200, "early_stopping": True, "decoder_start_token_id": 2,
                               "eos_token_id": 2, "pad_token_id": 1, "forced_eos_token_id": 2})
    assert (g.num_beams, g.max_length, g.early_stopping, g.forced_eos_token_id) == (5, 200, True, 2)
    # no generation_config.json: the generation attributes of config.json
    g = T.generation_settings(None, {"num_beams": 4, "max_length": 50, "d_model": 1024, "eos_token_id": 2})
    assert (g.num_beams, g.max_length) == (4, 50)
    assert T.generation_settings({"max_new_tokens": 30}).max_length == 31


def test_length_limits_raise_with_the_limit():
    with pytest.raises(ValueError, match="448"):
        T.generation_settings({"max_length": 449})
    with pytest.raises(ValueError, match="1022"):
        T.check_source_length(1023, T.MtConfig(**T.SMALL100_SHAPE))
    T.check_source_length(1022, T.MtConfig(**T.SMALL100_SHAPE))
    with pytest.raises(ValueError, match="num_beams"):
        T.generation_settings({"num_beams": 9})


def test_config_from_json_rejects_what_the_engine_lacks():
    base = {"d_model": 128, "encoder_attention_heads": 2, "decoder_attention_heads": 2, "encoder_layers": 2, "decoder_layers": 1,
            "encoder_ffn_dim": 512, "decoder_ffn_dim": 512, "vocab_size": 1000, "max_position_embeddings": 1024,
            "scale_embedding": True, "activation_function": "relu"}
    assert T.config_from_json(base) == MICRO
    with pytest.raises(ValueError, match="activation_function"):
        T.config_from_json({**base, "activation_function": "gelu"})
    with pytest.raises(ValueError, match="decoder_attention_heads"):
        T.config_from_json({**base, "decoder_attention_heads": 4})


# ------------------------------------------------------------------------------------------------ checkpoint
def _save(tmp_path, sd, fmt):
    if fmt == "bin":
        p = tmp_path / "pytorch_model.bin"
        torch.save(sd, p)
    else:
        from safetensors.torch import save_file
        p = tmp_path / "model.safetensors"
        save_file({k: v.contiguous() for k, v in sd.items()}, str(p))
    return str(tmp_path)


@pytest.mark.parametrize("fmt", ["bin", "safetensors"])
def test_checkpoint_reader_round_trip_and_tied_head(tmp_path, fmt):
    ck = T.random_checkpoint(MICRO, seed=1)
    sd = {k: torch.from_numpy(v.copy()) for k, v in ck.items()}
    sd["lm_head.weight"] = sd["model.shared.weight"].clone()
    sd["model.encoder.embed_tokens.weight"] = sd["model.shared.weight"].clone()
    got = T.read_checkpoint(_save(tmp_path, sd, fmt), MICRO)
    assert set(got) == set(ck)
    for k in ck:
        assert np.array_equal(got[k], ck[k]), k


def test_checkpoint_reader_rejects_by_name(tmp_path):
    ck = T.random_checkpoint(MICRO, seed=1)
    sd = {k: torch.from_numpy(v.copy()) for k, v in ck.items()}
    name = "model.decoder.layers.0.encoder_attn.k_proj.weight"
    bad = dict(sd)
    del bad[name]
    with pytest.raises(ValueError, match=name.replace(".", r"\.")):
        T.read_checkpoint(_save(tmp_path, bad, "bin"), MICRO)
    bad = dict(sd)
    bad[name] = torch.zeros(3, 3)
    with pytest.raises(ValueError, match="shape"):
        T.read_checkpoint(_save(tmp_path, bad, "bin"), MICRO)
    bad = dict(sd)
    bad[name] = torch.zeros(128, 128, dtype=torch.int32)
    with pytest.raises(ValueError, match="dtype"):
        T.read_checkpoint(_save(tmp_path, bad, "bin"), MICRO)
    bad = dict(sd)
    bad["lm_head.weight"] = sd["model.shared.weight"] + 1
    with pytest.raises(ValueError, match="tied"):
        T.read_checkpoint(_save(tmp_path, bad, "bin"), MICRO)


def test_resolve_snapshot_never_substitutes(tmp_path, monkeypatch):
    monkeypatch.setenv("WLB200_MT_MODEL", str(tmp_path / "absent"))
    with pytest.raises(FileNotFoundError):
        T.resolve_snapshot()
    monkeypatch.setenv("WLB200_MT_MODEL", str(tmp_path))
    assert T.resolve_snapshot() == str(tmp_path)


def test_engine_tensors_cover_the_engine_table():
    et = T.engine_tensors(T.random_checkpoint(MICRO, 2), MICRO)
    d = MICRO.d_model
    assert et["enc.0.qkv.w"].shape == (3 * d, d) and et["dec.xkv.w"].shape == (2 * d * MICRO.dec_layers, d)
    assert et["positions"].shape == (MICRO.max_positions + 2, d) and not et["positions"][MICRO.pad_id].any()
    assert len(et) == 2 + MICRO.enc_layers * 12 + 2 + MICRO.dec_layers * 18 + 2 + 2


# ------------------------------------------------------------------------------------------------ oracle vs Hugging Face
def _hf_model(ck, cfg):
    tr = pytest.importorskip("transformers")
    hc = tr.M2M100Config(vocab_size=cfg.vocab, d_model=cfg.d_model, encoder_layers=cfg.enc_layers, decoder_layers=cfg.dec_layers,
                         encoder_attention_heads=cfg.n_heads, decoder_attention_heads=cfg.n_heads, encoder_ffn_dim=cfg.ffn,
                         decoder_ffn_dim=cfg.ffn, max_position_embeddings=cfg.max_positions, scale_embedding=True,
                         dropout=0.0, attention_dropout=0.0, activation_dropout=0.0)
    m = tr.M2M100ForConditionalGeneration(hc).eval()
    missing, _ = m.load_state_dict({k: torch.from_numpy(v) for k, v in ck.items()}, strict=False)
    assert all("embed_tokens" in k or "lm_head" in k for k in missing), missing
    m.tie_weights()
    return m


def test_oracle_logits_and_beam_search_match_hugging_face():
    ck = T.random_checkpoint(MICRO, seed=5)
    m = _hf_model(ck, MICRO)
    orc = O.OracleM2M100(ck, MICRO)
    src = [905, 17, 230, 4, 99, 2]
    dec = [2, 905, 40, 41]
    with torch.no_grad():
        ref = m(input_ids=torch.tensor([src]), decoder_input_ids=torch.tensor([dec])).logits[0].double().numpy()
    got = orc.decoder_logits(orc.encode(src), dec)
    assert np.abs(got - ref).max() < 1e-4 * max(1.0, np.abs(ref).max())
    for gen in (T.GenSettings(num_beams=5, max_length=12), T.GenSettings(num_beams=5, max_length=12, early_stopping=True),
                T.GenSettings(num_beams=4, max_length=12, early_stopping="never", length_penalty=2.0),
                T.GenSettings(num_beams=1, max_length=12)):
        with torch.no_grad():
            out = m.generate(input_ids=torch.tensor([src]), num_beams=gen.num_beams, max_length=gen.max_length,
                             early_stopping=gen.early_stopping, length_penalty=gen.length_penalty, do_sample=False,
                             decoder_start_token_id=2, eos_token_id=2, pad_token_id=1, return_dict_in_generate=True,
                             output_scores=True)
        hf = out.sequences[0].tolist()[1:]
        r = orc.generate(src, gen)
        assert r.tokens == hf, (gen, r.tokens, hf)
        if gen.num_beams > 1:
            assert abs(float(out.sequences_scores[0]) - float(r.score)) < 1e-4


# ------------------------------------------------------------------------------------------------ tokenizer
@pytest.fixture(scope="module")
def tok_dir(tmp_path_factory):
    spm = pytest.importorskip("sentencepiece")
    d = tmp_path_factory.mktemp("small100_tok")
    rng = np.random.default_rng(0)
    words = ["hello", "world", "speech", "live", "whisper", "translate", "segment", "the", "a", "of", "good", "morning"]
    corpus = d / "corpus.txt"
    corpus.write_text("\n".join(" ".join(rng.choice(words, 8)) for _ in range(400)) + "\n")
    spm.SentencePieceTrainer.train(input=str(corpus), model_prefix=str(d / "sentencepiece.bpe"), vocab_size=60,
                                   model_type="bpe", num_threads=1, character_coverage=1.0)
    sp = spm.SentencePieceProcessor()
    sp.Load(str(d / "sentencepiece.bpe.model"))
    vocab = {"<s>": 0, "<pad>": 1, "</s>": 2, "<unk>": 3}
    for i in range(sp.get_piece_size()):
        p = sp.id_to_piece(i)
        if p not in vocab and p not in ("<unk>", "<s>", "</s>"):
            vocab[p] = len(vocab)
    del vocab[sp.id_to_piece(sp.get_piece_size() - 1)]   # one piece the vocabulary lacks: it maps to <unk>
    (d / "vocab.json").write_text(json.dumps(vocab))
    return str(d)


def test_tokenizer_layout(tok_dir):
    tok = T.Small100Tokenizer.from_dir(tok_dir)
    n = len(tok.encoder)
    ids = tok.encode("hello world", "fr")
    assert ids[0] == n + T.FAIRSEQ_LANGUAGE_CODES.index("fr") and ids[-1] == 2
    assert tok.encode("", "de") == [n + T.FAIRSEQ_LANGUAGE_CODES.index("de"), 2]
    assert tok.decode(ids) == "hello world"
    assert tok.decode([ids[0], 0, 1] + ids[1:]) == "hello world"     # special tokens skipped
    with pytest.raises(KeyError):
        tok.encode("hello", "xx")


# ------------------------------------------------------------------------------------------------ worker and client
class StubEngine:
    capacity = 64

    def __init__(self, delay=0.0):
        self.calls, self.delay = [], delay

    def translate_batch(self, texts, langs):
        self.calls.append(list(texts))
        time.sleep(self.delay)
        return [f"[{l}]{t}" if t.strip() else t for t, l in zip(texts, langs)]


def test_worker_coalesces_pending_requests_into_one_call():
    eng = StubEngine(delay=0.2)
    w = T.TranslationWorker(lambda: eng)
    w.submit("warm", "fr")                      # loads the engine; the next requests queue behind a busy call
    gate = threading.Event()
    res = {}

    def client(i):
        gate.wait()
        res[i] = w.submit(f"t{i}", "de")
    hold = threading.Thread(target=lambda: w.submit("busy", "fr"))
    hold.start()
    time.sleep(0.05)
    ths = [threading.Thread(target=client, args=(i,)) for i in range(12)]
    for t in ths:
        t.start()
    gate.set()
    for t in ths + [hold]:
        t.join()
    assert res == {i: f"[de]t{i}" for i in range(12)}
    assert len(eng.calls) == 3 and sorted(eng.calls[2]) == sorted(f"t{i}" for i in range(12))


def test_worker_failing_call_fails_only_its_requests():
    class Flaky(StubEngine):
        def translate_batch(self, texts, langs):
            if "boom" in texts:
                raise RuntimeError("boom")
            return super().translate_batch(texts, langs)
    w = T.TranslationWorker(lambda: Flaky())
    with pytest.raises(RuntimeError):
        w.submit("boom", "fr")
    assert w.submit("ok", "fr") == "[fr]ok"


class FakeSocket:
    def __init__(self):
        self.sent = []

    def send(self, msg):
        self.sent.append(json.loads(msg))


def test_client_messages_and_fallbacks():
    w = T.TranslationWorker(lambda: StubEngine())
    q = queue.Queue()
    ws = FakeSocket()
    c = T.DeviceTranslationClient("uid1", ws, q, target_language="fr", send_last_n_segments=2, worker=w)
    segs = [{"start": "0.0", "end": "1.0", "text": "hello", "completed": True},
            {"start": "1.0", "end": "2.0", "text": "partial", "completed": False},
            {"start": "2.0", "end": "3.0", "text": "   ", "completed": True},
            {"start": "3.0", "end": "4.0", "text": "world", "completed": True}]
    for s in segs:
        q.put(s)
    q.put(None)
    th = threading.Thread(target=c.speech_to_text)
    th.start()
    th.join(10)
    assert [m["uid"] for m in ws.sent] == ["uid1"] * 3
    assert ws.sent[0]["translated_segments"] == [{"start": "0.0", "end": "1.0", "text": "[fr]hello", "completed": True,
                                                  "target_language": "fr"}]
    assert [s["text"] for s in ws.sent[-1]["translated_segments"]] == ["   ", "[fr]world"]   # last n = 2
    c.set_target_language("de")
    assert c.translate_text("x") == "[de]x"
    bad = T.DeviceTranslationClient("uid2", FakeSocket(), queue.Queue(), target_language="xx", worker=w)
    assert not bad.model_loaded and bad.translate_text("hello") == "hello"
    c.cleanup()
    assert c.translated_segments == [] and c.exit


def test_switch_reads_the_environment(monkeypatch):
    monkeypatch.delenv("WLB200_TRANSLATE", raising=False)
    assert T.translate_mode() == "cpu"
    monkeypatch.setenv("WLB200_TRANSLATE", "device")
    assert T.translate_mode() == "device"
    monkeypatch.setenv("WLB200_TRANSLATE", "gpu")
    with pytest.raises(ValueError):
        T.translate_mode()


# ------------------------------------------------------------------------------------------------ pins against the reference
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
MICRO_DIR = os.path.join(GOLDEN, "small100_micro")


def _reference():
    with open(os.path.join(GOLDEN, "translate_reference.json")) as f:
        return json.load(f)


def _micro_cfg():
    with open(os.path.join(MICRO_DIR, "config.json")) as f:
        return T.config_from_json(json.load(f))


def test_tokenizer_matches_the_reference_tokenizer():
    pytest.importorskip("sentencepiece")
    tok = T.Small100Tokenizer.from_dir(MICRO_DIR)
    ref = _reference()["tokenizer"]
    n = len(tok.encoder)
    assert any(3 in r["ids"] for r in ref)            # an unknown piece is exercised
    for r in ref:
        ids = tok.encode(r["text"], r["lang"])
        assert ids == r["ids"], r
        assert tok.decode(ids) == r["decoded"], r
        assert tok.decode(ids + [0, 1, 3, n + 5, n + 100, n + 107]) == r["decoded_extra"], r


def test_oracle_matches_hugging_face_fixture():
    cfg = _micro_cfg()
    z = np.load(os.path.join(GOLDEN, "mt_hf.npz"))
    orc = O.OracleM2M100(T.random_checkpoint(cfg, _reference()["seed"]), cfg)
    prefix = z["prefix"].tolist()
    for i in range(3):
        src = z[f"src{i}"].tolist()
        ref = z[f"logits{i}"].astype(np.float64)
        got = orc.decoder_logits(orc.encode(src), prefix)
        assert np.abs(got - ref).max() < 1e-4 * max(1.0, np.abs(ref).max()), i
        for name, st in _reference()["translate"].items():
            gen = T.GenSettings(**{**dict(early_stopping=False, length_penalty=1.0), **st["settings"]})
            r = orc.generate(src, gen)
            assert r.tokens == z[f"seq{i}_{name}"].tolist()[1:], (i, name)
            if gen.num_beams > 1:
                assert abs(float(r.score) - float(z[f"score{i}_{name}"][0])) < 1e-4, (i, name)


class RecordedEngine:
    """Answers with the reference's own translate_text results (recorded under its default generation settings)."""
    capacity = 64

    def __init__(self, table):
        self.table, self.calls = table, 0

    def translate_batch(self, texts, langs):
        self.calls += 1
        out = []
        for t, lang in zip(texts, langs):
            if not t.strip():
                out.append(t)
            elif lang not in T.FAIRSEQ_LANGUAGE_CODES:
                out.append(KeyError(lang))
            else:
                out.append(self.table[(t, lang)])
        return out


def _run_device_client(worker, uid, lang, change_to=None):
    import importlib.util
    spec = importlib.util.spec_from_file_location("mgt", os.path.join(GOLDEN, "make_golden_translate.py"))
    mgt = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mgt)

    class Client(T.DeviceTranslationClient):
        def __init__(self, *a, **kw):
            super().__init__(*a, worker=worker, **kw)
    return mgt.run_client(Client, uid, lang, change_to=change_to)


def test_device_client_sends_what_the_reference_client_sends():
    ref = _reference()
    rows = ref["translate"]["beam1"]["rows"]   # the reference client's model ran with its snapshot's settings (greedy)
    table = {(r["text"], r["lang"]): r["translation"] for r in rows}
    w = T.TranslationWorker(lambda: RecordedEngine(table))
    assert _run_device_client(w, "uid-1", "fr", change_to="de") == ref["client"]["fr_then_de"]
    assert _run_device_client(w, "uid-2", "fr", change_to="xx") == ref["client"]["fr_then_unknown"]
    assert _run_device_client(w, "uid-3", "xx") == ref["client"]["unknown"]


def test_one_bad_request_fails_alone():
    """An unknown language or an over-long source fails its own request; the rest of the coalesced call is translated."""
    tok = T.Small100Tokenizer.from_dir(MICRO_DIR)

    class Tr(T.DeviceTranslator):
        def __init__(self):     # the host half of DeviceTranslator, without a device context
            self.cfg, self.tok, self.capacity, self.max_src_tokens = _micro_cfg(), tok, 2, 40
            self.calls = []

        def translate_ids(self, sources, gen=None):
            self.calls.append([len(s) for s in sources])
            return [[5, 6, 2] for _ in sources], [0.0] * len(sources)

        def close(self):
            pass
    tr = Tr()
    long = " ".join(["hello world"] * 40)
    out = tr.translate_batch(["hello world", "hello", long, "the live", "good morning", "   "], ["fr", "xx", "fr", "de", "fr", "fr"])
    assert isinstance(out[1], KeyError) and isinstance(out[2], ValueError) and out[5] == "   "
    assert all(isinstance(out[i], str) for i in (0, 3, 4))
    assert all(len(c) <= 2 and sum(c) <= 40 for c in tr.calls) and sum(len(c) for c in tr.calls) == 3


def test_max_length_must_fit_the_position_table():
    with pytest.raises(ValueError, match="position table"):
        T.generation_settings({"max_length": 40}, max_positions=32)
    assert T.generation_settings({"max_length": 33}, max_positions=32).max_length == 33


def test_pad_ids_take_hugging_face_positions():
    """A pad id inside a source: positions count the non-pad tokens only (create_position_ids_from_input_ids)."""
    m = _hf_model(T.random_checkpoint(MICRO, 4), MICRO)
    orc = O.OracleM2M100(T.random_checkpoint(MICRO, 4), MICRO)
    src = [905, 1, 17, 1, 230, 2]
    with torch.no_grad():
        ref = m.model.encoder(input_ids=torch.tensor([src])).last_hidden_state[0].double().numpy()
    assert np.abs(orc.encode(src) - ref).max() < 1e-4


def test_registry_counts_the_translator_until_it_is_loaded(monkeypatch):
    from tests.test_model_registry import Factory, Memory, _registry
    monkeypatch.setenv("WLB200_TRANSLATE", "device")
    monkeypatch.setenv("WLB200_DEVICES", "0")
    assert T.pending_translator_bytes(0, footprint=lambda: 50) == 50
    assert T.pending_translator_bytes(1, footprint=lambda: 50) == 0
    f = Factory(footprint={"a": 40})
    reg = _registry(f, footprint=lambda n: 40, mem_probe=Memory(f, 100),
                    translator_pending=lambda d: T.pending_translator_bytes(d, footprint=lambda: 70))
    try:
        with pytest.raises(MemoryError):
            reg.acquire("a")                      # 100 free - 70 spoken for by the translator < 40
    finally:
        reg.shutdown()
    monkeypatch.setenv("WLB200_TRANSLATE", "cpu")
    reg = _registry(f, footprint=lambda n: 40, mem_probe=Memory(f, 100),
                    translator_pending=lambda d: T.pending_translator_bytes(d, footprint=lambda: 70))
    try:
        reg.acquire("a")
    finally:
        reg.shutdown()
    monkeypatch.setenv("WLB200_TRANSLATE", "device")

    class Loaded:
        loaded = True
    monkeypatch.setattr(T.TranslationWorker, "_shared", Loaded())
    assert T.pending_translator_bytes(0, footprint=lambda: 50) == 0   # allocated: free memory already shows it
