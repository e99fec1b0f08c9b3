"""Pins of the translation path against the reference's own code (CPU; needs transformers, sentencepiece and the
reference tree).

    python tests/golden/make_golden_translate.py [--reference /path/to/WhisperLive]

Writes tests/golden/small100_micro/ (a sentencepiece BPE model trained on a seeded corpus with num_threads=1, its
vocab.json, and config.json of a micro M2M100: d 128, 2 heads, 2 encoder and 1 decoder layers; a rerun reuses the
committed tokenizer files), then, with the weights of whisperlive_b200.translation.random_checkpoint(seed=SEED):
  * translate_reference.json: the reference's SMALL100Tokenizer ids and decoded text for fixed texts and languages;
    its ServeClientTranslation.translate_text for those texts under several generation settings, with the source ids
    and Hugging Face's generated ids; the websocket messages of its queue loop;
  * mt_hf.npz: Hugging Face teacher-forced logits and generate sequences / scores at the micro shape.
The reference's tokenizer module needs one shim under transformers 5: ``transformers.tokenization_utils`` no longer
exports BatchEncoding / PreTrainedTokenizer.  A rerun reproduces both files byte for byte."""
from __future__ import annotations

import argparse
import json
import os
import queue
import shutil
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)

SEED = 3
MICRO_DIR = os.path.join(HERE, "small100_micro")
WORDS = ["hello", "world", "speech", "live", "whisper", "translate", "segment", "the", "a", "of", "good", "morning",
         "server", "client", "audio", "stream", "is", "and", "to", "we"]
TEXTS = ["", "   ", "hello world", "Hello, world! How are you?", "the live audio stream is good",
         "zzqx ünïcödé ☃", "whisper translate the segment and we stream to the client"]
LANGS = ["fr", "de", "ja"]
SETTINGS = {
    "beam1": dict(num_beams=1, max_length=16),
    "beam5": dict(num_beams=5, max_length=16),
    "beam5_early": dict(num_beams=5, max_length=16, early_stopping=True),
    "beam5_never_lp2": dict(num_beams=5, max_length=16, early_stopping="never", length_penalty=2.0),
    "beam5_lp0": dict(num_beams=5, max_length=16, length_penalty=0.0),
    "beam5_cut": dict(num_beams=5, max_length=5),
}


def train_tokenizer():
    import sentencepiece as spm
    os.makedirs(MICRO_DIR, exist_ok=True)
    model = os.path.join(MICRO_DIR, "sentencepiece.bpe.model")
    if not os.path.exists(model):
        rng = np.random.default_rng(SEED)
        with tempfile.TemporaryDirectory() as tmp:
            corpus = os.path.join(tmp, "corpus.txt")
            with open(corpus, "w") as f:
                for _ in range(2000):
                    f.write(" ".join(rng.choice(WORDS, int(rng.integers(3, 12)))) + "\n")
            spm.SentencePieceTrainer.train(input=corpus, model_prefix=os.path.join(tmp, "sp"), vocab_size=120, model_type="bpe",
                                           num_threads=1, character_coverage=1.0, seed_sentencepiece_size=100000)
            shutil.copy(os.path.join(tmp, "sp.model"), model)
    vocab_path = os.path.join(MICRO_DIR, "vocab.json")
    if not os.path.exists(vocab_path):
        sp = spm.SentencePieceProcessor()
        sp.Load(model)
        vocab = {"<s>": 0, "<pad>": 1, "</s>": 2, "<unk>": 3}
        for i in range(sp.get_piece_size()):
            p = sp.id_to_piece(i)
            if p not in vocab and p not in ("<unk>", "<s>", "</s>"):
                vocab[p] = len(vocab)
        del vocab[sp.id_to_piece(sp.get_piece_size() - 1)]   # one piece the vocabulary lacks: it maps to <unk>
        with open(vocab_path, "w") as f:
            json.dump(vocab, f, indent=0, sort_keys=True)
    with open(vocab_path) as f:
        return len(json.load(f))


def micro_config(n_vocab: int) -> dict:
    return dict(model_type="m2m_100", vocab_size=n_vocab + 100 + 8, d_model=128, encoder_layers=2, decoder_layers=1,
                encoder_attention_heads=2, decoder_attention_heads=2, encoder_ffn_dim=512, decoder_ffn_dim=512,
                max_position_embeddings=1024, scale_embedding=True, activation_function="relu", pad_token_id=1,
                bos_token_id=0, eos_token_id=2, decoder_start_token_id=2, dropout=0.0, attention_dropout=0.0,
                activation_dropout=0.0)


def shim():
    from transformers import M2M100ForConditionalGeneration  # noqa: F401  (resolve the lazy module first: it re-registers submodules)
    import transformers.tokenization_python as tp
    import transformers.tokenization_utils_base as tb
    m = types.ModuleType("transformers.tokenization_utils")
    m.BatchEncoding, m.PreTrainedTokenizer = tb.BatchEncoding, tp.PreTrainedTokenizer
    import transformers
    sys.modules["transformers.tokenization_utils"] = m
    transformers.tokenization_utils = m


def hf_model(cfg_json):
    import torch
    from transformers import M2M100Config, M2M100ForConditionalGeneration
    from whisperlive_b200 import translation as T
    cfg = T.config_from_json(cfg_json)
    m = M2M100ForConditionalGeneration(M2M100Config(**cfg_json)).eval()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in T.random_checkpoint(cfg, SEED).items()}, strict=False)
    m.tie_weights()
    return m


class Socket:
    def __init__(self):
        self.sent = []

    def send(self, msg):
        self.sent.append(json.loads(msg))


SEGMENTS = [dict(start="0.000", end="1.200", text="hello world", completed=True),
            dict(start="1.200", end="2.000", text="the live", completed=False),
            dict(start="1.200", end="3.100", text="   ", completed=True),
            dict(start="3.100", end="4.000", text="Hello, world! How are you?", completed=True)]
SEGMENTS_AFTER_CHANGE = [dict(start="4.000", end="5.500", text="the live audio stream is good", completed=True)]


def run_client(cls, uid, lang, change_to=None):
    ws, q = Socket(), queue.Queue()
    c = cls(uid, ws, q, target_language=lang, send_last_n_segments=2)
    for s in SEGMENTS:
        q.put(dict(s))
    q.put(None)
    c.speech_to_text()
    if change_to is not None:
        try:
            c.set_target_language(change_to)
        except Exception as e:   # the reference's tokenizer raises for an unknown language
            ws.sent.append({"set_target_language_raised": type(e).__name__})
        for s in SEGMENTS_AFTER_CHANGE:
            q.put(dict(s))
        q.put(None)
        c.speech_to_text()
    return ws.sent


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=os.environ.get("WHISPERLIVE_REFERENCE", "/root/reference"))
    a = ap.parse_args()
    import torch
    torch.manual_seed(0)
    torch.use_deterministic_algorithms(True)
    n_vocab = train_tokenizer()
    cfg_json = micro_config(n_vocab)
    with open(os.path.join(MICRO_DIR, "config.json"), "w") as f:
        json.dump(cfg_json, f, indent=1, sort_keys=True)
    shim()
    sys.path.insert(0, a.reference)
    from whisper_live.backend import translation_backend as RB
    from whisper_live.backend.tokenization_small100 import SMALL100Tokenizer

    model = hf_model(cfg_json)
    out = {"seed": SEED, "tokenizer": [], "translate": {}, "client": {}}
    with tempfile.TemporaryDirectory() as snap:
        model.save_pretrained(snap)
        for fn in ("vocab.json", "sentencepiece.bpe.model"):
            shutil.copy(os.path.join(MICRO_DIR, fn), snap)
        with open(os.path.join(snap, "tokenizer_config.json"), "w") as f:
            json.dump({"tokenizer_class": "SMALL100Tokenizer"}, f)
        tok = SMALL100Tokenizer(os.path.join(snap, "vocab.json"), os.path.join(snap, "sentencepiece.bpe.model"))
        n = len(tok.encoder)
        for lang in LANGS:
            tok.tgt_lang = lang
            for text in TEXTS:
                ids = tok(text)["input_ids"]
                extra = [0, 1, 3, n + 5, n + 100, n + 107]     # specials, a language token, made-up words
                out["tokenizer"].append(dict(text=text, lang=lang, ids=ids, decoded=tok.decode(ids, skip_special_tokens=True),
                                             decoded_extra=tok.decode(ids + extra, skip_special_tokens=True)))

        class Client(RB.ServeClientTranslation):
            def __init__(self, *args, **kw):
                kw["model_name"] = snap
                super().__init__(*args, **kw)

        for name, st in SETTINGS.items():
            c = Client("gen", Socket(), queue.Queue(), target_language="fr")
            assert c.model_loaded
            gc = c.translation_model.generation_config
            for k, v in {**dict(num_beams=1, max_length=20, early_stopping=False, length_penalty=1.0), **st}.items():
                setattr(gc, k, v)
            rows = []
            for lang in ("fr", "de"):
                c.set_target_language(lang)
                for text in TEXTS:
                    src = c.tokenizer(text)["input_ids"] if text.strip() else []
                    gen = []
                    if src:
                        with torch.no_grad():
                            r = c.translation_model.generate(input_ids=torch.tensor([src]))
                        gen = r[0].tolist()[1:]
                    rows.append(dict(text=text, lang=lang, src=src, generated=gen, translation=c.translate_text(text)))
            out["translate"][name] = dict(settings=st, rows=rows)
        out["client"]["fr_then_de"] = run_client(Client, "uid-1", "fr", change_to="de")
        out["client"]["fr_then_unknown"] = run_client(Client, "uid-2", "fr", change_to="xx")
        out["client"]["unknown"] = run_client(Client, "uid-3", "xx")

    with open(os.path.join(HERE, "translate_reference.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True, ensure_ascii=False)
        f.write("\n")

    # Hugging Face logits and generate at the micro shape
    rng = np.random.default_rng(SEED)
    V = cfg_json["vocab_size"]
    srcs = [[n_vocab + 24] + rng.integers(4, n_vocab, k).tolist() + [2] for k in (1, 6, 20)]
    prefix = [2] + rng.integers(4, V, 5).tolist()
    arrays = {}
    with torch.no_grad():
        for i, s in enumerate(srcs):
            arrays[f"src{i}"] = np.asarray(s, np.int64)
            arrays[f"logits{i}"] = model(input_ids=torch.tensor([s]), decoder_input_ids=torch.tensor([prefix])).logits[0].numpy()
            for name, st in SETTINGS.items():
                r = model.generate(input_ids=torch.tensor([s]), return_dict_in_generate=True, output_scores=True,
                                   do_sample=False, **{**dict(early_stopping=False, length_penalty=1.0), **st})
                arrays[f"seq{i}_{name}"] = r.sequences[0].numpy()
                if st["num_beams"] > 1:
                    arrays[f"score{i}_{name}"] = r.sequences_scores.numpy()
    arrays["prefix"] = np.asarray(prefix, np.int64)
    path = os.path.join(HERE, "mt_hf.npz")
    with open(path, "wb") as f:
        np.savez(f, **{k: arrays[k] for k in sorted(arrays)})
    print("wrote", os.path.join(HERE, "translate_reference.json"), path)


if __name__ == "__main__":
    main()
