"""Differential check of the host-side helpers against the reference's own Python, on seeded randomised inputs.

`python tests/golden/diff_reference_host.py --record REFERENCE_TREE` imports
whisper_live/transcriber/transcriber_faster_whisper.py from the reference tree with the same sys.modules stubs as
make_golden_transcribe.py, calls it on every case and stores what it returned in host_reference.json (48 bits of the
SHA-256 of each exact result; the detect_language probabilities and compression ratios themselves, compared with a tolerance).  Without arguments the same cases are run
through whisperlive_b200.transcriber and compared with that record.  The functions:
    _split_segments_by_timestamps (:970-1047)   get_prompt (:1480-1513)
    get_suppressed_tokens (:1831-1853)          merge_punctuations (:1856-1887)      get_compression_ratio (:1826-1828)
    detect_language (:1716-1789, multilingual model: first-segment threshold and majority vote)
Prints one JSON object {"cases": n, "mismatches": [...]}; tests/test_transcriber_host.py asserts the list is empty.
Executed in its own process because the stubs (fake ctranslate2 / faster_whisper modules) must not leak into pytest.
"""
import copy
import hashlib
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)

from tests.golden import make_golden_transcribe as G  # noqa: E402
from oracle.engine import OracleWhisper  # noqa: E402
from whisperlive_b200 import tokenizer as wtok  # noqa: E402
from whisperlive_b200 import transcriber as ours  # noqa: E402
from whisperlive_b200.config import dims_for  # noqa: E402
from oracle.mel import OracleFeatureExtractor  # noqa: E402
from whisperlive_b200.weights import random_init  # noqa: E402

RECORD = os.path.join(HERE, "host_reference.json")


def digest(x) -> str:
    """48 bits of the SHA-256 of a result's canonical JSON form (tuples as lists, numpy scalars as Python numbers)."""
    def conv(o):
        if hasattr(o, "item"):
            return o.item()
        if hasattr(o, "__dict__"):
            return vars(o)
        return str(o)
    return hashlib.sha256(json.dumps(x, default=conv, sort_keys=True).encode()).hexdigest()[:12]


class Side:
    """One side of the comparison: the reference's functions (recording) or ours against the stored record."""

    def __init__(self, ref_tree):
        self.recording = ref_tree is not None
        self.record = {"digests": [], "values": []} if self.recording else json.load(open(RECORD))
        self.i = self.j = 0

    def result(self, value):
        """value: the canonical result of the next case.  Returns the reference's digest when comparing."""
        d = digest(value)
        if self.recording:
            self.record["digests"].append(d)
            return d
        self.i += 1
        return self.record["digests"][self.i - 1]

    def value(self, value):
        """A result compared with a tolerance: stored as it is."""
        if self.recording:
            self.record["values"].append(value)
            return value
        self.j += 1
        return self.record["values"][self.j - 1]


def main():
    G.install_stubs()
    ref_tree = sys.argv[2] if len(sys.argv) > 2 and sys.argv[1] == "--record" else None
    side = Side(ref_tree)
    if ref_tree:
        sys.path.insert(0, ref_tree)
        from whisper_live.transcriber import transcriber_faster_whisper as ref
    else:
        ref = None

    rnd = random.Random(20260922)
    bad, n = [], 0
    for model_name in ("micro.en", "micro"):
        dims = dims_for(model_name)
        engine = OracleWhisper(random_init(dims, seed=0), dims)
        om = ours.B200WhisperModel(model_name, engine=engine, hf_tokenizer=wtok.build_synthetic_tokenizer(dims.vocab),
                                   feature_extractor=OracleFeatureExtractor(dims.n_mels))
        # the side under test: the reference's model while recording, ours otherwise
        rm = G.reference_model(ref, engine, dims) if ref else om
        mod = ref if ref else ours
        tok = wtok.Tokenizer(om.hf_tokenizer, dims.multilingual, task="transcribe" if dims.multilingual else None,
                             language="en" if dims.multilingual else None)
        tb = tok.timestamp_begin
        # ---- _split_segments_by_timestamps: random mixes of text and timestamp tokens, all edge shapes
        for _ in range(400):
            L = rnd.choice([0, 1, 2, 3, 5, 9, 17, 40])
            toks, ts = [], tb + rnd.randrange(0, 50)
            for _i in range(L):
                r = rnd.random()
                if r < 0.35:
                    ts += rnd.randrange(0, 40)
                    toks.append(min(ts, tb + 1500))
                else:
                    toks.append(rnd.randrange(0, min(tb, 50000)))
            if L and rnd.random() < 0.3:
                toks.append(toks[-1] if toks[-1] >= tb else tb + rnd.randrange(0, 1500))
            args = (tok, toks, rnd.choice([0.0, 30.0, 12.34]), rnd.choice([3000, 1234, 17]), rnd.choice([30.0, 12.34, 0.17]),
                    rnd.choice([0, 3000, 777]))
            if not toks:
                continue
            b = rm._split_segments_by_timestamps(tok, list(toks), *args[2:])
            b = (list(b[0]), b[1], bool(b[2]))
            n += 1
            if side.result(b) != digest(b):
                bad.append(("split", model_name, toks, args[2:], str(b)))
        # ---- get_prompt
        for _ in range(200):
            prev = [rnd.randrange(0, 50000) for _i in range(rnd.choice([0, 0, 3, 50, 223, 224, 300]))]
            kw = dict(without_timestamps=rnd.random() < 0.5, prefix=rnd.choice([None, None, "hello there", " world"]),
                      hotwords=rnd.choice([None, None, "foo bar", "x" * 400]))
            b = list(rm.get_prompt(tok, list(prev), **kw))
            n += 1
            if side.result(b) != digest(b):
                bad.append(("get_prompt", model_name, len(prev), kw, b[:8]))
        # ---- get_suppressed_tokens
        for sup in ([-1], [], [-1, 5, 7], [11, 12], [-1, tok.eot]):
            b = mod.get_suppressed_tokens(tok, sup)
            b = None if b is None else list(b)
            n += 1
            if side.result(b) != digest(b):
                bad.append(("get_suppressed_tokens", model_name, sup))
        # ---- detect_language wrapper (:1716-1789): threshold hit on the first segment, and the majority-vote path
        if dims.multilingual:
            from whisperlive_b200 import synth
            for sec, nseg, thr in ((7.0, 1, 0.5), (41.0, 2, 0.999), (65.0, 3, 0.0)):
                audio = synth.speech_like(sec, seed=int(sec))
                b = rm.detect_language(audio=audio, language_detection_segments=nseg, language_detection_threshold=thr)
                b = [b[0], float(b[1]), [[x[0], float(x[1])] for x in b[2]]]
                a = side.value(b)
                n += 1
                same = a[0] == b[0] and abs(a[1] - b[1]) < 1e-6 and [x[0] for x in a[2]] == [x[0] for x in b[2]] and \
                    all(abs(x[1] - y[1]) < 1e-6 for x, y in zip(a[2], b[2]))
                if not same:
                    bad.append(("detect_language", sec, nseg, thr, a[:2], b[:2]))
    # ---- merge_punctuations / get_compression_ratio (tokenizer independent)
    words = ["hello", " world", " \"", "quoted", ",", " and", " (", "paren", ")", ".", " ¿", "que", "?", " -", "dash", "!"]
    for _ in range(300):
        al = []
        for _i in range(rnd.randrange(0, 12)):
            w = rnd.choice(words)
            al.append(dict(word=w, tokens=[rnd.randrange(0, 1000) for _j in range(rnd.randrange(1, 3))],
                           start=rnd.random(), end=rnd.random(), probability=rnd.random()))
        b = copy.deepcopy(al)
        mod.merge_punctuations(b, "\"'“¿([{-", "\"'.。,，!！?？:：”)]}、")
        n += 1
        if side.result(b) != digest(b):
            bad.append(("merge_punctuations", al, b))
    for s in ("", "a", "aaaaaaaaaaaaaaaaaaaaaaaa", "the quick brown fox", "ab" * 200, "héllo wörld " * 7):
        if s:
            n += 1
            b = mod.get_compression_ratio(s)
            if abs(side.value(b) - b) > 1e-12:
                bad.append(("get_compression_ratio", s))
    if side.recording:
        json.dump(side.record, open(RECORD, "w"), separators=(",", ":"))
    print(json.dumps({"cases": n, "mismatches": [str(x)[:400] for x in bad[:10]], "n_mismatch": len(bad)}))


if __name__ == "__main__":
    main()
