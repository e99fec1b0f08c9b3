"""A batched file decoded at another beam than the live streams joins their running decode loop
(``BatchedInferencePipeline(model, scheduler=...).transcribe(..., beam_size=1)`` beside live beam-5 requests).

CPU, on the oracle engine whose decode session takes a per-stream width (tests/beams_oracle.py): the chunks are
admitted with rules while the live streams are still decoding, in the one session the live requests opened, and give
the one-shot pipeline's beam-1 segments; the live results are unchanged.  Under the rule that only an equal width may
join, the same scenario has to reopen the session.  GPU (tiny): the file through ``RoundScheduler`` on the device."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle.mel import OracleFeatureExtractor
from tests import stub_vad
from tests.beams_oracle import BeamsOracleSession, BeamsOracleWhisper
from tests.golden.make_golden_batched import GAPPED_75
from tests.golden.make_golden_transcribe import make_audio
from tests.test_batched_pipeline import _segments_json
from whisperlive_b200 import transcriber
from whisperlive_b200.config import dims_for
from whisperlive_b200.scheduler import BatchRequest, RoundScheduler
from whisperlive_b200.tokenizer import build_synthetic_tokenizer
from whisperlive_b200.transcriber import B200WhisperModel, BatchedInferencePipeline
from whisperlive_b200.weights import random_init

FILE_KW = dict(batch_size=4, max_new_tokens=12, beam_size=1)


@pytest.fixture(autouse=True)
def _threads():
    torch.set_num_threads(8)


def _model(seed=1, engine_cls=BeamsOracleWhisper):
    dims = dims_for("micro.en")
    eng = engine_cls(random_init(dims, seed=seed), dims)
    return B200WhisperModel("micro.en", engine=eng, hf_tokenizer=build_synthetic_tokenizer(dims.vocab),
                            feature_extractor=OracleFeatureExtractor(dims.n_mels), vad=stub_vad)


def _live_requests():
    # beam 5 (the default), one rung: the live streams never sample
    return [BatchRequest(audio=make_audio(("gapped", (40.0 + 5 * i,), 5)), language="en", use_vad=False,
                         word_timestamps=False, temperature=0.0) for i in range(2)]


class _Recorder:
    """Counts decode-session opens, and for every stream admitted with a width of its own, how many streams of the
    session's own width were still decoding at that moment."""

    def __init__(self, monkeypatch):
        self.sessions, self.joined_beside = [], []
        rec = self
        orig_init, orig_admit = BeamsOracleSession.__init__, BeamsOracleSession.admit

        def init(self, *a, **k):
            orig_init(self, *a, **k)
            self._plain = set()
            rec.sessions.append(self)

        def admit(self, features, prompts, max_lengths, indices=None, rules=None, sampling=None):
            running = len([i for i in self._plain if self._left.get(i, 0) > 0])
            idx = orig_admit(self, features, prompts, max_lengths, indices, rules, sampling)
            for i, r in zip(idx, rules or [None] * len(idx)):
                if r is None:
                    self._plain.add(i)
                elif int(r.get("beam_size", 0)) not in (0, self.beam_size):
                    rec.joined_beside.append(running)
            return idx
        monkeypatch.setattr(BeamsOracleSession, "__init__", init)
        monkeypatch.setattr(BeamsOracleSession, "admit", admit)


def _scenario(m):
    sched = RoundScheduler(m, max_batch_size=8, step_tokens=8)
    sched.start()
    try:
        lives = _live_requests()
        for r in lives:
            sched.submit(r)
        assert lives[0].admitted.wait(60)
        got = _segments_json(list(BatchedInferencePipeline(m, scheduler=sched).transcribe(make_audio(GAPPED_75),
                                                                                          **FILE_KW)[0]))
        for r in lives:
            assert r.future.wait(300) and r.error is None, r.error
        return got, lives, sched.rule_admissions
    finally:
        sched.stop()


def _old_rules_fit(ds, skw):
    """The rule before per-stream widths: only the session's own beam width joins with rules."""
    if not getattr(ds, "supports_rules", False):
        return False
    return int(skw.get("beam_size", 5)) == int(ds.beam_size) and int(skw.get("num_hypotheses", 1)) == 1


def test_beam1_file_joins_a_live_beam5_session(monkeypatch):
    want = _segments_json(list(BatchedInferencePipeline(_model()).transcribe(make_audio(GAPPED_75), **FILE_KW)[0]))
    rec = _Recorder(monkeypatch)
    m = _model()
    got, lives, rule_admissions = _scenario(m)
    assert got == want
    assert len(rec.sessions) == 1, "the live requests' session was reopened"
    assert rec.sessions[0].beam_size == 5 and rec.sessions[0].rows_per_stream == 5
    assert rule_admissions > 0 and rec.joined_beside and all(n > 0 for n in rec.joined_beside), rec.joined_beside
    for r in lives:
        alone = _model().transcribe_batch([r.audio], [r.kwargs()])[0][0]
        assert [(s.tokens, s.start, s.end) for s in r.result] == [(s.tokens, s.start, s.end) for s in alone]

    # the same scenario under the equal-width rule: the chunks wait for the loop to drain, which reopens it
    monkeypatch.setattr(transcriber, "_rules_fit", _old_rules_fit)
    rec_old = _Recorder(monkeypatch)
    got_old, lives_old, _ = _scenario(_model())
    assert got_old == want
    assert len(rec_old.sessions) >= 2 and not rec_old.joined_beside
    assert [[s.tokens for s in r.result] for r in lives_old] == [[s.tokens for s in r.result] for r in lives]


def test_rules_fit_takes_widths_up_to_the_rows():
    class S:
        supports_rules, beam_size, rows_per_stream = True, 5, 5
    for k in range(1, 6):
        assert transcriber._rules_fit(S(), dict(beam_size=k, num_hypotheses=1))
    assert not transcriber._rules_fit(S(), dict(beam_size=6, num_hypotheses=1))
    assert not transcriber._rules_fit(S(), dict(beam_size=1, num_hypotheses=2))

    class Greedy:
        supports_rules, beam_size, rows_per_stream = True, 1, 1
    assert not transcriber._rules_fit(Greedy(), dict(beam_size=5))     # a beam-5 live stream waits for the drain

    class NoRows:                                                       # a session that reports no rows: its own width
        supports_rules, beam_size = True, 5
    assert transcriber._rules_fit(NoRows(), dict(beam_size=5))
    assert not transcriber._rules_fit(NoRows(), dict(beam_size=1))


# ---------------------------------------------------------------------------------------------------------- GPU (tiny)
SR = 16000
CLIPS = [{"start": 0, "end": 24 * SR}, {"start": 25 * SR, "end": 47 * SR}, {"start": 48 * SR, "end": 61 * SR},
         {"start": 62 * SR, "end": 70 * SR}]


def _explain(eng, enc, prompt, a, b, what) -> float:
    """Two greedy decodes of one chunk that differ: the decision at their first differing step, teacher-forced on the
    device over the common prefix, must be a near-tie -- the two tokens' logits (EOT where a decode ended) within
    MARGIN_TOL, or, when one is a timestamp and the other text, the timestamp mass against the best text logit (rule
    e) within it.  Returns the margin."""
    from tests.test_gpu_parity import MARGIN_TOL
    i = next((k for k, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))
    ta, tb = (a[i] if i < len(a) else eng.eot), (b[i] if i < len(b) else eng.eot)
    lg = eng.decode_logits(enc, [list(prompt) + list(a[:i])])[0][-1].astype(np.float64)
    margin = abs(lg[ta] - lg[tb])
    if (ta >= eng.timestamp_begin) != (tb >= eng.timestamp_begin):
        ts = lg[eng.timestamp_begin:]
        lse_ts = ts.max() + np.log(np.exp(ts - ts.max()).sum())
        margin = min(margin, abs(lse_ts - lg[:eng.eot].max()))
    assert margin < MARGIN_TOL, (what, i, ta, tb, margin)
    return float(margin)


@pytest.mark.gpu
def test_beam1_file_through_the_scheduler_on_tiny():
    """On the device: a beam-1 file through ``RoundScheduler`` beside live beam-5 requests joins the live requests'
    beam-5 session with its own width; every chunk gives the one-shot pipeline's beam-1 tokens and token steps, and the
    file its segments exactly, unless a chunk's decode differs -- which it may only at a near-tie (``_explain``); the
    live results equal those of a run without the file.  A near-tie can flip because the one-shot group's rows (one per chunk) run the
    small-batch decode GEMM (up to 16 rows) while the session's 8 x 5 rows run the split-K one (DESIGN.md section 8g)."""
    from whisperlive_b200 import synth
    m = B200WhisperModel("tiny", weights="random", hf_tokenizer="synthetic", max_streams=8)
    eng = m.model
    audio = synth.speech_like(70.0, seed=31)
    kw = dict(language="en", vad_filter=False, clip_timestamps=CLIPS, batch_size=4, beam_size=1)

    def live_requests():
        return [BatchRequest(audio=synth.speech_like(20.0 + 3 * i, seed=50 + i), language="en", use_vad=False,
                             temperature=[0.0]) for i in range(3)]

    # the file's chunks (the last two clips share one) with their features as the pipeline computes them on the host
    p = BatchedInferencePipeline(m)
    p.resident_features = False
    p._segments = lambda run, batch_size: iter([run])
    chunks = next(p.transcribe(audio, **kw)[0])
    n_chunks = len(chunks.features)
    chunk_start = [md["segments"][0]["start"] / SR for md in chunks.metadata]

    # the one-shot pipeline: each chunk's prompt and tokens, in chunk order
    one_calls = []
    generate = eng.generate

    def recording_generate(features, prompts, **k):
        out = generate(features, prompts, **k)
        one_calls.extend((list(p), list(r.sequences_ids[0])) for p, r in zip(prompts, out))
        return out
    eng.generate = recording_generate
    one_shot = BatchedInferencePipeline(m)
    want = list(one_shot.transcribe(audio, **kw)[0])
    eng.generate = generate
    assert len(one_calls) == n_chunks

    # the session: the file's chunks are the streams admitted with width 1, in chunk order
    opened, sess_tokens = [], []
    open_session = eng.open_decode_session

    def counted(*a, **k):
        opened.append(k.get("beam_size"))
        ds = open_session(*a, **k)
        admit, collect, chunk_of = ds.admit, ds.collect, {}

        def rec_admit(features, prompts, max_lengths, indices=None, sampling=None, rules=None):
            idx = admit(features, prompts, max_lengths, indices=indices, sampling=sampling, rules=rules)
            for ix, r in zip(idx, rules or [None] * len(idx)):
                if r is not None and r.get("beam_size") == 1:
                    chunk_of[ix] = len(sess_tokens)
                    sess_tokens.append(None)
            return idx

        def rec_collect(ix):
            res = collect(ix)
            if ix in chunk_of:
                sess_tokens[chunk_of.pop(ix)] = list(res.sequences_ids[0])
            return res
        ds.admit, ds.collect = rec_admit, rec_collect
        return ds
    eng.open_decode_session = counted

    def run(with_file):
        sched = RoundScheduler(m, max_batch_size=8, step_tokens=8)
        sched.start()
        try:
            reqs = live_requests()
            for r in reqs:
                sched.submit(r)
            got, pipe = None, None
            if with_file:
                assert reqs[0].admitted.wait(120)
                pipe = BatchedInferencePipeline(m, scheduler=sched)
                got = list(pipe.transcribe(audio, **kw)[0])
            for r in reqs:
                assert r.future.wait(300) and r.error is None, r.error
            return got, pipe, [[s.tokens for s in r.result] for r in reqs], sched.rule_admissions
        finally:
            sched.stop()

    _none, _p, live_alone, _ = run(False)
    opened.clear()
    got, pipe, live_with, rules = run(True)
    eng.open_decode_session = open_session
    # the chunks joined the live requests' beam-5 loop with width 1 instead of waiting for it to drain
    assert rules > 0 and opened[0] == 5, (rules, opened)
    assert len(sess_tokens) == n_chunks and None not in sess_tokens
    assert live_with == live_alone

    steps_got, steps_want = pipe.group_steps[0], [n for g in one_shot.group_steps for n in g]
    differ = [k for k in range(n_chunks) if sess_tokens[k] != one_calls[k][1]]
    if not differ:                                  # the one-shot pipeline's segments exactly, as at beam 5
        assert [(s.id, s.seek, s.tokens, s.start, s.end) for s in got] == \
            [(s.id, s.seek, s.tokens, s.start, s.end) for s in want]
    for k in range(n_chunks):
        if k not in differ:
            assert steps_got[k] == steps_want[k], k
            continue
        # segments follow a chunk's tokens (random weights put their timestamps anywhere, so they are not matched to
        # chunks by time): the chunk's differing decode is what must be explained
        enc = eng.encode(np.asarray(chunks.features[k], dtype=np.float32)[None])
        margin = _explain(eng, enc, one_calls[k][0], sess_tokens[k], one_calls[k][1], f"chunk {k}")
        print(f"chunk {k}: session and one-shot beam-1 tokens differ at a near-tie, margin {margin:.4f}")
        enc.release()
