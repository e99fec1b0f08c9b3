"""``BatchedInferencePipeline(model, scheduler=...)``: a file's speech chunks decoded as streams of the scheduler's
running decode loop, on the CPU oracle engine whose decode session takes per-stream rules (tests/rules_oracle.py).

* every scenario of tests/golden/batched_reference.json gives the golden segments through the scheduler, alone and with
  a live request of other options decoding in the same loop (the chunks then join with rules of their own);
* closing the generator mid-file cancels the chunks in flight, and the scheduler keeps serving;
* a file's chunks hold at most ``max_share`` of the indices, and none enters while a live stream waits;
* a chunk that finishes before an earlier one waits for it: segments and ids come out in chunk order."""
from __future__ import annotations

import copy
import json
import os
import re
import time

import numpy as np
import pytest
import torch

from oracle.mel import OracleFeatureExtractor
from tests import stub_vad
from tests.golden.make_golden_batched import GAPPED_75, SCENARIOS
from tests.golden.make_golden_transcribe import make_audio
from tests.rules_oracle import RulesOracleSession, RulesOracleWhisper
from tests.test_batched_pipeline import _check_segments, _segments_json
from whisperlive_b200.config import dims_for
from whisperlive_b200.scheduler import BatchRequest, RequestCancelled, RoundScheduler
from whisperlive_b200.tokenizer import build_synthetic_tokenizer
from whisperlive_b200.transcriber import B200WhisperModel, BatchedInferencePipeline, TranscribeSession
from whisperlive_b200.weights import random_init

GOLD = os.path.join(os.path.dirname(__file__), "golden", "batched_reference.json")


@pytest.fixture(autouse=True)
def _threads():
    torch.set_num_threads(8)


def _model(name, seed, engine_cls=RulesOracleWhisper):
    dims = dims_for(name)
    eng = engine_cls(random_init(dims, seed=seed), dims)
    return B200WhisperModel(name, engine=eng, hf_tokenizer=build_synthetic_tokenizer(dims.vocab),
                            feature_extractor=OracleFeatureExtractor(dims.n_mels), vad=stub_vad)


def _scheduler(model, capacity=8):
    s = RoundScheduler(model, max_batch_size=capacity, step_tokens=8)
    s.start()
    return s


def _live_request(seconds=6.0):
    audio = make_audio(("gapped", (seconds,), 5))
    return BatchRequest(audio=audio, language="en", use_vad=False, word_timestamps=False)


@pytest.mark.parametrize("with_live", [False, True])
@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_scheduled_pipeline_matches_reference(name, with_live):
    gold = json.load(open(GOLD))[name]
    sc = SCENARIOS[name]
    m = _model(sc["model"], sc["seed"])
    sched = _scheduler(m)
    try:
        live = None
        if with_live:
            live = _live_request()
            sched.submit(live)
        pipe = BatchedInferencePipeline(m, scheduler=sched)
        kw = copy.deepcopy(sc["kw"])
        audio = make_audio(sc["audio"])
        if "raises" in gold:
            with pytest.raises({"RuntimeError": RuntimeError, "ValueError": ValueError}[gold["raises"]],
                               match=re.escape(gold["message"])):
                segs, _info = pipe.transcribe(audio, **kw)
                list(segs)
        else:
            segs, _info = pipe.transcribe(audio, **kw)
            _check_segments(_segments_json(list(segs)), gold["segments"])
        if live is not None:
            assert live.future.wait(120) and live.error is None, live.error
            # a fresh model: the sampling rungs' noise advances from call to call on an engine
            alone = _model(sc["model"], sc["seed"]).transcribe_batch([live.audio], [live.kwargs()])[0][0]
            assert [(s.tokens, s.start, s.end) for s in live.result] == [(s.tokens, s.start, s.end) for s in alone]
    finally:
        sched.stop()


def test_chunks_join_a_live_session_with_their_own_rules():
    """A live request of other options opens the decode session; the file's chunks join it with rules of their own
    (the live stream's session uses max_initial_timestamp_index 50, suppress_tokens [-1] mapped, beam 5; the chunks a
    suppress list of their own and length_penalty 0.5) and the result is still the one-shot pipeline's."""
    m = _model("micro.en", 1)
    audio = make_audio(GAPPED_75)
    kw = dict(batch_size=4, max_new_tokens=12, length_penalty=0.5, suppress_tokens=[5, 6, 7], word_timestamps=True)
    want = _segments_json(list(BatchedInferencePipeline(_model("micro.en", 1)).transcribe(audio, **kw)[0]))
    sched = _scheduler(m)
    try:
        lives = [_live_request(20.0 + i) for i in range(2)]
        for r in lives:
            sched.submit(r)
        assert lives[0].admitted.wait(60)
        got = _segments_json(list(BatchedInferencePipeline(m, scheduler=sched).transcribe(audio, **kw)[0]))
        for r in lives:
            assert r.future.wait(120) and r.error is None
    finally:
        sched.stop()
    assert got == want
    assert sum(getattr(s, "rule_admissions", 0) for s in _SESSIONS) > 0


_SESSIONS = []


@pytest.fixture(autouse=True)
def _record_sessions(monkeypatch):
    _SESSIONS.clear()
    orig = RulesOracleSession.__init__

    def init(self, *a, **k):
        orig(self, *a, **k)
        _SESSIONS.append(self)
    monkeypatch.setattr(RulesOracleSession, "__init__", init)


def test_closing_the_generator_cancels_the_file():
    m = _model("micro.en", 0)
    sched = _scheduler(m)
    try:
        pipe = BatchedInferencePipeline(m, scheduler=sched, max_share=0.125)     # one chunk at a time
        gen, _info = pipe.transcribe(make_audio(GAPPED_75), batch_size=8, max_new_tokens=12)
        first = next(gen)
        assert first.id == 1
        gen.close()
        live = _live_request()
        sched.submit(live)
        assert live.future.wait(120) and live.error is None          # the scheduler keeps serving
        for _ in range(200):
            if sched.files_in_flight == 0:
                break
            time.sleep(0.05)
        assert sched.files_in_flight == 0
        assert pipe.last_request.cancelled and isinstance(pipe.last_request.error, RequestCancelled)
    finally:
        sched.stop()


def _file_run(m, **kw):
    """The ``_ChunkRun`` the pipeline builds for the file (its one-shot path is not started)."""
    pipe = BatchedInferencePipeline(m)
    pipe._segments = lambda run, batch_size: iter([run])
    gen, _info = pipe.transcribe(make_audio(GAPPED_75), **kw)
    return next(gen)


def test_max_share_bound_and_live_first():
    m = _model("micro.en", 0)
    run = _file_run(m, batch_size=8, max_new_tokens=12)
    n_chunks = len(run.features)
    assert n_chunks >= 3
    sess = TranscribeSession(m)
    h = sess.add_file(run, max_share=0.25)
    sess.live_waiting = True
    sess.step_round(8)
    assert sess.file_streams() == 0 and not sess.files[h].active     # a live request waits: no chunk enters
    sess.live_waiting = False
    sess._feed_files()
    assert sess.file_streams() == 2                                   # max_share 0.25 of 8 indices
    peak = 0
    guard = 0
    while not sess.file_done(h):
        guard += 1
        assert guard < 500
        sess.step_round(8)
        peak = max(peak, sess.file_streams())
        assert sess.file_streams() <= 2                                # max_share 0.25 of 8 indices
    assert peak <= 2
    assert sess.file_error(h) is None and [s.id for s in sess.file_segments(h, 0)] == list(
        range(1, len(sess.file_segments(h, 0)) + 1))
    # a live stream waiting in the session itself holds the chunks back too
    run2 = _file_run(m, batch_size=8, max_new_tokens=12)
    sess2 = TranscribeSession(m)
    sess2.add_streams([make_audio(("gapped", (6.0,), 5))], [dict(language="en", vad_filter=False)])
    h2 = sess2.add_file(run2, max_share=0.5)
    sess2._feed_files()
    assert sess2.file_streams() == 0
    sess2.close()
    sess.close()


def test_max_share_counts_against_the_smaller_capacity():
    """A scheduler of fewer streams than the engine's max_streams bounds the file by its own capacity."""
    m = _model("micro.en", 0)                       # max_streams 8
    run = _file_run(m, batch_size=8, max_new_tokens=12)
    sess = TranscribeSession(m)
    h = sess.add_file(run, max_share=0.5, capacity=2)
    sess._feed_files()
    assert sess.file_streams() == 1 and len(sess.files[h].active) == 1
    sess.drop_file(h)
    sess.close()


def test_a_decoded_chunk_holding_its_slot_still_counts():
    """Word timestamps on an engine whose outputs cannot be joined: a decoded chunk keeps its encoder slot until it is
    finalised, so it still counts against the file's share and the scheduler's capacity."""
    from whisperlive_b200.transcriber import _FileRun
    m = _model("micro.en", 0)
    run = _file_run(m, batch_size=8, max_new_tokens=12)
    f = _FileRun(run, 0, 2)

    class E:
        def __init__(self, parent):
            self.parent = parent
    f.active = [E(object())]
    f.decoded = {1: E(object()), 2: E(None)}         # 1 keeps its slot, 2 gave it back
    assert f.held() == 2


class _SlowFirstSession(RulesOracleSession):
    """The first stream admitted runs 40 token steps longer: it finishes after the chunks admitted behind it."""

    order = []

    def admit(self, features, prompts, max_lengths, indices=None, rules=None):
        first = not hasattr(self, "_seen")
        self._seen = True
        idx = super().admit(features, prompts, max_lengths, indices, rules)
        if first:
            self._left[idx[0]] += 40
        return idx

    def collect(self, index):
        _SlowFirstSession.order.append(index)
        return super().collect(index)


class _SlowFirstWhisper(RulesOracleWhisper):
    def open_decode_session(self, capacity=None, **kw):
        return _SlowFirstSession(self, capacity or self.max_streams, **kw)


@pytest.mark.parametrize("words", [False, True])
def test_segment_order_when_a_late_chunk_finishes_first(words):
    kw = dict(batch_size=8, max_new_tokens=12, word_timestamps=words)
    audio = make_audio(GAPPED_75)
    one_shot = BatchedInferencePipeline(_model("micro.en", 1))
    want = _segments_json(list(one_shot.transcribe(audio, **kw)[0]))
    m = _model("micro.en", 1, engine_cls=_SlowFirstWhisper)
    sched = _scheduler(m)
    _SlowFirstSession.order = []
    try:
        pipe = BatchedInferencePipeline(m, scheduler=sched)
        got = _segments_json(list(pipe.transcribe(audio, **kw)[0]))
    finally:
        sched.stop()
    assert _SlowFirstSession.order[0] != 0            # chunk 0 (index 0) was not the first to finish
    assert got == want
    assert pipe.group_steps[0] == [n for g in one_shot.group_steps for n in g]    # every chunk, in chunk order
