"""``BatchedInferencePipeline(model, scheduler=...)`` on the device (tiny, random weights): a file's chunks decoded in
the scheduler's running decode loop beside live streams -- joining it with logits rules of their own -- give the
segments of the one-shot pipeline, with and without word timestamps, and the live streams' results do not change."""
from __future__ import annotations

import numpy as np
import pytest

from whisperlive_b200 import synth

pytestmark = pytest.mark.gpu

SR = 16000
CLIPS = [{"start": 0, "end": 24 * SR}, {"start": 25 * SR, "end": 47 * SR}, {"start": 48 * SR, "end": 61 * SR},
         {"start": 62 * SR, "end": 70 * SR}]


def _segs(segs):
    return [(s.id, s.seek, s.tokens, s.start, s.end,
             None if s.words is None else [(w.word, w.start, w.end) for w in s.words]) for s in segs]


@pytest.mark.parametrize("words", [False, True])
def test_scheduled_file_equals_one_shot_beside_live_streams(words):
    from whisperlive_b200.scheduler import BatchRequest, RoundScheduler
    from whisperlive_b200.transcriber import B200WhisperModel, BatchedInferencePipeline
    m = B200WhisperModel("tiny", weights="random", hf_tokenizer="synthetic", max_streams=8)
    audio = synth.speech_like(70.0, seed=31)
    kw = dict(language="en", vad_filter=False, clip_timestamps=CLIPS, batch_size=4, word_timestamps=words,
              length_penalty=0.6, suppress_tokens=[-1, 220])
    def live_requests():
        return [BatchRequest(audio=synth.speech_like(20.0 + 3 * i, seed=50 + i), language="en", use_vad=False,
                             temperature=[0.0]) for i in range(3)]
    one_shot = BatchedInferencePipeline(m)
    want = _segs(one_shot.transcribe(audio, **kw)[0])
    # the live streams through the scheduler without the file: what they must still give beside it
    sched = RoundScheduler(m, max_batch_size=8, step_tokens=8)
    sched.start()
    try:
        alone = live_requests()
        for r in alone:
            sched.submit(r)
        for r in alone:
            assert r.future.wait(300) and r.error is None, r.error
    finally:
        sched.stop()
    live_alone = [r.result for r in alone]
    reqs = live_requests()
    sched = RoundScheduler(m, max_batch_size=8, step_tokens=8)
    sched.start()
    try:
        for r in reqs:
            sched.submit(r)
        assert reqs[0].admitted.wait(120)
        pipe = BatchedInferencePipeline(m, scheduler=sched)
        got = _segs(pipe.transcribe(audio, **kw)[0])
        for r in reqs:
            assert r.future.wait(300) and r.error is None, r.error
    finally:
        sched.stop()
    assert got == want
    # the chunks' options differ from the live streams' (length_penalty, suppress list): they joined the live streams'
    # decode loop with rules of their own instead of waiting for it to drain
    assert sched.rule_admissions > 0, sched.rule_admissions
    assert pipe.group_steps[0] == [n for g in one_shot.group_steps for n in g]      # every chunk, the same steps
    for r, alone in zip(reqs, live_alone):
        assert [s.tokens for s in r.result] == [s.tokens for s in alone]
