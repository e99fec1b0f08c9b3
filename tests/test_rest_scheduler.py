"""The scheduler side of the REST route's file jobs, on fakes: settled segments are read past a per-request cursor
only (each once, nothing when no window settled), and speaker embeddings are answered in calls bounded by the
workspace the engine budgets for them."""

import numpy as np

from whisperlive_b200.scheduler import EMBED_CALL_SAMPLES, BatchRequest, RoundScheduler


class _Session:
    def __init__(self):
        self.segments = []
        self.asked = []

    def settled(self, cursors):
        self.asked.append(dict(cursors))
        return {h: self.segments[n:] for h, n in cursors.items() if len(self.segments) > n}


def test_settled_segments_are_read_past_the_cursor_once():
    sch = RoundScheduler(object(), max_batch_size=2)
    r = BatchRequest(audio=np.zeros(10, np.float32), want_segments=True)
    live = BatchRequest(audio=np.zeros(10, np.float32))
    sess = _Session()
    in_flight = {0: r, 1: live}
    sch._publish_settled(sess, in_flight)                  # nothing settled yet
    sess.segments = ["s1", "s2"]
    sch._publish_settled(sess, in_flight)
    sch._publish_settled(sess, in_flight)                  # no new window
    sess.segments = ["s1", "s2", "s3"]
    sch._publish_settled(sess, in_flight)
    assert r.settled.since(0) == ["s1", "s2", "s3"] and len(live.settled) == 0
    assert sess.asked == [{0: 0}, {0: 0}, {0: 2}, {0: 2}]


def test_settled_failure_leaves_the_owner_thread_alone():
    class Broken:
        def settled(self, cursors):
            raise RuntimeError("boom")
    sch = RoundScheduler(object(), max_batch_size=2)
    r = BatchRequest(audio=np.zeros(10, np.float32), want_segments=True)
    sch._publish_settled(Broken(), {0: r})
    assert len(r.settled) == 0


def test_embedding_calls_are_bounded_by_the_budgeted_workspace():
    calls = []

    class T:
        def speaker_embeddings(self, audios):
            calls.append([len(a) for a in audios])
            return np.stack([np.full(256, len(a), np.float32) for a in audios])
    sch = RoundScheduler(T(), max_batch_size=2)          # budget: 2 x 30 s per call
    seg = EMBED_CALL_SAMPLES // 2
    sizes = [seg] * 5 + [3 * EMBED_CALL_SAMPLES, seg]      # the long one goes alone
    reqs = sch.embed_many([np.zeros(n, np.float32) for n in sizes])
    sch._answer_embeddings()
    assert calls == [[seg] * 4, [seg], [3 * EMBED_CALL_SAMPLES], [seg]]
    assert all(r.future.is_set() and r.result[0] == n for r, n in zip(reqs, sizes))
    assert all(sum(c) <= 2 * EMBED_CALL_SAMPLES for c in calls if len(c) > 1)
