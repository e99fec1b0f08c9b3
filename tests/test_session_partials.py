"""Interim transcripts from the running decode loop and cancelling streams in flight: ``DecodeSession.peek`` /
``cancel`` (``wl_session_peek`` / ``wl_session_cancel``), ``TranscribeSession.partials`` / ``cancel``, the scheduler's
``want_partials`` / ``BatchRequest.cancel`` and the backend plugin's interim messages.

The CPU tests drive the transcriber, the scheduler and the plugin over the oracle engine with a CPU model of a decode
session that can peek and cancel (below): a running stream's interim tokens are the first ``step`` tokens of the result
the oracle gives it.  The GPU tests check the device session against the oracle and against unpeeked runs."""
import json
import sys
import threading
import time

import numpy as np
import pytest
import torch

from tests.test_boundary_cpu import REF, _oracle_model
from tests.test_session_sampling import SamplingOracleSession
from whisperlive_b200 import synth

GREEDY = dict(temperature=[0.0], beam_size=1, log_prob_threshold=None, compression_ratio_threshold=None,
              no_speech_threshold=None, vad_filter=False, language="en", max_new_tokens=40)


class PeekOracleSession(SamplingOracleSession):
    """CPU model of a decode session with ``peek`` / ``cancel``: a running stream reports the first ``step`` tokens of
    its oracle result, where ``step`` counts the token steps it has been decoding.  ``run_delay`` (s) makes each run
    take wall time, so a client thread can see the rounds go by."""

    run_delay = 0.0

    def __init__(self, engine, capacity, **kw):
        super().__init__(engine, capacity, **kw)
        self._total = {}
        self.peeks = 0
        self.cancelled = []

    def admit(self, features, prompts, max_lengths, indices=None, sampling=None):
        idx = super().admit(features, prompts, max_lengths, indices, sampling)
        for i in idx:
            self._total[i] = self._left[i]
        return idx

    def run(self, max_steps=16, break_on_finish=True):
        if self.run_delay:
            time.sleep(self.run_delay)
        return super().run(max_steps, break_on_finish)

    def peek(self, indices):
        if any(i not in self._res for i in indices):
            raise RuntimeError(f"peek: idle index in {list(indices)}")
        self.peeks += 1
        out = []
        for i in indices:
            r, step = self._res[i], self._total[i] - self._left[i]
            final = self._left[i] == 0
            out.append((list(r.sequences_ids[0] if final else r.sequences_ids[0][:step]), float(r.scores[0]),
                        float(r.no_speech_prob), step, final))
        return out

    def cancel(self, indices):
        if any(i not in self._res for i in indices) or len(set(indices)) != len(indices):
            raise RuntimeError(f"cancel: idle or repeated index in {list(indices)}")
        for i in indices:
            del self._res[i], self._left[i], self._total[i]
            self.cancelled.append(i)


def _peek_model():
    """The oracle transcriber with peek/cancel-capable decode sessions; every encoder output it hands out counts its
    release."""
    model = _oracle_model()
    orc = model.model
    sessions, enc = [], {"made": 0, "released": 0}

    def open_decode_session(capacity=None, **kw):
        sessions.append(PeekOracleSession(orc, capacity or 8, **kw))
        return sessions[-1]
    orc.open_decode_session = open_decode_session
    encode = model.encode

    def counted(features):
        out = encode(features)
        enc["made"] += 1
        out.release = lambda: enc.__setitem__("released", enc["released"] + 1)
        return out
    model.encode = counted
    return model, sessions, enc


def _segs(segs):
    return [(s.tokens, s.start, s.end) for s in segs or []]


# --------------------------------------------------------------------------------------------------------- CPU
def test_step_round_partials_are_prefixes_of_the_final_result():
    """After every step round, each stream's interim segments are its settled segments plus pieces whose tokens begin
    the corresponding final segment's; the final segments are those of a run that never asked for partials."""
    torch.set_num_threads(4)
    waves = [synth.speech_like(d, seed=200 + i) for i, d in enumerate((4.0, 36.0, 6.0))]

    def drive(with_partials):
        model, sessions, _ = _peek_model()
        sess = model.open_session()
        handles = sess.add_streams(waves, [GREEDY] * len(waves))
        seen = {h: [] for h in handles}
        results = {}
        while sess.pending():
            sess.step_round(4)
            for e in sess.pop_finished():
                results[e.handle] = sess.result_of(e)[0]
            if with_partials:
                for h, segs in sess.partials([h for h in handles if h not in results]).items():
                    seen[h].append(segs)
        sess.close()
        return results, seen, sessions

    final, seen, sessions = drive(True)
    plain, _, plain_sessions = drive(False)
    assert {h: _segs(s) for h, s in final.items()} == {h: _segs(s) for h, s in plain.items()}
    assert sum(s.peeks for s in sessions) > 0 and sum(s.peeks for s in plain_sessions) == 0
    interim = 0
    for h, history in seen.items():
        toks = [s.tokens for s in final[h]]
        for segs in history:
            for s in segs:
                assert s.words is None
                assert any(t[:len(s.tokens)] == s.tokens for t in toks), (h, s.tokens)
            interim += bool(segs)
    assert interim > 0
    assert any(len(a) < len(b) for hist in seen.values() for a, b in zip(hist, hist[1:]))   # the 36 s stream settles a window


def test_partials_leave_vad_mapped_words_of_settled_windows_alone():
    """A VAD-clipped stream with word timestamps and two windows: interim segments of the settled first window come with
    the VAD mapping of the final result, and asking for them every round changes nothing in the final segments or words
    (the mapping is applied to copies, never to the stream's own words)."""
    from tests import stub_vad
    torch.set_num_threads(4)
    wave = np.concatenate([synth.speech_like(17.0, seed=700), synth.silence(3.0), synth.speech_like(19.0, seed=701),
                           synth.silence(3.0), synth.speech_like(5.0, seed=702)]).astype(np.float32)
    kw = dict(GREEDY, vad_filter=True, word_timestamps=True, max_new_tokens=30)

    def drive(with_partials):
        model, _, _ = _peek_model()
        model._vad = stub_vad
        sess = model.open_session()
        h = sess.add_streams([wave], [kw])[0]
        seen = []
        result = None
        while sess.pending():
            sess.step_round(4)
            for e in sess.pop_finished():
                result = sess.result_of(e)[0]
            if with_partials and result is None:
                seen += [s for segs in sess.partials([h]).values() for s in segs if s.words]
        sess.close()
        return result, seen

    def full(segs):
        return [(s.tokens, s.start, s.end, [(w.word, w.start, w.end, w.probability) for w in s.words or []]) for s in segs]
    final, seen = drive(True)
    plain, _ = drive(False)
    assert any(s.words for s in final) and len(seen) >= 3     # settled words were mapped for interim text several times
    assert full(final) == full(plain)
    mapped = {(s.start, s.end) for s in final}
    assert all((s.start, s.end) in mapped for s in seen)      # interim copies of settled segments carry the final times


def _cancel_run(state):
    """Three streams; the middle one is cancelled in ``state`` (None: never added).  Returns the others' segments, the
    session and the encoder accounting."""
    model, sessions, enc = _peek_model()
    sess = model.open_session()
    forced = dict(GREEDY, temperature=[0.0, 0.5, 1.0], beam_size=2, best_of=2, log_prob_threshold=0.0, max_new_tokens=24)
    plain = dict(GREEDY, beam_size=2, max_new_tokens=24)
    waves = [synth.speech_like(d, seed=300 + i) for i, d in enumerate((5.0, 7.0, 6.0))]
    if state is None:
        handles = [sess.add_streams([waves[0]], [plain])[0], None, sess.add_streams([waves[2]], [plain])[0]]
    else:
        handles = sess.add_streams(waves, [plain, forced, plain])
    victim = handles[1]

    def entry():
        return next((e for e in sess.entries if e.handle == victim), None)
    done_state = {"window": lambda e: True, "running": lambda e: e.state == "running",
                  "between_rungs": lambda e: e.state == "decode" and e.job.temp_idx > 0,
                  "settled": lambda e: e.state == "done"}
    results, cancelled = {}, state is None
    rounds = 0
    while sess.pending() or not cancelled:
        if not cancelled and (e := entry()) is not None and done_state[state](e):
            parent = e.parent
            sess.cancel(victim)
            cancelled = True
            assert entry() is None
            assert parent is None or parent.left >= 0
            if sess._dsess is not None:
                assert all(x.handle != victim for x in sess._running.values())
        if not sess.pending():
            break
        sess.step_round(3)
        rounds += 1
        for e in sess.pop_finished() if state != "settled" or cancelled else []:
            results[e.handle] = sess.result_of(e)[0]
        assert rounds < 500
    for e in sess.pop_finished():
        results[e.handle] = sess.result_of(e)[0]
    live = [s.live for s in sessions]
    sess.close()
    return [_segs(results[handles[0]]), _segs(results[handles[2]])], live, sessions, enc, victim in results


@pytest.mark.parametrize("state", ["window", "running", "between_rungs", "settled"])
def test_cancel_in_any_state_frees_everything(state):
    """Cancelling a stream before its encode, while it decodes, between two rungs of its ladder, or after it settled
    but before it was popped leaves no decode index and no encoder slot behind, and the other streams' segments are
    those of a run without it."""
    torch.set_num_threads(4)
    segs, live, sessions, enc, victim_answered = _cancel_run(state)
    ref = _cancel_run(None)[0]
    assert segs == ref
    assert not victim_answered
    assert enc["made"] == enc["released"]                      # every encode group gave its slots back
    assert live == [0] * len(sessions)                         # no decode index still held when everything is done
    if state == "running":
        assert any(s.cancelled for s in sessions)


def _scheduler_run(waves, want, delay=0.0, cancel_at=None):
    from whisperlive_b200.scheduler import BatchRequest, RoundScheduler
    model, sessions, enc = _peek_model()
    PeekOracleSession.run_delay = delay

    class Req(BatchRequest):
        def kwargs(self_):
            return dict(GREEDY)
    published = []
    reqs = [Req(audio=w, want_partials=want) for w in waves]
    for r in reqs:
        pub = r.partial.publish

        def rec(segs, r=r, pub=pub):
            ok = pub(segs)
            published.append((id(r), sum(len(s.tokens) for s in segs), ok, r.future.is_set()))
            return ok
        r.partial.publish = rec
    sch = RoundScheduler(model, max_batch_size=2, step_tokens=4)
    try:
        for r in reqs:                      # all in the inbox before the owner starts: admission order is fixed
            sch.submit(r)
        sch.start()
        if cancel_at is not None:
            i, cond = cancel_at
            t0 = time.monotonic()
            while not cond(sessions) and time.monotonic() - t0 < 60:
                time.sleep(0.005)
            reqs[i].cancel()
        for r in reqs:
            assert r.future.wait(120)
    finally:
        sch.stop()
        PeekOracleSession.run_delay = 0.0
    return reqs, published, sessions, enc


def test_scheduler_publishes_partials_only_when_they_change():
    """With ``want_partials`` the owner thread publishes interim segments between rounds, a new version only when the
    token count changed, all before the final result; final segments equal a run without partials, which never peeks."""
    torch.set_num_threads(4)
    waves = [synth.speech_like(d, seed=400 + i) for i, d in enumerate((5.0, 8.0, 4.0))]
    on, published, s_on, _ = _scheduler_run(waves, True)
    off, none, s_off, _ = _scheduler_run(waves, False)
    assert [_segs(r.result) for r in on] == [_segs(r.result) for r in off]
    assert not none and sum(s.peeks for s in s_off) == 0 and sum(s.peeks for s in s_on) > 0
    assert any(r.partial.version > 0 for r in on)
    for r in on:
        mine = [p for p in published if p[0] == id(r)]
        last = 0
        for _rid, ntok, ok, after_final in mine:
            assert not after_final
            assert ok == (ntok != last)
            last = ntok if ok else last
        assert r.partial.version == sum(ok for *_x, ok, _f in mine)
        finals = [s.tokens for s in r.result]
        for s in r.partial.segments:
            assert any(t[:len(s.tokens)] == s.tokens for t in finals)


def test_scheduler_cancel_answers_with_cancellation_and_frees_the_index():
    """A request cancelled while it decodes is answered with ``RequestCancelled``, its decode index is cancelled in the
    session, its encoder slots come back, and the other requests' segments are unchanged."""
    from whisperlive_b200.scheduler import RequestCancelled
    torch.set_num_threads(4)
    waves = [synth.speech_like(d, seed=500 + i) for i, d in enumerate((5.0, 9.0, 4.0))]
    ref, _, _, _ = _scheduler_run([waves[0], waves[2]], False)
    # two requests fit at once: the second one is cancelled as soon as both decode
    reqs, _, sessions, enc = _scheduler_run(waves, False, delay=0.05,
                                            cancel_at=(1, lambda sessions: any(len(s._res) == 2 for s in sessions)))
    assert isinstance(reqs[1].error, RequestCancelled) and reqs[1].result is None
    assert any(s.cancelled for s in sessions)
    assert [_segs(reqs[0].result), _segs(reqs[2].result)] == [_segs(r.result) for r in ref]
    assert enc["made"] == enc["released"]


def _client(ws, **kw):
    sys.path.insert(0, REF)
    try:
        from whisperlive_b200.backend import ServeClientB200
    finally:
        sys.path.remove(REF)
    return ServeClientB200(ws, client_uid="u1", model="micro.en", use_vad=False, no_speech_thresh=1.1, **kw)


class _WS:
    def __init__(self):
        self.sent, self.closed = [], False

    def send(self, msg):
        self.sent.append(json.loads(msg))

    def close(self):
        self.closed = True


def _backend(partials, delay, timeout=30, exit_after=None):
    """One 3 s chunk through the plugin (reference ServeClientBase); returns the messages, which of them were interim,
    the requests and the sessions.  The plugin's scheduler runs rounds of 4 token steps: the oracle's random-weight
    decodes are short, and a chunk must span several rounds to have interim text."""
    sys.path.insert(0, REF)
    try:
        from whisperlive_b200 import backend
        from whisperlive_b200.backend import ServeClientB200
    finally:
        sys.path.remove(REF)
    from whisperlive_b200.scheduler import BatchRequest, RoundScheduler
    scheduler = backend.StreamScheduler
    backend.StreamScheduler = lambda *a, **k: RoundScheduler(*a, step_tokens=4, **k)
    model, sessions, _ = _peek_model()
    orig_kwargs = BatchRequest.kwargs
    BatchRequest.kwargs = lambda self: dict(orig_kwargs(self), temperature=[0.0], beam_size=2, log_prob_threshold=None,
                                            max_new_tokens=24)
    ServeClientB200.MODEL_FACTORY = lambda name: model
    saved = (ServeClientB200.PARTIALS, ServeClientB200.REQUEST_TIMEOUT_S)
    ServeClientB200.PARTIALS, ServeClientB200.REQUEST_TIMEOUT_S = partials, timeout
    PeekOracleSession.run_delay = delay
    interim_idx, reqs, untouched = [], [], []
    send_interim = ServeClientB200.send_interim

    def rec_interim(self, segs, duration):
        before = (json.dumps(self.transcript), self.timestamp_offset, list(self.text))
        n = len(ws.sent)
        send_interim(self, segs, duration)
        interim_idx.extend(range(n, len(ws.sent)))
        untouched.append(before == (json.dumps(self.transcript), self.timestamp_offset, list(self.text)))
    ServeClientB200.send_interim = rec_interim
    ws = _WS()
    try:
        client = _client(ws)
        submit = ServeClientB200.BATCH_WORKER.submit

        def rec_submit(r):
            cancel = r.cancel

            def rec_cancel():      # was the stream decoding in the session when the client gave up on it?
                r.decoding_at_cancel = any(s._res for s in sessions)
                cancel()
            r.cancel = rec_cancel
            reqs.append(r)
            submit(r)
        ServeClientB200.BATCH_WORKER.submit = rec_submit
        client.add_frames(synth.speech_like(3.0, seed=1))
        deadline = time.time() + 60
        if exit_after is not None:
            while time.time() < deadline and not reqs:
                time.sleep(0.01)
            time.sleep(exit_after)
        elif timeout < 30:
            while time.time() < deadline and not (reqs and reqs[0].future.is_set()):
                time.sleep(0.01)
        else:
            while time.time() < deadline and not any("segments" in m for i, m in enumerate(ws.sent) if i not in interim_idx):
                time.sleep(0.05)
        client.exit = True
        client.trans_thread.join(timeout=30)
        for r in reqs:
            r.future.wait(30)
    finally:
        backend.StreamScheduler = scheduler
        ServeClientB200.send_interim = send_interim
        BatchRequest.kwargs = orig_kwargs
        ServeClientB200.PARTIALS, ServeClientB200.REQUEST_TIMEOUT_S = saved
        PeekOracleSession.run_delay = 0.0
        ServeClientB200.shutdown()
        ServeClientB200.MODEL_FACTORY = None
    return ws.sent, set(interim_idx), reqs, sessions, untouched


def test_backend_sends_interim_lines_and_the_same_final_messages():
    """``PARTIALS``: the plugin sends interim text while the chunk decodes, as the reference's incomplete line
    (``completed: False``), without touching the transcript or any other commit state; the first final message equals
    that of a run without partials."""
    torch.set_num_threads(4)
    sent, interim, reqs, _, untouched = _backend(True, delay=0.2)
    plain, none, _, _, _ = _backend(False, delay=0.2)
    assert interim and not none and all(untouched)
    assert reqs[0].want_partials
    for i in interim:
        segs = sent[i]["segments"]
        assert segs and segs[-1]["completed"] is False and sent[i]["uid"] == "u1"
    finals = [m for i, m in enumerate(sent) if "segments" in m and i not in interim]
    plain_finals = [m for m in plain if "segments" in m]
    assert finals and plain_finals and finals[0] == plain_finals[0]
    first_final = next(i for i, m in enumerate(sent) if "segments" in m and i not in interim)
    assert min(interim) < first_final


@pytest.mark.parametrize("how", ["timeout", "exit"])
def test_backend_timeout_and_exit_cancel_the_request(how):
    """A request the client thread stops waiting for -- it timed out, or the client went away -- is cancelled: the
    scheduler answers it with ``RequestCancelled`` and takes its stream out of the decode session."""
    from whisperlive_b200.scheduler import RequestCancelled
    torch.set_num_threads(4)
    # admission takes well under 0.6 s here, and the chunk's decode several rounds of 0.5 s: the client gives up on a
    # stream that is decoding
    kw = dict(timeout=0.6) if how == "timeout" else dict(exit_after=0.6)
    _sent, _interim, reqs, sessions, _ = _backend(False, delay=0.5, **kw)
    assert reqs and reqs[0].cancelled and reqs[0].future.is_set()
    assert reqs[0].decoding_at_cancel
    assert isinstance(reqs[0].error, RequestCancelled)
    assert any(s.cancelled for s in sessions)


# --------------------------------------------------------------------------------------------------------- GPU
def _oracle_prefix_cums(orc, oenc_b, prompt, tokens, kw):
    """[k]: the oracle's cumulative log-probability of the first k tokens of ``tokens`` after ``prompt``."""
    from tests.test_gpu_parity import _oracle_cums
    return [0.0] + _oracle_cums(orc, oenc_b, 0, list(prompt), list(tokens), kw)


def _peeking_run(eng, views, prompts, lengths, kw, plan, peek=True, specs=None, cycle=16):
    """Admit stream groups (``plan``) one stream per admission call, run ``max_steps`` = 1, 2, ..., ``cycle``, 1, ...
    and peek every live index after each run.  Returns collected results, the peeks per stream and the join steps."""
    sess = eng.open_decode_session(capacity=4, **kw)
    where, got, peeks, joined = {}, {}, {}, {}
    queue = [list(g) for g in plan]
    k = 0
    while sess.live or queue:
        if queue and len(queue[0]) <= len(sess.free_indices()):
            for i in queue.pop(0):
                ix = sess.admit([views[i]], [prompts[i]], [lengths[i]],
                                **({"sampling": [specs.get(i)]} if specs else {}))[0]
                where[ix] = i
                joined[i] = sess.steps
                peeks[i] = []
        fin = sess.run(max_steps=k % cycle + 1, break_on_finish=False)
        k += 1
        if peek and sess.live:
            live = sorted(where)
            for ix, p in zip(live, sess.peek(live)):
                peeks[where[ix]].append(p)
        for ix in fin:
            got[where.pop(ix)] = sess.collect(ix)
        assert k < 2000
    sess.close()
    return got, peeks, joined


def _greedy_setup(name):
    from tests.test_session_sampling import _session_setup
    return _session_setup(name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny", "small.en"])
def test_peek_greedy_session(name):
    """Greedy session, streams joining at different steps, a peek after every run of 1 .. 16 steps: each interim
    token list is the first ``len`` tokens of the collected hypothesis, ``step`` counts them, its score is the oracle's
    cumulative log-probability of that prefix over its length, and a finished stream reports its final hypothesis.
    Peeking changes nothing: the collected hypotheses are bit-identical to an unpeeked run and agree with one-shot
    ``generate``."""
    from tests.test_gpu_parity import SCORE_TOL, _same_hypotheses
    eng, orc, views, oenc, prompts, lengths, encs = _greedy_setup(name)
    kw = dict(beam_size=1, suppress_tokens=[1, 2, 3], return_scores=True, return_no_speech_prob=True)
    plan = [[0, 1], [2], [3, 4], [5]]
    got, peeks, joined = _peeking_run(eng, views, prompts, lengths, kw, plan)
    plain, none, joined2 = _peeking_run(eng, views, prompts, lengths, kw, plan, peek=False)
    assert joined == joined2 and joined[3] > 0
    n_peeks = 0
    for i in range(6):
        assert got[i].sequences_ids == plain[i].sequences_ids and got[i].scores == plain[i].scores, i
        assert got[i].no_speech_prob == plain[i].no_speech_prob, i
        ref = eng.generate(views[i], [prompts[i]], max_length=lengths[i], **kw)[0]
        _same_hypotheses(got[i], ref, f"{name} stream {i}")
        final = got[i].sequences_ids[0]
        cums = _oracle_prefix_cums(orc, oenc.select([i]), prompts[i], final, kw)
        for toks, score, nsp, step, fin in peeks[i]:
            n_peeks += 1
            if fin:
                assert toks == final and score == got[i].scores[0], i
                continue
            assert toks == final[:len(toks)] and step == len(toks), (i, step, len(toks))
            assert abs(score - cums[len(toks)] / max(len(toks), 1)) < SCORE_TOL, (i, len(toks), score, cums[len(toks)])
            assert 0.0 <= nsp <= 1.0
    assert n_peeks > 50
    for e in encs:
        e.release()


@pytest.mark.gpu
@pytest.mark.parametrize("beam", [4, 5])
def test_peek_beam_session_reports_the_leading_beam(beam):
    """Beam session: the interim hypothesis at ``step`` is the oracle trace's best live beam (``alive[0]``,
    ``alive_cum[0]``) after that many steps; where it is not, the two runs sit on a near-tie the oracle's own numbers
    show (the collected hypotheses then pass ``_explain_beam_divergence``)."""
    from oracle.search import GenOptions, search_stream
    from tests.test_gpu_parity import BEAM_TIE_TOL, _explain_beam_divergence
    eng, orc, views, oenc, prompts, lengths, encs = _greedy_setup("tiny")
    kw = dict(beam_size=beam, suppress_tokens=[1, 2, 3], return_scores=True, return_no_speech_prob=True)
    got, peeks, _ = _peeking_run(eng, views, prompts, lengths, kw, [[0, 1], [2], [3, 4], [5]])
    exact = total = 0
    for i in range(6):
        opts = GenOptions(beam_size=beam, suppress_tokens=[1, 2, 3], max_length=lengths[i], trace=True)
        on_oracle = search_stream(orc._stream_step_fn(oenc.select([i]), 0), list(prompts[i]), orc.spec, opts)
        tr, explained = on_oracle.trace, False
        for toks, score, _nsp, step, fin in peeks[i]:
            if fin or step >= len(tr):
                continue
            total += 1
            alive, cum = tr[step]["alive"], tr[step]["alive_cum"]
            if tuple(toks) == alive[0]:
                exact += 1
                assert abs(score * max(len(toks), 1) - cum[0]) < BEAM_TIE_TOL, (i, step, score, cum[0])
                continue
            near = [c for a, c in zip(alive, cum) if a == tuple(toks)]
            if near and cum[0] - near[0] < BEAM_TIE_TOL:
                continue                                   # the engine ranks a near-tied live beam first
            # the engine's beams left the oracle's: its collected hypothesis must differ too, by an explained near-tie
            assert got[i].sequences_ids[0] != on_oracle.sequences_ids[0], (i, step)
            if not explained:
                _explain_beam_divergence(eng, views[i], orc, oenc.select([i]), 0, prompts[i],
                                         dict(kw, max_length=lengths[i]), got[i], on_oracle, f"beam {beam} stream {i}")
                explained = True
    print(f"beam {beam}: {exact} of {total} interim hypotheses equal the oracle's best live beam")
    assert total > 20 and exact > 0
    for e in encs:
        e.release()


@pytest.mark.gpu
def test_peek_sampled_stream_reports_its_best_alive_row():
    """A sampled stream in a beam session reports an alive row: ``step`` tokens, a prefix of one of its collected
    hypotheses, and of those still alive the one with the highest cumulative log-probability (up to fp16 noise)."""
    eng, orc, views, oenc, prompts, lengths, encs = _greedy_setup("tiny")
    kw = dict(beam_size=4, suppress_tokens=[1, 2, 3], return_scores=True, return_no_speech_prob=True)
    specs = {1: (1.0, 4, 17, 0), 3: (0.8, 3, 18, 1)}
    got, peeks, _ = _peeking_run(eng, views, prompts, lengths, kw, [[0, 1], [2, 3]], specs=specs)
    checked = 0
    for i in specs:
        hyps = got[i].sequences_ids
        cums = {tuple(h): _oracle_prefix_cums(orc, oenc.select([i]), prompts[i], h, kw) for h in hyps}
        for toks, _score, _nsp, step, fin in peeks[i]:
            if fin or step == 0:
                continue
            alive = [h for h in hyps if len(h) >= step]
            if not alive:
                continue
            assert len(toks) == step and any(h[:step] == toks for h in alive), (i, step)
            mine = max(cums[tuple(h)][step] for h in alive if h[:step] == toks)
            best = max(cums[tuple(h)][step] for h in alive)
            assert mine >= best - 0.05, (i, step, mine, best)
            checked += 1
    assert checked > 10
    for e in encs:
        e.release()


@pytest.mark.gpu
def test_cancel_leaves_the_other_streams_bit_identical():
    """A neighbour cancelled mid-decode leaves the other streams bit-identical to a run where it was never admitted,
    and a stream admitted into the just-cancelled index gives its one-shot result."""
    from tests.test_gpu_parity import _same_hypotheses
    eng, orc, views, oenc, prompts, lengths, encs = _greedy_setup("tiny")
    kw = dict(beam_size=4, suppress_tokens=[1, 2, 3], return_scores=True, return_no_speech_prob=True)

    def run(with_victim):
        sess = eng.open_decode_session(capacity=4, **kw)
        sess.admit([views[0]], [prompts[0]], [lengths[0]], indices=[0])
        if with_victim:
            sess.admit([views[3]], [prompts[3]], [lengths[3]], indices=[1])
        sess.admit([views[2]], [prompts[2]], [lengths[2]], indices=[2])
        got, late = {}, None
        steps = 0
        while sess.live:
            fin = sess.run(max_steps=3, break_on_finish=False)
            steps += 3
            if with_victim and steps == 6:
                assert 1 in sess._held and 1 not in fin
                sess.cancel([1])
                assert 1 in sess.free_indices()
                late = sess.admit([views[5]], [prompts[5]], [lengths[5]], indices=[1])[0]
            for ix in fin:
                got[ix] = sess.collect(ix)
        sess.close()
        return got, late
    a, late = run(True)
    b, _ = run(False)
    for ix in (0, 2):
        assert a[ix].sequences_ids == b[ix].sequences_ids and a[ix].scores == b[ix].scores, ix
        assert a[ix].no_speech_prob == b[ix].no_speech_prob, ix
    ref = eng.generate(views[5], [prompts[5]], max_length=lengths[5], **kw)[0]
    _same_hypotheses(a[late], ref, "stream admitted into a cancelled index")
    for e in encs:
        e.release()


@pytest.mark.gpu
def test_peek_of_a_finished_stream_is_what_collect_returns_first():
    """A finished, uncollected index reports exactly the hypothesis ``collect`` then returns first -- tokens and score
    bit for bit -- under a length penalty whose ranking needs ``powf`` (0.6), with several hypotheses per stream."""
    eng, orc, views, oenc, prompts, lengths, encs = _greedy_setup("tiny")
    kw = dict(beam_size=5, num_hypotheses=3, length_penalty=0.6, patience=2, suppress_tokens=[1, 2, 3])
    sess = eng.open_decode_session(capacity=4, **kw)
    where = dict(zip(sess.admit(views[:4], prompts[:4], lengths[:4]), range(4)))
    checked = 0
    while sess.live:
        fin = sess.run(max_steps=16, break_on_finish=True)
        for ix, (toks, score, _nsp, _step, final) in zip(fin, sess.peek(fin) if fin else []):
            assert final
            got = sess.collect(ix)
            assert toks == got.sequences_ids[0] and score == got.scores[0], where[ix]
            checked += 1
    sess.close()
    assert checked == 4
    for e in encs:
        e.release()


@pytest.mark.gpu
def test_peek_and_cancel_errors_change_nothing():
    """Peek or cancel of an idle index, an index outside the session or a repeated cancel index fails before anything
    launches; the running stream is untouched and collects the result of an undisturbed run."""
    from whisperlive_b200._lib import WlError
    eng, orc, views, oenc, prompts, lengths, encs = _greedy_setup("tiny")
    kw = dict(beam_size=4, suppress_tokens=[1, 2, 3], return_scores=True, return_no_speech_prob=True)
    sess = eng.open_decode_session(capacity=3, **kw)
    sess.admit([views[0]], [prompts[0]], [lengths[0]], indices=[0])
    sess.run(max_steps=4, break_on_finish=False)
    launches = eng.lib.wl_kernel_launches(eng.ctx)
    for bad in ([1], [0, 2], [3], [-1]):
        with pytest.raises(WlError, match="idle|outside"):
            sess.peek(bad)
        with pytest.raises(WlError, match="idle|outside"):
            sess.cancel(bad)
    with pytest.raises(WlError, match="twice"):
        sess.cancel([0, 0])
    assert eng.lib.wl_kernel_launches(eng.ctx) == launches
    assert sess.live == 1 and sess.peek([0])[0][3] == 4
    while not sess.run(max_steps=16, break_on_finish=False):
        pass
    got = sess.collect(0)
    with pytest.raises(WlError, match="idle"):
        sess.peek([0])
    sess.close()
    ref = eng.open_decode_session(capacity=3, **kw)
    ref.admit([views[0]], [prompts[0]], [lengths[0]], indices=[0])
    while not ref.run(max_steps=4, break_on_finish=False):
        pass
    want = ref.collect(0)
    ref.close()
    assert got.sequences_ids == want.sequences_ids and got.scores == want.scores
    for e in encs:
        e.release()


@pytest.mark.gpu
def test_scheduler_partials_on_the_device():
    """The product scheduler on the device with partials on: final segments equal a partials-off run, and every chunk
    that decoded more than 16 tokens received interim text before its final result."""
    from tests.test_gpu_parity import engine
    from whisperlive_b200.feature_extractor import FeatureExtractor
    from whisperlive_b200.scheduler import BatchRequest, RoundScheduler
    from whisperlive_b200.tokenizer import build_synthetic_tokenizer
    from whisperlive_b200.transcriber import B200WhisperModel
    eng, _ = engine("tiny", seed=0)
    m = B200WhisperModel("tiny", engine=eng, hf_tokenizer=build_synthetic_tokenizer(eng.dims.vocab),
                         feature_extractor=FeatureExtractor(eng, eng.dims.n_mels))
    waves = [synth.speech_like(d, seed=600 + i) for i, d in enumerate((6.0, 9.0, 4.0, 12.0, 7.0, 5.0))]
    kwargs = dict(GREEDY, beam_size=4, language=None, suppress_blank=False, suppress_tokens=[-1, eng.eot],
                  max_new_tokens=60)

    n_new = [30 + 9 * i for i in range(len(waves))]

    class Req(BatchRequest):
        def kwargs(self_):
            # the decode emits min(max_length / 2, max_length - prompt) tokens (CT2), the prompt here is sot, language,
            # task; with the end-of-text token suppressed chunk i decodes exactly n_new[i] > 16 tokens
            return dict(kwargs, max_new_tokens=2 * self_.n_new - 3)

    def run(want):
        reqs = [Req(audio=w, want_partials=want) for w in waves]
        for r, n in zip(reqs, n_new):
            r.n_new = n
        sch = RoundScheduler(m, max_batch_size=4, step_tokens=16)
        for r in reqs:                  # everything queued before the owner starts: the later chunks join mid-flight
            sch.submit(r)
        sch.start()
        try:
            for r in reqs:
                assert r.future.wait(300)
                assert r.error is None, r.error
        finally:
            sch.stop()
        return reqs, sch
    on, s_on = run(True)
    off, s_off = run(False)
    assert s_on.admitted_mid_flight > 0
    assert [_segs(r.result) for r in on] == [_segs(r.result) for r in off]
    assert all(r.partial.version == 0 for r in off)
    assert all(r.partial.version >= 1 for r in on), [r.partial.version for r in on]
