"""Per-stream logits rules in a decode session (``DecodeSession.admit(..., rules=[...])``, ``wl_stream_rules``).

Kernel level: a session whose streams decode on the scripted logits of ``wl_test_search`` (``wl_test_session_script``)
mixes streams with different rules in one launch -- initial-timestamp cap 0 / 50 / none, different suppress lists,
``suppress_blank`` on and off, ``length_penalty`` 0 / 1 / 0.6, patience 1 / 2.  Each stream must give what
``oracle.search`` gives under the stream's own options (seeds chosen so that no decision margin falls in (0, 1e-5]),
exactly what the one-shot ``wl_test_search`` gives it under those options, and the same result whichever streams share
its launch.  Session level (tiny): the same against one-shot ``generate`` on the decoder, peek agreeing with collect.
"""
from __future__ import annotations

import functools
from typing import Dict, List, Optional

import numpy as np
import pytest

from oracle.search import GenOptions, search_stream
from tests.search_script import Script, ScriptStep
from tests.test_search_kernels import MAX_BEAM, MAX_STREAMS, NOSPEECH_TOL, SCORE_TOL, V3, bench_suppress, near_ties, \
    prompt_kinds

SP = V3
TB = SP.timestamp_begin
SESSION = dict(suppress_tokens=bench_suppress(SP), suppress_blank=True, max_initial_timestamp_index=50, length_penalty=1.0,
               patience=1.0)
NONE_CAP = 1500            # past the last timestamp: no initial-timestamp cap
RULES: List[Optional[dict]] = [
    None,
    dict(max_initial_timestamp_index=0, suppress_tokens=[1, 2, 3, 50, TB + 1], suppress_blank=False, length_penalty=0.0,
         patience=1.0),
    dict(max_initial_timestamp_index=NONE_CAP, suppress_tokens=list(range(100, 400)), suppress_blank=True,
         length_penalty=0.6, patience=2.0),
    dict(max_initial_timestamp_index=50, suppress_tokens=[], suppress_blank=False, length_penalty=1.0, patience=2.0),
    None,
    dict(max_initial_timestamp_index=0, suppress_tokens=bench_suppress(SP), suppress_blank=True, length_penalty=0.6,
         patience=1.0),
    dict(max_initial_timestamp_index=NONE_CAP, suppress_tokens=[SP.eot], suppress_blank=False, length_penalty=0.0,
         patience=2.0),
]
PROMPTS = [prompt_kinds(SP, i) for i in range(len(RULES))]
MAX_LEN = [36, 40, 30, 44, 32, 38, 34]
SCRIPT = {1: (501, -1), 4: (503, -1)}       # beam width -> script (seed, pattern)


def stream_kw(b: int) -> dict:
    return dict(SESSION, **(RULES[b] or {}))


def stream_opts(beam: int, b: int) -> GenOptions:
    kw = stream_kw(b)
    return GenOptions(beam_size=beam, patience=kw["patience"], num_hypotheses=1, length_penalty=kw["length_penalty"],
                      max_length=MAX_LEN[b], suppress_blank=kw["suppress_blank"], suppress_tokens=kw["suppress_tokens"],
                      max_initial_timestamp_index=kw["max_initial_timestamp_index"], trace=True)


@functools.lru_cache(maxsize=None)
def oracle_run(beam: int):
    out = []
    for b, prompt in enumerate(PROMPTS):
        o = stream_opts(beam, b)
        step = ScriptStep(Script(SP, prompt, o, *SCRIPT[beam]))
        out.append((search_stream(step, prompt, SP, o, stream_index=b), step.events))
    return out


# ---------------------------------------------------------------------------------------------------------- CPU part
@pytest.mark.parametrize("beam", [1, 4])
def test_rules_scenario_has_no_near_tie(beam):
    for b, (res, events) in enumerate(oracle_run(beam)):
        assert not near_ties(res, events, beam), (beam, b, near_ties(res, events, beam)[:5])
        assert res.sequences_ids, (beam, b)


def test_rules_change_the_oracle_result():
    """The per-stream options matter: under the session's options the streams with rules of their own decode
    differently (otherwise the device comparison below would not show that the rules reached the kernels)."""
    differ = 0
    for b in range(len(RULES)):
        if RULES[b] is None:
            continue
        o = stream_opts(4, b)
        s = GenOptions(**{**o.__dict__, **dict(SESSION, trace=True)})
        res = search_stream(ScriptStep(Script(SP, PROMPTS[b], s, *SCRIPT[4])), PROMPTS[b], SP, s, stream_index=b)
        differ += res.sequences_ids != oracle_run(4)[b][0].sequences_ids or res.scores != oracle_run(4)[b][0].scores
    assert differ >= 4, differ


# ---------------------------------------------------------------------------------------------------------- GPU part
def _engine():
    from tests.test_search_kernels import engine
    return engine()


def _session(eng, beam: int, capacity: int = 8):
    sess = eng.open_decode_session(capacity=capacity, beam_size=beam, num_hypotheses=1, **SESSION)
    sess.script(SCRIPT[beam])
    return sess


def _rule(b: int):
    r = RULES[b]
    return None if r is None else dict(r)


def _drain(sess, where: Dict[int, int], got: Dict[int, object], peeked: Dict[int, tuple]) -> None:
    guard = 0
    while sess.live:
        guard += 1
        assert guard < 500
        done = sess.run(max_steps=5)
        if done:
            for (toks, score, _ns, _step, final), ix in zip(sess.peek(done), done):
                assert final, ix
                peeked[where[ix]] = (toks, score)
        for ix in done:
            got[where.pop(ix)] = sess.collect(ix)


def _run_session(eng, beam: int, order: List[int], first: int, capacity: int = 8):
    """Admit ``order[:first]``, run a few steps, then admit the rest as indices free up; results by stream."""
    sess = _session(eng, beam, capacity)
    where, got, peeked = {}, {}, {}
    queue = list(order)

    def admit(k):
        take = [queue.pop(0) for _ in range(min(k, len(queue), len(sess.free_indices())))]
        if take:
            idx = sess.admit([None] * len(take), [PROMPTS[b] for b in take], [MAX_LEN[b] for b in take],
                             rules=[_rule(b) for b in take])
            where.update(zip(idx, take))
    admit(first)
    sess.run(max_steps=3)
    while sess.live or queue:
        admit(len(queue))
        for ix in sess.run(max_steps=4):
            got[where.pop(ix)] = sess.collect(ix)
    _drain(sess, where, got, peeked)
    sess.close()
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("beam", [1, 4])
def test_mixed_rules_in_one_session_match_the_oracle(beam):
    eng = _engine()
    sess = _session(eng, beam)
    idx = sess.admit([None] * len(PROMPTS), PROMPTS, MAX_LEN, rules=[_rule(b) for b in range(len(RULES))])
    where = dict(zip(idx, range(len(PROMPTS))))
    got, peeked = {}, {}
    _drain(sess, where, got, peeked)
    sess.close()
    for b, (res, _ev) in enumerate(oracle_run(beam)):
        g, what = got[b], f"beam {beam} stream {b} rules {RULES[b]}"
        assert g.sequences_ids == res.sequences_ids[:1], what
        np.testing.assert_allclose(g.scores, res.scores[:1], rtol=0, atol=SCORE_TOL, err_msg=what)
        assert abs(g.no_speech_prob - res.no_speech_prob) <= NOSPEECH_TOL, what
        assert g.steps == res.steps + len(PROMPTS[b]) - 1, (what, g.steps, res.steps)
        # peek of the finished index reports what collect returns first
        assert peeked[b][0] == g.sequences_ids[0] and peeked[b][1] == g.scores[0], what


@pytest.mark.gpu
@pytest.mark.parametrize("beam", [1, 4])
def test_session_rules_equal_one_shot_and_do_not_depend_on_neighbours(beam):
    """Each stream bit for bit as the one-shot wl_test_search decodes it under its own options (a stream admitted
    without rules: the session's options, the path that existed before per-stream rules), and the same whether it
    shares the loop with all the others, joins late, or decodes in a smaller session."""
    eng = _engine()
    n = len(PROMPTS)
    runs = [_run_session(eng, beam, list(range(n)), n),
            _run_session(eng, beam, list(reversed(range(n))), 2),
            _run_session(eng, beam, [3, 0, 6, 1, 5, 2, 4], 1, capacity=3)]
    for b in range(n):
        kw = stream_kw(b)
        one, _nh, _ = eng.test_search([PROMPTS[b]], SCRIPT[beam], beam_size=beam, num_hypotheses=1, max_length=MAX_LEN[b],
                                      prefill=True, **kw)
        for k, run in enumerate(runs):
            g, what = run[b], f"beam {beam} stream {b} run {k}"
            assert g.sequences_ids == one[0].sequences_ids, what
            assert g.scores == one[0].scores, what
            assert g.steps == one[0].steps, what
            assert g.no_speech_prob == one[0].no_speech_prob, what


@pytest.mark.gpu
def test_bad_rules_fail_the_whole_admission():
    from whisperlive_b200._lib import WlError
    eng = _engine()
    sess = _session(eng, 4)
    good = dict(RULES[1])
    for bad, field in ((dict(good, beam_size=5), "beam_size"), (dict(good, patience=4.3), "patience"),
                       (dict(good, patience=0.0), "patience"), (dict(good, length_penalty=float("nan")), "length_penalty"),
                       (dict(good, max_initial_timestamp_index=-1), "max_initial_timestamp_index")):
        with pytest.raises(WlError, match=field):
            sess.admit([None, None], PROMPTS[:2], MAX_LEN[:2], rules=[good, bad])
        assert sess.live == 0 and len(sess.free_indices()) == 8
    with pytest.raises(ValueError, match="num_hypotheses"):
        sess.admit([None], PROMPTS[:1], MAX_LEN[:1], rules=[dict(good, num_hypotheses=2)])
    # the session is untouched: a good admission decodes as before
    idx = sess.admit([None], PROMPTS[1:2], MAX_LEN[1:2], rules=[good])
    got, peeked = {}, {}
    _drain(sess, {idx[0]: 1}, got, peeked)
    assert got[1].sequences_ids == oracle_run(4)[1][0].sequences_ids[:1]
    sess.close()


@pytest.mark.gpu
def test_rule_tables_are_counted_in_device_bytes():
    """The per-index rule tables (mask words + four ints per index) are allocated once, with the session state."""
    from whisperlive_b200.config import WhisperDims
    from whisperlive_b200.engine import B200Whisper
    from whisperlive_b200.weights import random_init
    dims = WhisperDims("micro-51866", 128, 2, 2, 2, 80, 51866)
    eng = B200Whisper(dims, random_init(dims, seed=0), max_streams=MAX_STREAMS, max_beam=MAX_BEAM)
    before = eng.device_bytes
    sess = eng.open_decode_session(beam_size=4)
    grown = eng.device_bytes - before
    words = (51866 + 31) // 32 + 1
    assert grown >= MAX_STREAMS * (words * 4 + 16), grown
    sess.close()
    assert eng.device_bytes == before + grown     # a closed session keeps its state for the next one
    eng.destroy()


# ---------------------------------------------------------------------------------------------------------- tiny
SCORE_TOL_TINY = 0.05      # a near-tie between two engine runs, in length-normalised score (tests/test_gpu_parity.py)


def _score_tol(n: int, length_penalty: float, per_token: float) -> float:
    """A tolerance on cum / n^length_penalty that is ``per_token`` on cum / n: a penalty below 1 leaves more of the
    summed per-token differences in the score."""
    return per_token * max(1, n) ** (1.0 - length_penalty)


@pytest.mark.gpu
@pytest.mark.parametrize("beam", [1, 5])
def test_mixed_rules_on_tiny_equal_one_shot_generate(beam):
    """On the decoder (tiny, random weights): streams with mixed rules in one session give the hypotheses one-shot
    ``generate`` gives each under its own options, and the oracle's up to explained near-ties; peek agrees with
    collect."""
    from tests.test_gpu_parity import MARGIN_TOL, _explain_beam_divergence, engine, feats_for
    eng, orc = engine("tiny", seed=0)
    dims, sp = eng.dims, orc.spec
    n = 4
    feats = np.stack([feats_for(dims, d, 90 + i) for i, d in enumerate([6.0, 9.0, 5.0, 12.0])])
    enc, oenc = eng.encode(feats), orc.encode(feats)
    base = [sp.sot, sp.sot + 1, sp.sot + 1 + dims.num_languages + 1]
    prompts = [base, base, [sp.timestamp_begin - 3, 400, 1234, 11] + base, base]
    session_kw = dict(beam_size=beam, suppress_tokens=[1, 2, 3], return_scores=True, return_no_speech_prob=True)
    rules = [None,
             dict(max_initial_timestamp_index=0, suppress_tokens=[1, 2, 3, 50, 220], suppress_blank=True,
                  length_penalty=0.6, patience=2.0),
             dict(max_initial_timestamp_index=50, suppress_tokens=[-1], suppress_blank=False, length_penalty=0.0,
                  patience=1.0),
             dict(max_initial_timestamp_index=NONE_CAP, suppress_tokens=list(range(300, 700)), suppress_blank=True,
                  length_penalty=1.0, patience=2.0)]
    own = [dict(session_kw, **(r or {})) for r in rules]
    sess = eng.open_decode_session(capacity=n, **session_kw)
    idx = sess.admit([enc.select([b]) for b in range(n)], prompts, [448] * n, rules=rules)
    where = dict(zip(idx, range(n)))
    got, peeked = {}, {}
    _drain(sess, where, got, peeked)
    sess.close()
    for b in range(n):
        what = f"tiny beam {beam} stream {b}"
        g = got[b]
        lp, toks = own[b].get("length_penalty", 1.0), g.sequences_ids[0]
        assert peeked[b][0] == toks and peeked[b][1] == g.scores[0], what
        # the engine alone: the prefill's splits differ with the rows sharing the pass, so the same tokens or a near-tie
        one = eng.generate(enc.select([b]), [prompts[b]], max_length=448, **own[b])[0]
        assert abs(g.no_speech_prob - one.no_speech_prob) < 2e-3, what
        tol = 2e-3 if one.sequences_ids[0] == toks else SCORE_TOL_TINY
        assert abs(g.scores[0] - one.scores[0]) <= _score_tol(len(toks), lp, tol), (what, g.scores, one.scores)
        # the oracle under the stream's own options: the same tokens, or an explained divergence
        ref = orc.generate(oenc.select([b]), [prompts[b]], max_length=448, **own[b])[0]
        if ref.sequences_ids[0] == toks:
            assert abs(g.scores[0] - ref.scores[0]) <= _score_tol(len(toks), lp, 0.02), (what, g.scores, ref.scores)
        elif beam > 1:
            _explain_beam_divergence(eng, enc.select([b]), orc, oenc.select([b]), 0, prompts[b], dict(own[b], max_length=448),
                                     g, ref, what)
        else:
            i = next((k for k, (x, y) in enumerate(zip(toks, ref.sequences_ids[0])) if x != y), len(toks))
            margins = ref.margins[max(0, i - 1): i + 2]
            assert margins and min(margins) < MARGIN_TOL, (what, i, margins)
    enc.release()
