"""Per-stream beam width in a decode session (``wl_stream_rules.beam_size``, ``DecodeSession.admit(rules=[{"beam_size":
k, ...}])``, k <= rows per stream).

Kernel level: sessions whose streams decode on the scripted logits of ``wl_test_search`` (``wl_test_session_script``).
A beam-5 session mixes streams of width 1 (CTranslate2's greedy search), 2, 3, 4 and 5, a sampled stream and some of
``test_session_rules.RULES``; a greedy session of ``num_hypotheses = 4`` takes widths up to 4.  Each stream must give
what ``oracle.search`` gives under its own ``GenOptions(beam_size=k, ...)`` (seeds chosen so that no decision margin
falls in (0, 1e-5]), bit for bit what the one-shot ``wl_test_search`` gives it at that width, and the same result in
three arrangements of neighbours and admission steps; peek agrees with collect.  A width above the rows, or
round(width x patience) above 16, fails the admission by name and leaves the streams in flight alone.
Session level (tiny): streams at beam 1, 2 and 5 in one beam-5 session against one-shot ``generate`` at those beams.
"""
from __future__ import annotations

import functools
from typing import Dict, List, Optional

import numpy as np
import pytest

from oracle.search import GenOptions, search_stream
from tests.search_script import Script, ScriptStep
from tests.test_search_kernels import NOSPEECH_TOL, SCORE_TOL, near_ties, prompt_kinds
from tests.test_session_rules import RULES, SESSION, SP, _drain

# (width, rules of test_session_rules.RULES or None) per stream; "sample" = a sampled stream.  Width 0 = no rules at
# all: the session's own search.
BEAM5 = [(1, None), (2, 1), (3, 2), (4, 3), (0, None), (1, 5), ("sample", None), (5, 6), (3, None), (2, 0)]
GREEDY4 = [(0, None), (2, 1), (3, 2), (4, 3), (1, 5), (4, None)]
SAMPLE = (0.7, 3, 1234, 0)        # temperature, num_hypotheses, seed, noise key
MAX_LEN = [36, 40, 30, 44, 32, 38, 34, 42, 33, 37]
SCRIPT = {5: (611, -1), 1: (617, -1)}        # session beam -> script (seed, pattern)


def _streams(session_beam: int):
    return BEAM5 if session_beam == 5 else GREEDY4


def prompts(session_beam: int) -> List[List[int]]:
    return [prompt_kinds(SP, i) for i in range(len(_streams(session_beam)))]


def stream_kw(session_beam: int, b: int) -> dict:
    """generate's options for stream b: the session's, updated by its rules; beam_size = its width."""
    width, rule = _streams(session_beam)[b]
    kw = dict(SESSION, **(RULES[rule] or {})) if rule is not None else dict(SESSION)
    kw["beam_size"] = width if width else session_beam
    return kw


def rules_for(session_beam: int, b: int) -> Optional[dict]:
    """What stream b is admitted with: None (the session's options), or every option spelled out -- a key a rules dict
    leaves out takes generate's default, not the session's."""
    width, rule = _streams(session_beam)[b]
    if width == "sample" or (width == 0 and rule is None):
        return None
    r = stream_kw(session_beam, b)
    if not width:
        del r["beam_size"]
    return r


def nh(session_beam: int) -> int:
    return 1 if session_beam > 1 else 4


def stream_opts(session_beam: int, b: int) -> GenOptions:
    kw = stream_kw(session_beam, b)
    return GenOptions(beam_size=kw["beam_size"], patience=kw["patience"], num_hypotheses=nh(session_beam),
                      length_penalty=kw["length_penalty"], max_length=MAX_LEN[b], suppress_blank=kw["suppress_blank"],
                      suppress_tokens=kw["suppress_tokens"], max_initial_timestamp_index=kw["max_initial_timestamp_index"],
                      trace=True)


@functools.lru_cache(maxsize=None)
def oracle_run(session_beam: int) -> Dict[int, tuple]:
    out = {}
    for b, prompt in enumerate(prompts(session_beam)):
        if _streams(session_beam)[b][0] == "sample":
            continue
        o = stream_opts(session_beam, b)
        step = ScriptStep(Script(SP, prompt, o, *SCRIPT[session_beam]))
        out[b] = (search_stream(step, prompt, SP, o, stream_index=b), step.events)
    return out


# ---------------------------------------------------------------------------------------------------------- CPU part
@pytest.mark.parametrize("session_beam", [5, 1])
def test_beams_scenario_has_no_near_tie(session_beam):
    for b, (res, events) in oracle_run(session_beam).items():
        k = stream_opts(session_beam, b).beam_size
        assert not near_ties(res, events, k), (session_beam, b, near_ties(res, events, k)[:5])
        assert res.sequences_ids, (session_beam, b)


def test_widths_change_the_oracle_result():
    """The widths matter: at the session's width the narrower streams decode differently, so the device comparison
    below shows that each width reached the kernels."""
    differ = 0
    for b, (res, _ev) in oracle_run(5).items():
        o = stream_opts(5, b)
        if o.beam_size == 5:
            continue
        s = GenOptions(**{**o.__dict__, "beam_size": 5})
        alt = search_stream(ScriptStep(Script(SP, prompts(5)[b], s, *SCRIPT[5])), prompts(5)[b], SP, s, stream_index=b)
        differ += alt.sequences_ids[:1] != res.sequences_ids[:1] or alt.scores[:1] != res.scores[:1]
    assert differ >= 4, differ


# ---------------------------------------------------------------------------------------------------------- GPU part
def _engine():
    from tests.test_search_kernels import engine
    return engine()


def _session(eng, session_beam: int, capacity: int = 10):
    sess = eng.open_decode_session(capacity=capacity, beam_size=session_beam, num_hypotheses=nh(session_beam), **SESSION)
    sess.script(SCRIPT[session_beam])
    return sess


def _admit(sess, session_beam: int, take: List[int]) -> List[int]:
    ps = prompts(session_beam)
    specs = [SAMPLE if _streams(session_beam)[b][0] == "sample" else None for b in take]
    return sess.admit([None] * len(take), [ps[b] for b in take], [MAX_LEN[b] for b in take],
                      sampling=specs if any(s is not None for s in specs) else None,
                      rules=[rules_for(session_beam, b) for b in take])


def _run_session(eng, session_beam: int, order: List[int], first: int, capacity: int = 10):
    """Admit ``order[:first]``, run a few steps, then admit the rest as indices free up; results and the peek of each
    finished index, by stream."""
    sess = _session(eng, session_beam, capacity)
    where, got, peeked = {}, {}, {}
    queue = list(order)

    def admit(k):
        take = [queue.pop(0) for _ in range(min(k, len(queue), len(sess.free_indices())))]
        if take:
            where.update(zip(_admit(sess, session_beam, take), take))
    admit(first)
    sess.run(max_steps=3)
    while queue:
        admit(len(queue))
        done = sess.run(max_steps=4)
        if done:
            for (toks, score, _ns, _step, final), ix in zip(sess.peek(done), done):
                assert final, ix
                peeked[where[ix]] = (toks, score)
        for ix in done:
            got[where.pop(ix)] = sess.collect(ix)
    _drain(sess, where, got, peeked)
    sess.close()
    return got, peeked


def _one_shot(eng, session_beam: int, b: int):
    p = prompts(session_beam)[b]
    if _streams(session_beam)[b][0] == "sample":
        t, n, seed, _key = SAMPLE
        kw = dict(SESSION, beam_size=1, num_hypotheses=n, sampling_topk=0, sampling_temperature=t, seed=seed)
    else:
        kw = dict(stream_kw(session_beam, b), num_hypotheses=nh(session_beam))
    one, _nh, _ = eng.test_search([p], SCRIPT[session_beam], max_length=MAX_LEN[b], prefill=True, **kw)
    return one[0]


ARRANGEMENTS = {5: [(None, None, 10), ("reversed", 2, 10), ([3, 0, 6, 9, 1, 5, 8, 2, 7, 4], 1, 3)],
                1: [(None, None, 6), ("reversed", 2, 6), ([3, 0, 5, 1, 4, 2], 1, 2)]}


@pytest.mark.gpu
@pytest.mark.parametrize("session_beam", [5, 1])
def test_mixed_widths_match_the_oracle_and_one_shot(session_beam):
    eng = _engine()
    n = len(_streams(session_beam))
    runs = []
    for order, first, cap in ARRANGEMENTS[session_beam]:
        if order is None:
            order, first = list(range(n)), n
        elif order == "reversed":
            order = list(reversed(range(n)))
        runs.append(_run_session(eng, session_beam, order, first, cap))
    oracle = oracle_run(session_beam)
    for b in range(n):
        one = _one_shot(eng, session_beam, b)
        for k, (got, peeked) in enumerate(runs):
            g, what = got[b], f"session beam {session_beam} stream {b} {_streams(session_beam)[b]} run {k}"
            # bit for bit the one-shot search at the stream's own width (width 1: the greedy one-shot)
            assert g.sequences_ids == one.sequences_ids, what
            assert g.scores == one.scores, what
            assert g.steps == one.steps, what
            assert g.no_speech_prob == one.no_speech_prob, what
            if b in peeked:
                assert peeked[b][0] == g.sequences_ids[0] and peeked[b][1] == g.scores[0], what
        if b in oracle:
            res, g = oracle[b][0], runs[0][0][b]
            what = f"session beam {session_beam} stream {b} against the oracle"
            assert g.sequences_ids == res.sequences_ids[:len(g.sequences_ids)], what
            np.testing.assert_allclose(g.scores, res.scores[:len(g.scores)], rtol=0, atol=SCORE_TOL, err_msg=what)
            assert abs(g.no_speech_prob - res.no_speech_prob) <= NOSPEECH_TOL, what
            assert g.steps == res.steps + len(prompts(session_beam)[b]) - 1, (what, g.steps, res.steps)


@pytest.mark.gpu
def test_peek_of_running_streams_at_every_width():
    """A stream still decoding reports its leading row -- row 0 of its own beam, or its greedy row -- and that row is
    the prefix of what one-shot decoding at its width has generated by then (the interim hypothesis of a beam need not
    be a prefix of the final one, so only its length and step are checked against the final)."""
    eng = _engine()
    sess = _session(eng, 5)
    take = [0, 1, 3, 4, 5]
    idx = _admit(sess, 5, take)
    sess.run(max_steps=6, break_on_finish=False)
    for (toks, _score, _ns, step, final), b in zip(sess.peek(idx), take):
        one = _one_shot(eng, 5, b)
        assert not final or toks == one.sequences_ids[0], b
        if not final:
            assert len(toks) <= step <= 6, (b, len(toks), step)
            if stream_kw(5, b)["beam_size"] == 1:
                assert toks == one.sequences_ids[0][:len(toks)], b       # greedy: a prefix of its final text
    sess.close()


@pytest.mark.gpu
def test_bad_widths_fail_the_whole_admission():
    from whisperlive_b200._lib import WlError
    eng = _engine()
    for session_beam, rows in ((5, 5), (1, 4)):
        sess = _session(eng, session_beam)
        # streams already in the loop, one of them narrower than the session
        first = [0, 3] if session_beam == 5 else [1, 4]
        idx = _admit(sess, session_beam, first)
        where = dict(zip(idx, first))
        sess.run(max_steps=3)
        free = len(sess.free_indices())
        good = dict(RULES[1])
        for bad, field in ((dict(good, beam_size=rows + 1), "beam_size"), (dict(good, beam_size=-1), "beam_size"),
                           (dict(good, beam_size=rows, patience=16.6 / rows + 0.1), "patience")):
            with pytest.raises(WlError, match=field):
                sess.admit([None, None], prompts(session_beam)[:2], MAX_LEN[:2], rules=[good, bad])
            assert sess.live == len(first) and len(sess.free_indices()) == free
        # the patience bound is the stream's own width times its patience: 3 x 4.3 = 12.9 fits
        ok = sess.admit([None], prompts(session_beam)[2:3], MAX_LEN[2:3], rules=[dict(good, beam_size=3, patience=4.3)])
        got, peeked = {}, {}
        _drain(sess, {**where, ok[0]: -1}, got, peeked)
        for b in first:
            one = _one_shot(eng, session_beam, b)
            assert got[b].sequences_ids == one.sequences_ids and got[b].scores == one.scores, (session_beam, b)
        kw = {**SESSION, **good, "beam_size": 3, "patience": 4.3}
        one, _nh, _ = eng.test_search([prompts(session_beam)[2]], SCRIPT[session_beam], max_length=MAX_LEN[2], prefill=True,
                                      num_hypotheses=nh(session_beam), **kw)
        assert got[-1].sequences_ids == one[0].sequences_ids and got[-1].scores == one[0].scores
        sess.close()


# ---------------------------------------------------------------------------------------------------------- tiny
@pytest.mark.gpu
def test_widths_on_tiny_equal_one_shot_generate():
    """On the decoder (tiny, random weights): streams at beam 1, 2 and 5 in one beam-5 session give the hypotheses
    one-shot ``generate`` gives each at its beam -- the same tokens, or a divergence explained as a near-tie."""
    from tests.test_gpu_parity import MARGIN_TOL, _explain_beam_divergence, engine, feats_for
    from tests.test_session_rules import SCORE_TOL_TINY, _score_tol
    eng, orc = engine("tiny", seed=0)
    dims, sp = eng.dims, orc.spec
    widths = [1, 2, 5, 1]
    n = len(widths)
    feats = np.stack([feats_for(dims, d, 120 + i) for i, d in enumerate([6.0, 9.0, 5.0, 12.0])])
    enc = eng.encode(feats)
    base = [sp.sot, sp.sot + 1, sp.sot + 1 + dims.num_languages + 1]
    prompts_ = [base, base, base, [sp.timestamp_begin - 3, 400, 1234, 11] + base]
    session_kw = dict(beam_size=5, suppress_tokens=[1, 2, 3], return_scores=True, return_no_speech_prob=True)
    rules = [dict(beam_size=1, suppress_tokens=[1, 2, 3]), dict(beam_size=2, suppress_tokens=[1, 2, 3], patience=2.0),
             None, dict(beam_size=1, suppress_tokens=[1, 2, 3], length_penalty=0.6)]
    own = [dict(session_kw, **(r or {})) for r in rules]
    sess = eng.open_decode_session(capacity=n, **session_kw)
    idx = sess.admit([enc.select([b]) for b in range(n)], prompts_, [448] * n, rules=rules)
    where = dict(zip(idx, range(n)))
    got, peeked = {}, {}
    _drain(sess, where, got, peeked)
    sess.close()
    oenc = None
    for b in range(n):
        what = f"tiny width {widths[b]} stream {b}"
        g, toks = got[b], got[b].sequences_ids[0]
        lp = own[b].get("length_penalty", 1.0)
        assert peeked[b][0] == toks and peeked[b][1] == g.scores[0], what
        one = eng.generate(enc.select([b]), [prompts_[b]], max_length=448, **own[b])[0]
        assert abs(g.no_speech_prob - one.no_speech_prob) < 2e-3, what
        if one.sequences_ids[0] == toks:
            assert abs(g.scores[0] - one.scores[0]) <= _score_tol(len(toks), lp, 2e-3), (what, g.scores, one.scores)
            continue
        # the prefill's and the decode GEMMs' splits differ with the rows sharing a call: a near-tie, explained on the
        # oracle
        if oenc is None:
            oenc = orc.encode(feats)
        ref = orc.generate(oenc.select([b]), [prompts_[b]], max_length=448, **own[b])[0]
        if ref.sequences_ids[0] == toks:
            assert abs(g.scores[0] - ref.scores[0]) <= _score_tol(len(toks), lp, 0.02), (what, g.scores, ref.scores)
        elif widths[b] > 1:
            _explain_beam_divergence(eng, enc.select([b]), orc, oenc.select([b]), 0, prompts_[b],
                                     dict(own[b], max_length=448), g, ref, what)
        else:
            i = next((k for k, (x, y) in enumerate(zip(toks, ref.sequences_ids[0])) if x != y), len(toks))
            margins = ref.margins[max(0, i - 1): i + 2]
            assert margins and min(margins) < MARGIN_TOL, (what, i, margins)
        assert abs(g.scores[0] - one.scores[0]) <= _score_tol(len(toks), lp, SCORE_TOL_TINY), (what, g.scores, one.scores)
    enc.release()
