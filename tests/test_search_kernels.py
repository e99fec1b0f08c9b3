"""The search kernels of csrc/search.cu (search_rows, search_streams, decode_init, loop_condition) against
``oracle.search`` on scripted logits.

``wl_test_search`` is ``wl_generate`` with the decoder replaced by ``scripted_logits_kernel``: a row's logits are a pure
function of the tokens it has consumed, restated bit for bit by tests/search_script.py.  The oracle runs on the CPU with
a step function serving the same numbers, so:

* every scenario's seeds are chosen so that no decision margin of the oracle's run falls in (0, 1e-5] -- the candidate
  boundaries of every beam step, the timestamp-probability rule, the arg-max / Gumbel-max of every greedy or sampled
  row.  The device's fp32 log-softmax differs from torch's by ~1e-7, so the comparison is exact: same tokens, same
  order, same step count; scores to 1e-4 and the no-speech probability to 1e-6.  Exact ties (margin 0) are kept on
  purpose: they break by token id, then by row, on both sides;
* the CPU part (the oracle on the script, the margins, the coverage tallies and the patience rounding) runs without a
  GPU; the device comparisons are marked ``gpu``.
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np
import pytest

from oracle.search import GenOptions, VocabSpec, max_candidates, search_stream
from tests.search_script import Script, ScriptStep

MARGIN = 1e-5
SCORE_TOL = 1e-4
NOSPEECH_TOL = 1e-6
MAX_STREAMS, MAX_BEAM = 32, 8

V3 = VocabSpec.from_vocab_size(51866)     # large-v3's vocabulary: 2 padding columns in a row of 51868


def sot_seq(sp: VocabSpec) -> List[int]:
    if sp.vocab < 51865:
        return [sp.sot]
    return [sp.sot, sp.sot + 1, sp.timestamp_begin - 5]      # <|en|> <|transcribe|>


def sot_prev(sp: VocabSpec) -> int:
    return sp.timestamp_begin - 3


def bench_suppress(sp: VocabSpec) -> List[int]:
    """Like the benchmark's: EOT, the special tokens of the sot sequence and a set of punctuation-like text ids."""
    tb = sp.timestamp_begin
    return sorted({sp.eot, sp.sot, tb - 6, tb - 5, tb - 4, tb - 3, tb - 2, 1, 2, 7, 8, 9, 10, 14, 25, 26, 27, 28, 29, 31,
                   58, 59, 60, 61, 62, 63, 90, 91, 92, 93})


def prompt_kinds(sp: VocabSpec, i: int) -> List[int]:
    """Prompt i of a cycle: plain sot sequence, <|startofprev|> history, a prefix with and without a leading <|0.00|>,
    <|notimestamps|>, and sot as the last prompt token."""
    s = sot_seq(sp)
    tb = sp.timestamp_begin
    kinds = [
        s,
        [sot_prev(sp), 1000 + i, 2000 + 7 * i, tb + 20, 3000] + s,
        s + [440 + i, 1212],
        s + [tb, 900 + i, 1700],
        s + [sp.no_timestamps],
        [sot_prev(sp), 500 + i, sp.sot],
        [sp.sot],
    ]
    return kinds[i % len(kinds)]


@dataclass
class Scenario:
    name: str
    prompts: List[List[int]]
    kw: Dict
    script: Tuple[int, int]
    max_length: List[int] = field(default_factory=list)

    def opts(self, b: int) -> GenOptions:
        kw = self.kw
        return GenOptions(beam_size=kw.get("beam_size", 5), patience=kw.get("patience", 1.0),
                          num_hypotheses=kw.get("num_hypotheses", 1), length_penalty=kw.get("length_penalty", 1.0),
                          max_length=self.max_length[b], suppress_blank=kw.get("suppress_blank", True),
                          suppress_tokens=kw.get("suppress_tokens", ()),
                          max_initial_timestamp_index=kw.get("max_initial_timestamp_index", 50),
                          sampling_topk=kw.get("sampling_topk", 1), sampling_temperature=kw.get("sampling_temperature", 1.0),
                          seed=kw.get("seed", 0), trace=True)

    def device_kw(self) -> Dict:
        return dict(self.kw, max_length=max(self.max_length), max_length_per_stream=self.max_length)


def _scenarios() -> List[Scenario]:
    sp = V3
    sc: List[Scenario] = []
    # the benchmark's shape: 32 streams x beam 4 = 128 rows, EOT suppressed, ragged max_length
    sc.append(Scenario("bench_b32_k4", [prompt_kinds(sp, i) if i % 4 == 1 else sot_seq(sp) for i in range(32)],
                       dict(beam_size=4, suppress_tokens=bench_suppress(sp), suppress_blank=False), (11, -1),
                       [2 * (6 + i % 7) for i in range(32)]))
    sc.append(Scenario("beam8", [prompt_kinds(sp, i) for i in range(6)], dict(beam_size=8, num_hypotheses=4), (23, -1),
                       [40] * 6))
    for nh in (1, 3):
        sc.append(Scenario(f"greedy_nh{nh}", [prompt_kinds(sp, i) for i in range(7)], dict(beam_size=1, num_hypotheses=nh),
                           (5 + nh, -1), [48] * 7))
    for T, seed, nh in ((0.3, 3, 4), (1.0, 17, 8), (1.7, 29, 6)):
        sc.append(Scenario(f"sample_t{T}", [prompt_kinds(sp, i) for i in range(7)],
                           dict(beam_size=1, num_hypotheses=nh, sampling_topk=0, sampling_temperature=T, seed=seed),
                           (40 + seed, -1), [30] * 7))
    for lp in (0.0, 1.0, 0.6):
        sc.append(Scenario(f"length_penalty_{lp}", [prompt_kinds(sp, i) for i in range(7)],
                           dict(beam_size=4, num_hypotheses=4, length_penalty=lp), (60 + int(10 * lp), -1), [36] * 7))
    for K, pat in ((5, 0.5), (4, 1.0), (3, 1.5), (5, 3.0)):
        sc.append(Scenario(f"patience_k{K}_{pat}", [prompt_kinds(sp, i) for i in range(7)],
                           dict(beam_size=K, patience=pat, num_hypotheses=min(16, max_candidates(K, pat) + K - 1)),
                           (80 + K, -1), [44] * 7))
    # every special token suppressed and a history ending in <text> <|ts|> near the end of the vocabulary: the first step
    # allows EOT and the last few timestamps only, so an EOT closure finds no secondary candidate
    V, tb = sp.vocab, sp.timestamp_begin
    sc.append(Scenario("few_candidates", [sot_seq(sp) + [100 + i, V - 1] for i in range(6)],
                       dict(beam_size=4, num_hypotheses=3, suppress_blank=False, suppress_tokens=list(range(sp.eot + 1, tb))),
                       (7, -1), [30] * 6))
    # beam 8, patience 2 (max_cand 16) and most text suppressed, so EOT closes often: the last step closes up to 8
    # hypotheses on top of as many as 15, and the table must hold all 23
    keep = set(range(3000, 3040))
    sc.append(Scenario("hyp_table", [sot_seq(sp) + [sp.no_timestamps]] * 2,
                       dict(beam_size=8, patience=2.0, num_hypotheses=16,
                            suppress_tokens=[t for t in range(sp.eot) if t not in keep]), (300, -1), [28, 26]))
    for pattern in range(6):
        sc.append(Scenario(f"pattern_{pattern}", [prompt_kinds(sp, i) for i in range(7)], dict(beam_size=4, num_hypotheses=2),
                           (100 + pattern, pattern), [30] * 7))
    return sc


SCENARIOS = {s.name: s for s in _scenarios()}


@functools.lru_cache(maxsize=None)
def oracle_run(name: str):
    """The oracle on every stream of a scenario: (results, step events) per stream."""
    s = SCENARIOS[name]
    out = []
    for b, prompt in enumerate(s.prompts):
        o = s.opts(b)
        step = ScriptStep(Script(V3, prompt, o, *s.script))
        res = search_stream(step, prompt, V3, o, stream_index=b)
        out.append((res, step.events))
    return out


def near_ties(res, events, K: int) -> List[str]:
    """Decisions of one oracle run whose margin lies in (0, MARGIN]."""
    bad = []
    for ev in events:
        if ev["rule_e"] is not None and 0 < ev["rule_e_margin"] <= MARGIN:
            bad.append(f"rule e margin {ev['rule_e_margin']:.3g}")
    if K > 1:
        for i, t in enumerate(res.trace):
            tot = [c[2] for c in t["cand"][:2 * K + 1] if math.isfinite(c[2])]
            for a, b in zip(tot, tot[1:]):
                if 0 < a - b <= MARGIN:
                    bad.append(f"step {i}: candidate gap {a - b:.3g}")
    else:
        margins = list(res.margins) + [m for ms in res.row_margins.values() for m in ms]
        bad += [f"arg-max margin {m:.3g}" for m in margins if 0 < m <= MARGIN]
    return bad


# ---------------------------------------------------------------------------------------------------------- CPU part
@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_scenario_has_no_near_tie(name):
    """The seeds keep every decision of the oracle's run away from (0, 1e-5]: the device comparison can be exact."""
    s = SCENARIOS[name]
    K = s.kw.get("beam_size", 5)
    for b, (res, events) in enumerate(oracle_run(name)):
        assert not near_ties(res, events, K), (name, b, near_ties(res, events, K)[:5])
        assert res.sequences_ids, (name, b)


def test_coverage_tallies():
    """Across the scenario set every fragile branch of the search is taken at least once."""
    tally = dict.fromkeys(["rule_e_fires", "rule_e_holds", "rule_c_no_ts", "rule_c_no_text", "rule_d_cutoff", "first_step_bound",
                           "eot_refilled", "secondary_ran_out", "stop_max_cand", "last_step_closure", "tie",
                           "tie_same_thread", "tie_between_rows"] + [f"pattern_{p}" for p in range(6)], 0)
    for name, s in SCENARIOS.items():
        K = s.kw.get("beam_size", 5)
        for res, events in oracle_run(name):
            for ev in events:
                tally[f"pattern_{ev['pattern']}"] += 1
                tally["rule_e_fires"] += ev["rule_e"] is True
                tally["rule_e_holds"] += ev["rule_e"] is False
                tally["rule_c_no_ts"] += ev["rule_c"] == "no_ts"
                tally["rule_c_no_text"] += ev["rule_c"] == "no_text"
                tally["rule_d_cutoff"] += bool(ev["rule_d"])
                tally["first_step_bound"] += bool(ev["first"])
                tally["tie"] += bool(ev.get("tie"))
                tally["tie_same_thread"] += bool(ev.get("tie_same_thread"))
            if K > 1:
                tally["stop_max_cand"] += res.stop == "max_cand"
                for t in res.trace:
                    tally["eot_refilled"] += t.get("refilled", 0) > 0 and t.get("closed_eot", 0) > 0
                    tally["secondary_ran_out"] += t.get("ran_out", 0) > 0 and t.get("n_alive", K) < K
                    tally["last_step_closure"] += t.get("closed_last", 0) > 0
                    top = [c for c in t["cand"][:2 * K] if math.isfinite(c[2])]
                    tally["tie_between_rows"] += any(a[2] == b[2] and a[0] != b[0] for a, b in zip(top, top[1:]))
    missing = [k for k, v in tally.items() if v == 0]
    assert not missing, (missing, tally)


def test_oracle_patience_rounds_half_away_from_zero():
    assert max_candidates(5, 0.5) == 3
    assert max_candidates(3, 1.5) == 5
    assert max_candidates(5, 2.5) == 13
    assert max_candidates(4, 1.0) == 4
    assert max_candidates(5, 0.01) == 1          # at least one hypothesis
    assert max_candidates(8, 2.0) == 16


def test_hypothesis_table_scenario_overflows_sixteen():
    """A stream of the hypothesis-table scenario finishes with more than 16 hypotheses: the device's table must hold
    max_cand + K - 1 of them (a table of 16 drops the last ones and, at the last step, possibly the best)."""
    res = [r for r, _ in oracle_run("hyp_table")]
    assert max(r.n_hypotheses for r in res) > 16, [r.n_hypotheses for r in res]


def all_masked_prompt(sp: VocabSpec) -> Tuple[List[int], Dict]:
    """Timestamps on, max_initial_timestamp_index = 0 and <|0.00|> suppressed: the first step masks every token."""
    return sot_seq(sp), dict(max_initial_timestamp_index=0, suppress_tokens=[sp.timestamp_begin])


@pytest.mark.parametrize("beam", [1, 4])
def test_oracle_row_with_every_token_masked(beam):
    prompt, kw = all_masked_prompt(V3)
    o = GenOptions(beam_size=beam, num_hypotheses=2, max_length=20, trace=True, **kw)
    res = search_stream(ScriptStep(Script(V3, prompt, o, 1, 0)), prompt, V3, o)
    assert res.steps == 1
    if beam == 1:
        assert res.sequences_ids == [[], []] and res.scores == [0.0, 0.0]
    else:
        assert res.sequences_ids == [] and res.n_hypotheses == 0


# ---------------------------------------------------------------------------------------------------------- GPU part
_ENG: Dict[int, object] = {}


def engine(vocab: int = 51866):
    """A micro-shaped context (the decoder is never run) with the given vocabulary."""
    if vocab not in _ENG:
        from whisperlive_b200.config import WhisperDims
        from whisperlive_b200.engine import B200Whisper
        from whisperlive_b200.weights import random_init
        dims = WhisperDims(f"micro-{vocab}", 128, 2, 2, 2, 80, vocab)
        _ENG[vocab] = B200Whisper(dims, random_init(dims, seed=0), max_streams=MAX_STREAMS, max_beam=MAX_BEAM)
    return _ENG[vocab]


@pytest.mark.gpu
@pytest.mark.parametrize("vocab", [51864, 51865, 51866])
@pytest.mark.parametrize("search", ["beam4", "sample3", "feed"])
def test_first_step_logits_bit_exact(vocab, search):
    """The hook's first-step logits equal the numpy script bit for bit in every row; inactive rows and the padding
    columns are NaN."""
    eng = engine(vocab)
    sp = VocabSpec.from_vocab_size(vocab)
    prompts = [prompt_kinds(sp, i) for i in range(7)]
    kw = dict(suppress_tokens=[t for t in bench_suppress(sp) if t != sp.eot], max_length=40)
    if search == "beam4":
        kw.update(beam_size=4, prefill=True)
    elif search == "sample3":
        kw.update(beam_size=1, num_hypotheses=3, sampling_topk=0, sampling_temperature=0.7, prefill=True)
    else:
        kw.update(beam_size=4, prefill=False)
    Kr = kw["beam_size"] if kw["beam_size"] > 1 else kw["num_hypotheses"]
    _, _, logits = eng.test_search(prompts, (7, -1), return_logits=True, **kw)
    Vld = (vocab + 3) // 4 * 4
    assert logits.shape == (len(prompts) * Kr, Vld)
    o = GenOptions(beam_size=kw["beam_size"], max_length=40, suppress_tokens=kw["suppress_tokens"])
    for b, prompt in enumerate(prompts):
        script = Script(sp, prompt, o, 7, -1)
        active = (Kr if search == "sample3" else 1)
        for j in range(Kr):
            row = logits[b * Kr + j]
            if j >= active:
                assert np.isnan(row).all(), (b, j)
                continue
            seq = prompt if search != "feed" else prompt[:1]
            want = script.logits(seq)
            np.testing.assert_array_equal(row[:vocab].view(np.uint32), want.view(np.uint32), err_msg=f"stream {b} row {j}")
            assert np.isnan(row[vocab:]).all()


def compare(name: str, got, nhyp) -> None:
    s = SCENARIOS[name]
    K = s.kw.get("beam_size", 5)
    for b, ((res, _), g) in enumerate(zip(oracle_run(name), got)):
        where = f"{name} stream {b}"
        assert g.sequences_ids == res.sequences_ids, where
        np.testing.assert_allclose(g.scores, res.scores, rtol=0, atol=SCORE_TOL, err_msg=where)
        assert abs(g.no_speech_prob - res.no_speech_prob) <= NOSPEECH_TOL, (where, g.no_speech_prob, res.no_speech_prob)
        assert g.steps == res.steps + len(s.prompts[b]) - 1, (where, g.steps, res.steps)
        want_hyps = res.n_hypotheses if K > 1 else len(res.row_tokens)
        assert nhyp[b] == want_hyps, (where, nhyp[b], want_hyps)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_search_matches_oracle(name):
    """Every feeding mode and loop mode gives the oracle's tokens, order, scores, no-speech probability and steps, and
    the four runs give bit-identical tokens, scores and steps.  (The no-speech probability of a stream whose sot
    precedes its last prompt token comes from the prefill pass in one feeding mode and from search_rows in the other,
    so it is held to the oracle's tolerance only.)"""
    eng = engine()
    s = SCENARIOS[name]
    runs = []
    for prefill in (True, False):
        for graph in (True, False):
            got, nhyp, _ = eng.test_search(s.prompts, s.script, prefill=prefill, use_cuda_graph=graph, **s.device_kw())
            compare(name, got, nhyp)
            runs.append([(g.sequences_ids, g.scores, g.steps, nh) for g, nh in zip(got, nhyp)])
    assert all(r == runs[0] for r in runs[1:])


@pytest.mark.gpu
@pytest.mark.parametrize("beam", [1, 4])
def test_row_with_every_token_masked(beam):
    eng = engine()
    prompt, kw = all_masked_prompt(V3)
    o = GenOptions(beam_size=beam, num_hypotheses=2, max_length=20, **kw)
    want = search_stream(ScriptStep(Script(V3, prompt, o, 1, 0)), prompt, V3, o)
    for prefill in (True, False):
        got, nhyp, _ = eng.test_search([prompt], (1, 0), beam_size=beam, num_hypotheses=2, max_length=20, prefill=prefill, **kw)
        assert got[0].sequences_ids == want.sequences_ids and got[0].scores == want.scores
        assert got[0].steps == want.steps + len(prompt) - 1


@pytest.mark.gpu
def test_patience_above_the_table_is_an_error():
    from whisperlive_b200._lib import WlError
    eng = engine()
    with pytest.raises(WlError, match="limit of 16"):
        eng.test_search([sot_seq(V3)], (1, 0), beam_size=8, patience=2.1, max_length=20)
    with pytest.raises(WlError, match="limit of 16"):
        eng.open_decode_session(beam_size=8, patience=2.1)
    got, _, _ = eng.test_search([sot_seq(V3)], (1, 0), beam_size=8, patience=2.0, max_length=20)   # 16 is allowed
    assert got[0].sequences_ids
