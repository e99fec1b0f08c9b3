"""Temperature-fallback sampling inside the running decode loop: a stream admitted into a decode session with a
per-stream sampling spec (``DecodeSession.admit(..., sampling=...)``, ``wl_session_admit_ex``) and the transcriber's step
rounds, which send every rung of the ladder that fits the open session there instead of to a run-to-completion
``generate`` call.

The CPU tests drive the transcriber over the oracle engine with a CPU model of such a session (below): a sampled
stream's result is what the oracle's search gives it with that seed and with the noise key as its stream index.  The
GPU tests check the device session against one-shot ``generate`` calls."""
import math

import numpy as np
import pytest
import torch

from oracle.engine import GenerationResult, OracleDecodeSession
from oracle.search import GenOptions, search_stream
from tests.test_boundary_cpu import _oracle_model
from whisperlive_b200 import synth

# every window climbs the whole ladder: no average log-probability reaches 0
FORCED = dict(temperature=[0.0, 0.2, 0.4, 0.6, 0.8, 1.0], beam_size=5, best_of=5, log_prob_threshold=0.0,
              compression_ratio_threshold=None, no_speech_threshold=None, language="en", vad_filter=False)


def oracle_sample(orc, feature, prompt, max_length, kw, temperature, n, seed, key) -> GenerationResult:
    """What the oracle's ``generate(seed=seed)`` returns for a stream at batch position ``key`` (Gumbel-max sampling,
    ``n`` independent rows), with the per-row key margins of the search."""
    opts = GenOptions(beam_size=1, num_hypotheses=int(n), length_penalty=kw.get("length_penalty", 1),
                      max_length=int(max_length), suppress_blank=kw.get("suppress_blank", True),
                      suppress_tokens=[t for t in (kw.get("suppress_tokens") or ()) if t >= 0],
                      max_initial_timestamp_index=kw.get("max_initial_timestamp_index", 50), sampling_topk=0,
                      sampling_temperature=float(temperature), seed=int(seed))
    r = search_stream(orc._stream_step_fn(orc._as_encoded(feature), 0), list(prompt), orc.spec, opts, stream_index=int(key))
    g = GenerationResult(r.sequences_ids, r.scores, r.no_speech_prob, r.steps, r.margins)
    g.row_margins, g.row_tokens = r.row_margins, r.row_tokens
    return g


class SamplingOracleSession(OracleDecodeSession):
    """CPU model of a decode session whose streams may sample (``sampling`` specs of ``DecodeSession.admit``).  Records
    the session step of every sampled admission."""

    def __init__(self, engine, capacity, **kw):
        super().__init__(engine, capacity, **kw)
        beam = int(kw.get("beam_size", 5))
        self.rows_per_stream = beam if beam > 1 else int(kw.get("num_hypotheses", 1))
        self.sampled_at = []

    def admit(self, features, prompts, max_lengths, indices=None, sampling=None):
        if sampling is None:
            return super().admit(features, prompts, max_lengths, indices)
        free = self.free_indices()
        if indices is None:
            if len(prompts) > len(free):
                raise RuntimeError(f"admit: {len(prompts)} streams for {len(free)} free indices")
            indices = free[:len(prompts)]
        for sp in sampling:
            if sp is not None and not (1 <= sp[1] <= self.rows_per_stream and math.isfinite(sp[0]) and sp[0] > 0 and sp[3] >= 0):
                raise ValueError(f"admit: bad sampling spec {sp}")
        for i, f, p, ml, sp in zip(indices, features, prompts, max_lengths, sampling):
            if sp is None:
                super().admit([f], [p], [ml], [i])
                continue
            r = oracle_sample(self.engine, f, p, ml, self.kw, *sp)
            self._res[i] = r
            self._left[i] = max(1, int(r.steps) - (len(p) - 1))
            self.sampled_at.append(self.steps)
        return list(indices)


def _sampling_oracle_model():
    """The oracle transcriber with sampling-capable decode sessions; every ``generate`` call is recorded."""
    model = _oracle_model()
    orc = model.model
    sessions, calls = [], []

    def open_decode_session(capacity=None, **kw):
        sessions.append(SamplingOracleSession(orc, capacity or 8, **kw))
        return sessions[-1]
    orc.open_decode_session = open_decode_session
    generate = orc.generate

    def counted(*a, **kw):
        calls.append(kw)
        return generate(*a, **kw)
    orc.generate = counted
    return model, sessions, calls


def _sampling_calls(calls):
    return sum(1 for kw in calls if kw.get("beam_size", 5) == 1 and kw.get("sampling_temperature", 0) > 0)


def _step_rounds(model, waves, kws, late_rounds, max_steps=4):
    """Step rounds over ``waves``: stream i is added before round ``late_rounds[i]`` (in stream order)."""
    sess = model.open_session()
    handles, results, rounds = [], {}, 0
    todo = list(range(len(waves)))
    while todo or sess.pending():
        while todo and late_rounds[todo[0]] <= rounds:
            i = todo.pop(0)
            handles += sess.add_streams([waves[i]], [kws[i]])
        sess.step_round(max_steps)
        rounds += 1
        for e in sess.pop_finished():
            results[e.handle] = sess.result_of(e)
        assert rounds < 2000
    sess.close()
    out = []
    for h in handles:
        segs, _info = results[h]
        out.append([(s.tokens, s.start, s.end, s.temperature) for s in segs])
    return out, sess


def _segments_equal(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert x == y, f"stream {i}"


@pytest.fixture(scope="module")
def forced_runs():
    torch.set_num_threads(4)
    waves = [synth.speech_like(d, seed=90 + i) for i, d in enumerate((34.0, 41.0, 33.0, 38.0, 36.0))]
    kws = [dict(FORCED, max_new_tokens=16)] * len(waves)
    runs = {}
    for name, late in (("together", [0, 0, 0, 0, 0]), ("staggered", [0, 0, 2, 5, 9])):
        model, sessions, calls = _sampling_oracle_model()
        segs, sess = _step_rounds(model, waves, kws, late)
        runs[name] = dict(segs=segs, sessions=sessions, calls=calls, admitted=list(sess.admitted_steps))
    return runs


def test_sampling_rungs_join_the_running_loop(forced_runs):
    """Every sampling rung of a forced ladder (beam 5, best_of 5) is decoded inside the open decode session: the engine
    gets no sampling ``generate`` call, and sampled streams join a loop that is already running."""
    for name, run in forced_runs.items():
        assert _sampling_calls(run["calls"]) == 0, name
        sampled = [s for ses in run["sessions"] for s in ses.sampled_at]
        assert len(sampled) >= 5 * len(run["segs"]), (name, len(sampled))   # >= 5 rungs per stream's first window
        assert any(s > 0 for s in sampled), name
        temps = {t for segs in run["segs"] for (_tok, _s, _e, t) in segs}
        assert temps and max(temps) > 0, name                            # sampled windows reach the segments


def test_sampled_segments_do_not_depend_on_arrival(forced_runs):
    """Streams added together and streams added over several rounds (same order) give identical segments: a sampled
    stream's noise depends only on the stream itself, not on who shares its rounds."""
    _segments_equal(forced_runs["staggered"]["segs"], forced_runs["together"]["segs"])


def test_rungs_that_do_not_fit_take_the_one_shot_path():
    """beam_size=2, best_of=5: a sampling rung needs more rows than the session has, so it runs through ``generate``
    as before, and every stream still completes."""
    torch.set_num_threads(4)
    model, sessions, calls = _sampling_oracle_model()
    waves = [synth.speech_like(d, seed=110 + i) for i, d in enumerate((6.0, 33.0, 5.0))]
    kws = [dict(FORCED, beam_size=2, max_new_tokens=12)] * len(waves)
    segs, sess = _step_rounds(model, waves, kws, [0, 0, 1])
    assert len(segs) == 3                                  # result_of raised for none of them
    assert _sampling_calls(calls) >= 5 * 3
    assert not any(ses.sampled_at for ses in sessions)
    assert sessions and all(ses.rows_per_stream == 2 for ses in sessions)


def test_session_noise_seed_is_documented_mix():
    from whisperlive_b200.transcriber import session_noise_seed
    from oracle.search import _hash_u32

    def h(x):
        return int(_hash_u32(np.asarray([x & 0xFFFFFFFF], dtype=np.uint32))[0])
    for handle, seek, rung in ((0, 0, 1), (3, 3000, 5), (17, 123456, 2)):
        assert session_noise_seed(handle, seek, rung) == h(h(h(handle) ^ seek) ^ rung)
    seeds = {session_noise_seed(a, s, r) for a in range(4) for s in (0, 3000) for r in range(6)}
    assert len(seeds) == 4 * 2 * 6


# --------------------------------------------------------------------------------------------------------- GPU
def _explained_sample(got, ref, orow, n, what, margin_tol):
    """A stream sampled in the session against the one-shot ``generate`` of it (same seed, batch position = key):
    identical, or every differing hypothesis equals an oracle row or leaves the closest one where the oracle's own
    perturbed arg-max was a near-tie."""
    assert len(got.sequences_ids) == n and got.scores == sorted(got.scores, reverse=True), what
    assert abs(got.no_speech_prob - ref.no_speech_prob) < 2e-3, what
    if got.sequences_ids == ref.sequences_ids:
        assert np.allclose(got.scores, ref.scores, atol=2e-3), (what, got.scores, ref.scores)
        return True
    rows = [tuple(t) for t in orow.row_tokens]
    refs = {tuple(s) for s in ref.sequences_ids}
    for gs in got.sequences_ids:
        if tuple(gs) in refs or tuple(gs) in rows:
            continue

        def lcp(t):
            return next((k for k, (x, y) in enumerate(zip(gs, t)) if x != y), min(len(gs), len(t)))
        j = max(range(len(rows)), key=lambda q: lcp(rows[q]))
        i = lcp(rows[j])
        m = orow.row_margins[j][max(0, i - 1): i + 2]
        print(f"{what}: a hypothesis leaves oracle row {j} at token {i}, key margins there {m}")
        assert m and min(m) < margin_tol, (what, j, i, m)
    return False


def _session_setup(name):
    from tests.test_gpu_parity import engine, feats_for
    eng, orc = engine(name, seed=0)
    dims, sp = eng.dims, orc.spec
    durs = [6.0, 9.0, 5.0, 12.0, 7.0, 4.0]
    feats = np.stack([feats_for(dims, d, 60 + i) for i, d in enumerate(durs)])
    enc_a, enc_b = eng.encode(feats[:4]), eng.encode(feats[4:])
    oenc = orc.encode(feats)
    views = [enc_a.select([i]) for i in range(4)] + [enc_b.select([i]) for i in range(2)]
    base = [sp.sot] if not dims.multilingual else [sp.sot, sp.sot + 1, sp.sot + 1 + dims.num_languages + 1]
    rng = np.random.default_rng(23)
    prev = lambda n: [sp.timestamp_begin - 3] + rng.integers(256, 40000, n).tolist()
    prompts = [base, prev(40) + base, base, prev(150) + base, base + [sp.no_timestamps], prev(9) + base]
    lengths = [2 * 30, 448, 2 * 18, 448, 2 * 25, 2 * 40]
    return eng, orc, views, oenc, prompts, lengths, (enc_a, enc_b)


def _run_session(eng, views, prompts, lengths, kw, specs, plan, run_steps=3):
    """Admit stream groups at fixed token steps (``plan``: lists of stream numbers, one list per slice of ``run_steps``
    steps, later lists waiting for free indices), run to the end, collect everything."""
    sess = eng.open_decode_session(capacity=4, **kw)
    where, got, joined_at = {}, {}, {}
    queue = [list(g) for g in plan]
    guard = 0
    while sess.live or queue:
        if queue and len(queue[0]) <= len(sess.free_indices()):
            take = queue.pop(0)
            idx = sess.admit([views[i] for i in take], [prompts[i] for i in take], [lengths[i] for i in take],
                             sampling=[specs.get(i) for i in take])
            for i, ix in zip(take, idx):
                where[ix] = i
                joined_at[i] = sess.steps
        for ix in sess.run(max_steps=run_steps, break_on_finish=False):
            got[where.pop(ix)] = sess.collect(ix)
        guard += 1
        assert guard < 400
    sess.close()
    return got, joined_at, sess


@pytest.mark.gpu
@pytest.mark.parametrize("name,beam", [("micro.en", 5), ("micro", 4), ("tiny", 5)])
def test_mixed_session_samples_like_one_shot_generate(name, beam):
    """Beam streams and sampling streams (T 0.2 / 0.6 / 1.0, 1 / 3 / all rows, noise keys 0 and 1) share one session,
    admitted at different token steps.  Each sampling stream gets what a one-shot sampling ``generate`` with the same
    seed gives it at batch position = key; each beam stream what the one-shot beam ``generate`` gives it."""
    from tests.test_gpu_parity import MARGIN_TOL, _same_hypotheses
    eng, orc, views, oenc, prompts, lengths, encs = _session_setup(name)
    Kr = beam
    kw = dict(beam_size=beam, suppress_tokens=[1, 2, 3], return_scores=True, return_no_speech_prob=True)
    specs = {1: (0.2, 1, 11, 0), 3: (0.6, 3, 12, 1), 5: (1.0, Kr, 13, 0)}
    got, joined_at, sess = _run_session(eng, views, prompts, lengths, kw, specs, [[0, 1], [2], [3, 4], [5]])
    assert sorted(got) == list(range(6))
    assert joined_at[0] == 0 and joined_at[2] > 0 and joined_at[3] > joined_at[2]
    exact = 0
    for i in range(6):
        if i not in specs:
            ref = eng.generate(views[i], [prompts[i]], max_length=lengths[i], **kw)[0]
            _same_hypotheses(got[i], ref, f"{name} beam stream {i}")
            continue
        t, n, seed, key = specs[i]
        skw = dict(kw, beam_size=1, num_hypotheses=n, sampling_topk=0, sampling_temperature=t, seed=seed)
        other = (i + 1) % 6                                # batch position `key` holds the stream, 0 another one
        batch = [views[i]] if key == 0 else [views[other], views[i]]
        ps = [prompts[i]] if key == 0 else [prompts[other], prompts[i]]
        mls = [lengths[i]] if key == 0 else [lengths[other], lengths[i]]
        joined = batch[0] if len(batch) == 1 else batch[0].join(batch)
        ref = eng.generate(joined, ps, max_length=max(mls), max_length_per_stream=mls, **skw)[key]
        orow = oracle_sample(orc, oenc.select([i]), prompts[i], lengths[i], kw, t, n, seed, key)
        exact += _explained_sample(got[i], ref, orow, n, f"{name} sampling stream {i}", MARGIN_TOL)
    print(f"mixed session {name} beam {beam}: joined at {joined_at}, {exact} of {len(specs)} sampling streams token-exact")
    for e in encs:
        e.release()


@pytest.mark.gpu
def test_beam_stream_isolated_from_sampling_neighbours():
    """A beam stream's tokens, scores and no-speech probability are bit-identical whether the other indices hold
    sampling streams or beam streams (same admission schedule, same neighbour prompts)."""
    eng, orc, views, oenc, prompts, lengths, encs = _session_setup("micro.en")
    kw = dict(beam_size=5, suppress_tokens=[1, 2, 3], return_scores=True, return_no_speech_prob=True)
    plan = [[0, 1], [2], [3]]          # never more streams than indices: admissions do not wait for anybody to finish
    a, ja, _ = _run_session(eng, views, prompts, lengths, kw, {1: (0.7, 5, 5, 0), 2: (1.0, 2, 6, 1)}, plan)
    b, jb, _ = _run_session(eng, views, prompts, lengths, kw, {}, plan)
    for i in (0, 3):
        assert ja[i] == jb[i]
        assert a[i].sequences_ids == b[i].sequences_ids, i
        assert a[i].scores == b[i].scores, i
        assert a[i].no_speech_prob == b[i].no_speech_prob, i
    for e in encs:
        e.release()


@pytest.mark.gpu
def test_session_sampling_spec_errors():
    """A bad sampling spec fails the whole admission and leaves the index free; the next valid one succeeds."""
    from tests.test_gpu_parity import engine, feats_for
    eng, orc = engine("micro.en", seed=0)
    dims, sp = eng.dims, orc.spec
    enc = eng.encode(np.stack([feats_for(dims, 5.0, 1), feats_for(dims, 5.0, 2)]))
    v0, v1 = enc.select([0]), enc.select([1])
    sess = eng.open_decode_session(capacity=2, beam_size=4)
    assert sess.rows_per_stream == 4
    for bad in ((0.5, 5, 1, 0), (0.0, 2, 1, 0), (-1.0, 2, 1, 0), (float("nan"), 2, 1, 0), (float("inf"), 2, 1, 0),
                (0.5, 0, 1, 0), (0.5, 2, 1, -1)):
        with pytest.raises(Exception, match="sampl|noise key"):
            sess.admit([v0, v1], [[sp.sot], [sp.sot]], [20, 20], sampling=[None, bad])
        assert sess.free_indices() == [0, 1] and sess.live == 0
    i0, i1 = sess.admit([v0, v1], [[sp.sot], [sp.sot]], [20, 20], sampling=[None, (0.5, 4, 1, 0)])
    done = set()
    for _ in range(40):
        done |= set(sess.run(max_steps=4))
        if len(done) == 2:
            break
    assert done == {i0, i1}
    assert len(sess.collect(i0).sequences_ids) == 1 and len(sess.collect(i1).sequences_ids) == 4
    sess.close()
    enc.release()


@pytest.mark.gpu
def test_transcriber_step_rounds_sample_in_the_session(monkeypatch):
    """The transcriber on step rounds with forced ladders on the device: no one-shot sampling ``generate`` call, and
    streams added together or over several rounds give identical segments."""
    from tests.test_gpu_parity import engine
    from whisperlive_b200.feature_extractor import FeatureExtractor
    from whisperlive_b200.tokenizer import build_synthetic_tokenizer
    from whisperlive_b200.transcriber import B200WhisperModel
    eng, _ = engine("micro.en", seed=0)
    dims = eng.dims
    m = B200WhisperModel("micro.en", engine=eng, hf_tokenizer=build_synthetic_tokenizer(dims.vocab),
                         feature_extractor=FeatureExtractor(eng, dims.n_mels))
    calls = []
    generate = eng.generate

    def counted(*a, **kw):
        calls.append(kw)
        return generate(*a, **kw)
    monkeypatch.setattr(eng, "generate", counted)
    waves = [synth.speech_like(d, seed=120 + i) for i, d in enumerate((34.0, 8.0, 41.0, 6.0))]
    kws = [dict(FORCED)] * len(waves)
    together, s1 = _step_rounds(m, waves, kws, [0, 0, 0, 0], max_steps=5)
    staggered, s2 = _step_rounds(m, waves, kws, [0, 0, 2, 4], max_steps=5)
    assert _sampling_calls(calls) == 0
    assert any(a > 0 for a in s2.admitted_steps)
    assert max(t for segs in together for (_tok, _s, _e, t) in segs) > 0
    _segments_equal(staggered, together)
    print(f"transcriber step rounds: admissions at session steps {s2.admitted_steps}")
