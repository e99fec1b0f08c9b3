"""``BatchedInferencePipeline`` (whisperlive_b200/transcriber.py) on the host, over the CPU oracle engine, against
tests/golden/batched_reference.json: the reference's vendored pipeline executed over the same engine, with the two
faster-whisper 1.2.0 adaptations written down in tests/golden/make_golden_batched.py.  The deterministic VAD
detector of tests/stub_vad.py runs on both sides, so both cut the same chunks."""
import copy
import dataclasses
import json
import os
import re

import numpy as np
import pytest
import torch

from oracle.engine import OracleWhisper
from oracle.mel import OracleFeatureExtractor
from tests import stub_vad
from tests.golden.make_golden_batched import GAPPED_75, SCENARIOS, info_to_json
from tests.golden.make_golden_transcribe import make_audio
from whisperlive_b200.config import dims_for
from whisperlive_b200.tokenizer import build_synthetic_tokenizer
from whisperlive_b200.transcriber import BatchedInferencePipeline, B200WhisperModel
from whisperlive_b200.weights import random_init

GOLD = os.path.join(os.path.dirname(__file__), "golden", "batched_reference.json")


def _pipeline(model_name, seed):
    dims = dims_for(model_name)
    eng = OracleWhisper(random_init(dims, seed=seed), dims)
    m = B200WhisperModel(model_name, engine=eng, hf_tokenizer=build_synthetic_tokenizer(dims.vocab),
                         feature_extractor=OracleFeatureExtractor(dims.n_mels), vad=stub_vad)
    return BatchedInferencePipeline(m)


def _segments_json(segs):
    out = []
    for s in segs:
        d = dataclasses.asdict(s)
        for k in ("start", "end", "avg_logprob", "compression_ratio", "no_speech_prob"):
            d[k] = float(d[k])
        for w in d["words"] or []:
            for k in ("start", "end", "probability"):
                w[k] = float(w[k])
        out.append(d)
    return out


def _check_segments(got, gold):
    assert len(got) == len(gold)
    for s, g in zip(got, gold):
        assert (s["id"], s["seek"], s["tokens"], s["text"], s["temperature"]) == \
               (g["id"], g["seek"], g["tokens"], g["text"], g["temperature"])
        for k in ("start", "end", "avg_logprob", "compression_ratio", "no_speech_prob"):
            assert s[k] == pytest.approx(g[k], abs=1e-6), k
        if g["words"] is None:
            assert s["words"] is None
            continue
        assert [(w["word"], w["start"], w["end"]) for w in s["words"]] == [(w["word"], w["start"], w["end"]) for w in g["words"]]
        for w, gw in zip(s["words"], g["words"]):
            assert w["probability"] == pytest.approx(gw["probability"], abs=1e-6)


@pytest.fixture(autouse=True)
def _threads():
    torch.set_num_threads(8)


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_pipeline_matches_reference(name):
    gold = json.load(open(GOLD))[name]
    sc = SCENARIOS[name]
    pipe = _pipeline(sc["model"], sc["seed"])
    audio = make_audio(sc["audio"])
    kw = copy.deepcopy(sc["kw"])
    if "raises" in gold:
        with pytest.raises({"RuntimeError": RuntimeError, "ValueError": ValueError}[gold["raises"]],
                           match=re.escape(gold["message"])):
            segs, _info = pipe.transcribe(audio, **kw)
            list(segs)
        return
    segs, info = pipe.transcribe(audio, **kw)
    got_info = info_to_json(info)        # before the generator runs: the info object is complete up front
    _check_segments(_segments_json(list(segs)), gold["segments"])
    for k in ("language", "duration", "duration_after_vad", "transcription_options", "vad_options"):
        assert got_info[k] == gold["info"][k], k
    assert got_info["language_probability"] == pytest.approx(gold["info"]["language_probability"], abs=1e-6)
    if gold["info"]["all_language_probs"] is None:
        assert got_info["all_language_probs"] is None
    else:
        assert [k for k, _ in got_info["all_language_probs"]] == [k for k, _ in gold["info"]["all_language_probs"]]
        np.testing.assert_allclose([p for _, p in got_info["all_language_probs"]],
                                   [p for _, p in gold["info"]["all_language_probs"]], atol=1e-6)


def test_golden_scenarios_cover_the_chunking_they_name():
    gold = json.load(open(GOLD))
    chunks = lambda n: len({s["seek"] for s in gold[n]["segments"]})
    assert chunks("vad_groups_of_two") >= 3 and chunks("words_across_groups") >= 3
    assert chunks("batch_larger_than_chunks") < SCENARIOS["batch_larger_than_chunks"]["kw"]["batch_size"]
    assert gold["all_silence"]["segments"] == [] and gold["all_silence"]["info"]["duration_after_vad"] == 0
    assert any(w for s in gold["words_across_groups"]["segments"] for w in (s["words"] or []))
    assert gold["long_no_vad_raises"]["raises"] == "RuntimeError" and gold["prompt_too_long_raises"]["raises"] == "ValueError"


@pytest.mark.parametrize("kw", [dict(word_timestamps=True), dict(without_timestamps=False)])
def test_batch_size_does_not_change_the_output(kw):
    """Chunks are decoded independently and the word-timestamp carry-over runs through them in order, so grouping 1, 2
    or 8 chunks per decode gives the same segments and words."""
    audio = make_audio(GAPPED_75)
    outs = []
    for bs in (1, 2, 8):
        pipe = _pipeline("micro.en", 1)
        segs, _info = pipe.transcribe(audio, batch_size=bs, max_new_tokens=16, **kw)
        outs.append(_segments_json(list(segs)))
        sizes = [len(g) for g in pipe.group_steps]
        assert all(n == bs for n in sizes[:-1]) and 0 < sizes[-1] <= bs and sum(sizes) >= 3
    assert outs[0] == outs[1] == outs[2]


def test_segment_ids_continue_across_groups_and_groups_decode_lazily():
    pipe = _pipeline("micro.en", 0)
    segs, _info = pipe.transcribe(make_audio(GAPPED_75), batch_size=1, max_new_tokens=8)
    first = next(segs)
    assert first.id == 1 and len(pipe.group_steps) == 1          # only the first group has been decoded
    rest = list(segs)
    assert len(pipe.group_steps) >= 3
    assert [s.id for s in [first] + rest] == list(range(1, len(rest) + 2))


@pytest.mark.parametrize("option,value", [("repetition_penalty", 1.2), ("no_repeat_ngram_size", 3)])
def test_rejected_options_raise_naming_the_option(option, value):
    pipe = _pipeline("micro.en", 0)
    with pytest.raises(NotImplementedError, match=option):
        pipe.transcribe(make_audio(GAPPED_75), **{option: value})


def test_all_silence_yields_nothing_with_info():
    pipe = _pipeline("micro", 0)
    segs, info = pipe.transcribe(np.zeros(16000 * 12, dtype=np.float32), language="de")
    assert list(segs) == [] and info.duration_after_vad == 0 and info.duration == 12 and info.language == "de"


# --------------------------------------------------------------------------------------- on the device (H100)
GAPPED_150 = ("gapped", (14.0, 2.0, 12.0, 3.0, 9.0, 1.5, 13.0, 2.5, 11.0, 2.0, 10.0, 3.0, 12.0, 1.5, 14.0, 2.0, 9.0, 2.5,
                         11.0, 2.0, 12.0), 61)


def _device_and_oracle(name, seed=0, **engine_kw):
    from tests.test_gpu_parity import engine
    from whisperlive_b200.engine import B200Whisper
    from whisperlive_b200.feature_extractor import FeatureExtractor
    if "enc_slots" in engine_kw:                  # the shared engines of test_gpu_parity keep the default pool
        dims = dims_for(name)
        w = random_init(dims, seed=seed)
        eng, orc = B200Whisper(dims, w, max_beam=5, **engine_kw), OracleWhisper(w, dims)
    else:
        eng, orc = engine(name, seed=seed, **engine_kw)
    dims = eng.dims
    hf = build_synthetic_tokenizer(dims.vocab)
    gpu = B200WhisperModel(name, engine=eng, hf_tokenizer=hf, feature_extractor=FeatureExtractor(eng, dims.n_mels), vad=stub_vad)
    cpu = B200WhisperModel(name, engine=orc, hf_tokenizer=hf, feature_extractor=OracleFeatureExtractor(dims.n_mels), vad=stub_vad)
    return eng, orc, BatchedInferencePipeline(gpu), BatchedInferencePipeline(cpu)


def _by_chunk(segs):
    out = {}
    for s in segs:
        out.setdefault(s.seek, []).append(s)
    return out


def _explain_chunk(eng, orc, pipe, audio, info, seek, kw, what):
    """Decode the chunk at ``seek`` on both engines from the SAME (oracle) features with the pipeline's prompt and
    generate arguments; a differing hypothesis must be an explained near-tie (test_gpu_parity._compare_generation)."""
    from oracle import mel as omel
    from tests.test_gpu_parity import _compare_generation
    from whisperlive_b200 import vad as wvad
    from whisperlive_b200.tokenizer import Tokenizer
    o = info.transcription_options
    chunks, meta = wvad.collect_chunks(audio, o.clip_timestamps, max_duration=30)
    k = next(i for i, md in enumerate(meta) if int(md["offset"] * 100) == seek)
    feats = omel.pad_or_trim(omel.log_mel(chunks[k], eng.dims.n_mels)[:, :-1])[None]
    tok = Tokenizer(pipe.model.hf_tokenizer, eng.dims.multilingual, task="transcribe", language=info.language)
    prompt = pipe.model.get_prompt(tok, [], without_timestamps=o.without_timestamps)
    gkw = dict(beam_size=o.beam_size, patience=o.patience, length_penalty=o.length_penalty,
               max_length=len(prompt) + kw["max_new_tokens"], suppress_blank=o.suppress_blank,
               suppress_tokens=list(o.suppress_tokens), return_scores=True, return_no_speech_prob=True)
    enc, oenc = eng.encode(feats), orc.encode(feats)
    got, ref = eng.generate(enc, [prompt], **gkw), orc.generate(oenc, [prompt], **gkw)
    _compare_generation(got, ref, what, orc, oenc, [prompt], gkw, eng=eng, enc=enc)
    enc.release()


def _compare_pipelines(eng, orc, pipe, audio, got, ref, info, kw, what):
    """Chunk by chunk: identical tokens (times equal, word times within ALIGN_MAX_SHIFT frames), or an explained
    divergence of that chunk's hypothesis."""
    from tests.test_gpu_parity import ALIGN_MAX_SHIFT
    g, r = _by_chunk(got), _by_chunk(ref)
    assert sorted(g) == sorted(r) and len(g) >= 3
    same = 0
    for seek in sorted(r):
        gs, rs = g[seek], r[seek]
        if [s.tokens for s in gs] != [s.tokens for s in rs]:
            print(f"{what}: chunk at seek {seek} differs: {gs[0].tokens[:8]} vs {rs[0].tokens[:8]}")
            _explain_chunk(eng, orc, pipe, audio, info, seek, kw, f"{what} chunk {seek}")
            assert gs[0].avg_logprob == pytest.approx(rs[0].avg_logprob, abs=0.3)
            continue
        same += 1
        for a, b in zip(gs, rs):
            assert a.avg_logprob == pytest.approx(b.avg_logprob, abs=0.05)
            if a.words is None:
                assert (a.start, a.end) == (b.start, b.end)
                continue
            assert [w.word for w in a.words] == [w.word for w in b.words]
            for wa, wb in zip(a.words, b.words):
                assert abs(wa.start - wb.start) <= ALIGN_MAX_SHIFT * 0.02 + 0.011, (seek, wa, wb)
                assert abs(wa.end - wb.end) <= ALIGN_MAX_SHIFT * 0.02 + 0.011, (seek, wa, wb)
    print(f"{what}: {len(r)} chunks, {same} identical")
    return same


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny.en", "micro"])
def test_device_pipeline_matches_oracle_pipeline(name):
    """2.5 min of gapped speech, word timestamps, 4 chunks per group: the device pipeline (wl_mel, wl_encode_windows,
    wl_generate, wl_align) against the same pipeline over the oracle engine."""
    eng, orc, gpu, cpu = _device_and_oracle(name, max_streams=4)
    audio = make_audio(GAPPED_150)
    kw = dict(batch_size=8, max_new_tokens=24, word_timestamps=True, language="en")
    segs, info = gpu.transcribe(audio, **kw)
    got = list(segs)
    rsegs, rinfo = cpu.transcribe(audio, **kw)
    ref = list(rsegs)
    assert info.transcription_options.clip_timestamps == rinfo.transcription_options.clip_timestamps
    assert [len(g) for g in gpu.group_steps][0] == 4          # groups of min(batch_size, max_streams)
    _compare_pipelines(eng, orc, gpu, audio, got, ref, info, kw, name)


@pytest.mark.gpu
def test_device_pipeline_more_chunks_than_streams_and_slots():
    """6 chunks on an engine with 2 streams and 2 encoder slots, one slot held by an encoder output outside the
    pipeline: each group of 2 is encoded in two rounds, three groups run, every slot is free afterwards -- and
    batch_size 1 (a different decoder row count per call) gives the hypotheses of batch_size 2, or explained ones."""
    import gc
    eng, orc, gpu, _cpu = _device_and_oracle("micro.en", seed=0, max_streams=2, enc_slots=2)
    audio = make_audio(GAPPED_150)
    kw = dict(max_new_tokens=24, word_timestamps=True)
    held = eng.encode(np.zeros((1, eng.dims.n_mels, 3000), dtype=np.float32))
    assert eng.free_slots() == 1
    a = list(gpu.transcribe(audio, batch_size=2, **kw)[0])
    steps2 = gpu.group_steps
    held.release()
    segs, info = gpu.transcribe(audio, batch_size=1, **kw)
    b = list(segs)
    assert sum(len(g) for g in steps2) >= 5 and max(len(g) for g in steps2) == 2 and len(gpu.group_steps) >= 5
    ga, gb = _by_chunk(a), _by_chunk(b)
    assert sorted(ga) == sorted(gb)
    for seek in ga:
        if [s.tokens for s in ga[seek]] != [s.tokens for s in gb[seek]]:
            print(f"batch 2 vs 1: chunk {seek} differs")
            _explain_chunk(eng, orc, gpu, audio, info, seek, kw, f"batch 1 chunk {seek}")
            assert ga[seek][0].avg_logprob == pytest.approx(gb[seek][0].avg_logprob, abs=0.3)
        else:
            assert [(s.start, s.end) for s in ga[seek]] == [(s.start, s.end) for s in gb[seek]]
    gc.collect()
    assert eng.free_slots() == eng.enc_slots


@pytest.mark.gpu
def test_device_pipeline_resident_and_host_features_agree():
    eng, _orc, gpu, _cpu = _device_and_oracle("micro.en", seed=0, max_streams=4)
    audio = make_audio(GAPPED_75)                                   # 3 chunks: they fit one resident mel call
    kw = dict(batch_size=2, max_new_tokens=24, word_timestamps=True)
    resident = _segments_json(list(gpu.transcribe(audio, **kw)[0]))
    gpu.resident_features = False
    host = _segments_json(list(gpu.transcribe(audio, **kw)[0]))
    gpu.resident_features = True
    assert resident == host
    # features replaced by a later mel call while the generator is held are computed again
    segs, _info = gpu.transcribe(audio, **kw)
    first = next(segs)
    eng.mel_device([audio[:16000]])
    assert _segments_json([first] + list(segs)) == resident


@pytest.mark.gpu
def test_device_pipeline_between_step_rounds_leaves_the_session_alone():
    """A pipeline call (one-shot encode / generate / align on the same engine) between two step_rounds of an open
    TranscribeSession: the session's streams get the segments of an undisturbed run."""
    from whisperlive_b200 import synth
    eng, _orc, gpu, _cpu = _device_and_oracle("micro.en", seed=0, max_streams=4)
    m = gpu.model
    audios = [synth.speech_like(d, seed=80 + i) for i, d in enumerate((33.0, 8.0, 14.0))]
    kws = [dict(temperature=[0.0], beam_size=5, log_prob_threshold=None, compression_ratio_threshold=None,
                word_timestamps=(i == 2)) for i in range(3)]

    def run(interrupt):
        sess = m.open_session()
        handles = sess.add_streams(audios, [dict(k) for k in kws])
        results, rounds, piped = {}, 0, None
        while sess.pending():
            sess.step_round(max_steps=5)
            rounds += 1
            if interrupt and rounds == 2:
                piped = list(gpu.transcribe(make_audio(GAPPED_75), batch_size=4, max_new_tokens=24,
                                            word_timestamps=True)[0])
            for e in sess.pop_finished():
                results[e.handle] = sess.result_of(e)
            assert rounds < 500
        sess.close()
        return [results[h][0] for h in handles], piped

    base, _ = run(False)
    got, piped = run(True)
    assert piped and len(piped) > 0
    for a, b in zip(got, base):
        assert [s.tokens for s in a] == [s.tokens for s in b]
        assert [(s.start, s.end) for s in a] == [(s.start, s.end) for s in b]
        assert [[(w.word, w.start, w.end) for w in s.words or []] for s in a] == \
               [[(w.word, w.start, w.end) for w in s.words or []] for s in b]
