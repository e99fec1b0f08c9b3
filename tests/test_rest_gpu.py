"""The REST route's model on the device: ``rest.ScheduledWhisperModel`` served by a ``RoundScheduler`` over the CUDA
engine gives the segments of the same model over the CPU oracle engine (tests/test_rest_host.py pins the oracle side
against the reference's route), the file's speaker embeddings take one ``wl_spk_embed`` call, and an upload cancelled
mid-file leaves the live streams' results unchanged."""
import numpy as np
import pytest

from tests.test_gpu_parity import ALIGN_MAX_SHIFT, _compare_transcripts, engine
from whisperlive_b200 import synth

pytestmark = pytest.mark.gpu


def _models(name):
    from oracle.mel import OracleFeatureExtractor
    from whisperlive_b200.feature_extractor import FeatureExtractor
    from whisperlive_b200.tokenizer import build_synthetic_tokenizer
    from whisperlive_b200.transcriber import B200WhisperModel
    eng, orc = engine(name, seed=0)
    hf = build_synthetic_tokenizer(eng.dims.vocab)
    gpu = B200WhisperModel(name, engine=eng, hf_tokenizer=hf, feature_extractor=FeatureExtractor(eng, eng.dims.n_mels))
    cpu = B200WhisperModel(name, engine=orc, hf_tokenizer=hf, feature_extractor=OracleFeatureExtractor(eng.dims.n_mels))
    return gpu, cpu


def _serve(model):
    from whisperlive_b200.rest import ScheduledWhisperModel
    from whisperlive_b200.scheduler import RoundScheduler
    sch = RoundScheduler(model, max_batch_size=4)
    sch.start()
    return sch, ScheduledWhisperModel("small", scheduler=sch)


def _jfk():
    return np.load("tests/golden/jfk_16k_i16.npy").astype(np.float32) / 32768.0


def _upload():
    return np.concatenate([_jfk(), synth.speech_like(52.0, seed=21)]).astype(np.float32)


@pytest.mark.parametrize("name", ["tiny"])
@pytest.mark.parametrize("kw", [dict(), dict(word_timestamps=True, language="en", initial_prompt="hello there")])
def test_scheduled_model_matches_the_oracle_engine(name, kw):
    gpu, cpu = _models(name)
    # one window: in later windows random weights decode long repetitive hypotheses whose near-ties compound through
    # the previous-text prompt beyond what _compare_transcripts can explain
    audio = _jfk()
    got, ref = [], []
    for model, out in ((gpu, got), (cpu, ref)):
        sch, m = _serve(model)
        try:
            segments, info = m.transcribe(audio, **kw)
            out.append((list(segments), info))
        finally:
            sch.stop()
    if not kw.get("word_timestamps"):
        _compare_transcripts(got, ref)
        return
    # a DTW jump moves by up to ALIGN_MAX_SHIFT frames; word durations are differences of two jumps, and the reference's
    # long-word rule clips ends at twice their median, so a derived time moves by up to 4 x ALIGN_MAX_SHIFT frames
    tol = 4 * ALIGN_MAX_SHIFT * 0.02 + 1e-6
    (gs, gi), (rs, ri) = got[0], ref[0]
    assert gi.language == ri.language and [a.tokens for a in gs] == [b.tokens for b in rs] and gs
    for a, b in zip(gs, rs):
        assert abs(a.start - b.start) <= tol and abs(a.end - b.end) <= tol
        assert [w.word for w in a.words] == [w.word for w in b.words]
        for wa, wb in zip(a.words, b.words):
            assert abs(wa.start - wb.start) <= tol and abs(wa.end - wb.end) <= tol


def test_file_embeddings_take_one_call_and_cancel_leaves_live_streams_alone():
    from whisperlive_b200.scheduler import BatchRequest
    from whisperlive_b200.transcriber import B200WhisperModel
    model = B200WhisperModel("tiny", weights="random", hf_tokenizer="synthetic", max_streams=4)
    sch, m = _serve(model)
    try:
        segs = [synth.speech_like(1.0 + 0.5 * i, seed=90 + i) for i in range(12)]
        before = sch.embedding_calls
        out = [r.wait(60) for r in sch.embed_many(segs)]
        assert sch.embedding_calls == before + 1 and all(v.shape == (256,) for v in out)

        class Req(BatchRequest):
            def kwargs(self):
                return dict(super().kwargs(), temperature=[0.0], log_prob_threshold=None)
        waves = [synth.speech_like(20.0 + 5 * i, seed=70 + i) for i in range(2)]

        def live():
            reqs = [Req(audio=w, use_vad=False, language="en") for w in waves]
            for r in reqs:
                sch.submit(r)
            return reqs
        alone = live()
        assert all(r.future.wait(120) for r in alone)
        segments, _info = m.transcribe(_upload())
        beside = live()
        next(segments, None)
        segments.close()                                           # the SSE client went away
        assert all(r.future.wait(120) for r in beside)
        for a, b in zip(alone, beside):
            assert a.error is None and b.error is None
            assert [(s.tokens, s.start, s.end) for s in a.result] == [(s.tokens, s.start, s.end) for s in b.result]
    finally:
        sch.stop()


def test_speaker_decisions_match_the_oracle_embeddings():
    """The embeddings the REST diarizer asks for (two enrolled references and every segment of a multi-window upload,
    one ``embed_many`` batch) on the device against tests/spk_oracle.py with the same weights: every similarity within
    the measured error, and the reference's first decision -- best enrolled speaker, and whether it clears the 0.55
    threshold -- equal wherever it is not within that error of a tie."""
    from tests import spk_oracle
    from whisperlive_b200 import speaker
    from whisperlive_b200.transcriber import B200WhisperModel
    model = B200WhisperModel("tiny", weights="random", hf_tokenizer="synthetic", max_streams=4)
    sch, m = _serve(model)
    try:
        audio = _upload()
        segments, _info = m.transcribe(audio)
        spans = [audio[max(0, int(s.start * 16000)):min(len(audio), int(s.end * 16000))] for s in segments]
        spans = [a for a in spans if len(a) >= 4800]
        refs = [synth.speech_like(3.0, seed=31), synth.speech_like(3.0, seed=32)]
        assert len(spans) >= 2
        before = sch.embedding_calls
        dev = np.stack([r.wait(120) for r in sch.embed_many(refs + spans)]).astype(np.float64)
        assert sch.embedding_calls == before + 1
    finally:
        sch.stop()
    w = speaker.random_weights(0)
    orc = np.stack([spk_oracle.embed(a, w) for a in refs + spans])
    dn = dev / np.linalg.norm(dev, axis=1, keepdims=True)
    on = orc / np.linalg.norm(orc, axis=1, keepdims=True)
    err = float(np.abs(dn @ dn.T - on @ on.T).max())
    print(f"{len(spans)} segments, device similarity error {err:.2e}")
    assert err < 2e-3
    for k in range(2, len(refs) + len(spans)):
        sd, so = dn[k] @ dn[:2].T, on[k] @ on[:2].T
        if abs(so[0] - so[1]) > 2 * err:
            assert int(np.argmax(sd)) == int(np.argmax(so))
        if abs(so.max() - 0.55) > err:
            assert (sd.max() >= 0.55) == (so.max() >= 0.55)
