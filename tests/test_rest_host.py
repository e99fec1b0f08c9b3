"""The reference's REST route served by the resident model's scheduler (``whisperlive_b200.rest.install``), on the CPU
oracle engine: every response body equals the one the reference's own route gives over the oracle engine
(tests/golden/rest_reference.json, tests/golden/make_golden_rest.py), and the upload is one request of the running
scheduler -- admitted beside live streams, cancelled when its SSE client leaves, failing alone."""
import asyncio
import json
import threading
import time

import httpx
import numpy as np
import pytest
import torch

from tests import rest_app

pytestmark = pytest.mark.skipif(not rest_app.reference_present(), reason="reference tree not present")

MODEL_SEED, SPK_SEED = 5, 0     # as tests/golden/make_golden_rest.py


def _oracle_model():
    from oracle.engine import OracleWhisper
    from oracle.mel import OracleFeatureExtractor
    from tests import spk_oracle
    from whisperlive_b200 import speaker
    from whisperlive_b200.config import dims_for
    from whisperlive_b200.tokenizer import build_synthetic_tokenizer
    from whisperlive_b200.transcriber import B200WhisperModel
    from whisperlive_b200.weights import random_init
    dims = dims_for("micro")
    model = B200WhisperModel("micro", engine=OracleWhisper(random_init(dims, seed=MODEL_SEED), dims),
                             hf_tokenizer=build_synthetic_tokenizer(dims.vocab),
                             feature_extractor=OracleFeatureExtractor(dims.n_mels))
    w = speaker.random_weights(SPK_SEED)
    model.speaker_embeddings = lambda audios: np.stack([spk_oracle.embed(a, w) for a in audios]).astype(np.float32)
    return model


@pytest.fixture(scope="module")
def served():
    """The reference app with ``install()``; models come from the registry, built by ``MODEL_FACTORY``."""
    torch.set_num_threads(8)
    server = rest_app.server_module()
    import whisper_live.diarization as diarization
    from whisperlive_b200 import rest
    from whisperlive_b200.backend import ServeClientB200
    saved = (server.WhisperModel, diarization.SpeakerDiarizer, diarization.load_audio,
             server.TranscriptionServer.__dict__["_speaker_labels_for_segments"])
    rest.install(server)
    models = []

    def factory(name):
        models.append(_oracle_model())
        return models[-1]
    ServeClientB200.MODEL_FACTORY = factory
    from starlette.testclient import TestClient
    app = rest_app.build_app(server)
    try:
        yield dict(client=TestClient(app), app=app, registry=ServeClientB200.model_registry(), models=models,
                   ref_labels=saved[3].__func__, ref_diarizer=saved[1])
    finally:
        ServeClientB200.shutdown()
        ServeClientB200.MODEL_FACTORY = None
        server.WhisperModel, diarization.SpeakerDiarizer, diarization.load_audio = saved[:3]
        server.TranscriptionServer._speaker_labels_for_segments = saved[3]


def _entry(served):
    return served["registry"].entries()["small"]


@pytest.mark.parametrize("case", list(rest_app.cases()))
def test_bodies_equal_the_reference_route(served, case):
    before = {k: e.connections for k, e in served["registry"].entries().items()}
    got = rest_app.post(served["client"], case)
    assert got == rest_app.load_golden()[case]
    after = {k: e.connections for k, e in served["registry"].entries().items()}
    assert after == {k: before.get(k, 0) for k in after}          # the registry connection is back


def test_sampling_rung_answers_well_formed(served):
    r = served["client"].post("/v1/audio/transcriptions", data={"response_format": "verbose_json", "temperature": "0.7"},
                              files=[("file", ("a.wav", rest_app.wav_bytes(rest_app.audios()["jfk"]), "audio/wav"))])
    assert r.status_code == 200
    body = r.json()
    assert set(body) == {"task", "language", "duration", "text", "segments"} and body["duration"] == 11.0
    assert body["segments"] and all(s["temperature"] == 0.7 for s in body["segments"])
    assert body["text"] == " ".join(s["text"] for s in body["segments"])


def test_unsupported_container_fails_alone(served):
    got = rest_app.post(served["client"], "json", pcm=b"ID3\x04" + bytes(64), filename="a.mp3")
    assert got["status"] == 500 and "unsupported container" in json.loads(got["body"])["error"]
    assert rest_app.post(served["client"], "json") == rest_app.load_golden()["json"]     # the scheduler still serves


class _Live:
    """A live connection's chunk, as ServeClientB200 submits it, with a short decode for the CPU oracle."""

    def __new__(cls, audio):
        from whisperlive_b200.scheduler import BatchRequest

        class Req(BatchRequest):
            def kwargs(self):
                return dict(super().kwargs(), temperature=[0.0], log_prob_threshold=None, max_new_tokens=24)
        return Req(audio=audio, use_vad=False, language="en")


def _live_results(sch, waves):
    reqs = [_Live(w) for w in waves]
    for r in reqs:
        sch.submit(r)
    return reqs


def test_upload_joins_the_running_session_beside_live_streams(served):
    from whisperlive_b200 import synth
    client = served["client"]
    rest_app.post(client, "json")                                  # the model is resident
    sch = _entry(served).scheduler
    waves = [synth.speech_like(40.0, seed=60 + i) for i in range(2)]
    alone = _live_results(sch, waves)
    assert all(r.future.wait(300) for r in alone)
    mid = sch.admitted_mid_flight
    live = _live_results(sch, waves)
    deadline = time.monotonic() + 60
    while sch.rounds_run == 0 or not any(r.admitted.is_set() for r in live):
        assert time.monotonic() < deadline
        time.sleep(0.01)
    admitted_at = {}
    orig_submit = sch.submit

    def submit(r):                                                 # the upload's own request: when was it admitted
        orig_submit(r)
        threading.Thread(target=lambda: admitted_at.setdefault("t", r.admitted.wait(300) and time.monotonic())).start()
    sch.submit = submit
    try:
        got = rest_app.post(client, "multi_window")
    finally:
        sch.submit = orig_submit
    assert all(r.future.wait(300) for r in live)
    assert got == rest_app.load_golden()["multi_window"]
    assert sch.admitted_mid_flight > mid
    assert admitted_at["t"] < min(r.finished_at for r in live)     # admitted while the live streams were decoding
    for a, b in zip(alone, live):
        assert a.error is None and b.error is None
        assert [(s.tokens, s.start, s.end) for s in a.result] == [(s.tokens, s.start, s.end) for s in b.result]


def test_sse_client_that_leaves_cancels_its_request(served):
    """The client reads the first event and disconnects: the upload's request is cancelled at the next round boundary
    and its session index is free again."""
    from whisperlive_b200.scheduler import RequestCancelled
    client = served["client"]
    rest_app.post(client, "json")
    sch = _entry(served).scheduler
    submitted = []
    orig_submit = sch.submit
    sch.submit = lambda r: (submitted.append(r), orig_submit(r))[1]
    upload, fields, _refs = rest_app.cases()["stream_words"]
    req = httpx.Request("POST", "http://testserver/v1/audio/transcriptions", data=fields,
                        files=[("file", ("a.wav", rest_app.wav_bytes(rest_app.audios()[upload]), "audio/wav"))])
    body = req.read()
    scope = {"type": "http", "asgi": {"version": "3.0", "spec_version": "2.3"}, "http_version": "1.1", "method": "POST",
             "scheme": "http", "path": "/v1/audio/transcriptions", "raw_path": b"/v1/audio/transcriptions",
             "query_string": b"", "root_path": "", "server": ("testserver", 80), "client": ("127.0.0.1", 1234),
             "headers": [(k.lower().encode(), v.encode()) for k, v in req.headers.items()]}
    events = []

    async def run():
        first = asyncio.Event()
        sent = False

        async def receive():
            nonlocal sent
            if not sent:
                sent = True
                return {"type": "http.request", "body": body, "more_body": False}
            await first.wait()
            return {"type": "http.disconnect"}

        async def send(message):
            if message["type"] == "http.response.body" and message.get("body"):
                events.append(message["body"])
                first.set()
                await asyncio.sleep(0)
        await served["app"](scope, receive, send)
    try:
        asyncio.run(run())
    finally:
        sch.submit = orig_submit
    assert len(events) == 1 and events[0].startswith(b"data: {")
    assert len(submitted) == 1
    r = submitted[0]
    assert r.future.wait(60) and isinstance(r.error, RequestCancelled)
    assert _entry(served).connections == 0
    assert rest_app.post(client, "json") == rest_app.load_golden()["json"]


def test_labels_match_the_reference_matching_in_one_embedding_call(served):
    """The batched labels against the reference's one-at-a-time loop on the same vectors: enrolled speakers, new
    speakers, the ``max_speakers`` cap and the 0.3 s rule; the enrolments and all segments take one embedding call."""
    import whisper_live.diarization as diarization
    from types import SimpleNamespace
    rng = np.random.default_rng(3)
    centres = rng.standard_normal((5, 256))
    n = 30
    vecs = [(centres[rng.integers(5)] + 0.4 * rng.standard_normal(256)) for _ in range(n + 2)]
    vecs = [v / np.linalg.norm(v) for v in vecs]
    audio = np.zeros(16000 * (n + 1), np.float32)
    segs = [SimpleNamespace(start=i + (0.8 if i == 7 else 0.0), end=i + 1.0) for i in range(n)]   # segment 7: 0.2 s
    for max_speakers in (10, 3):
        ref = served["ref_diarizer"](max_speakers=max_speakers, speaker_names=["alice", "bob", "carol"])
        feed = iter(vecs[:2] + [v for i, v in enumerate(vecs[2:]) if i != 7])
        ref._load_model = lambda: None
        ref._model = lambda wf: next(feed)
        assert ref.enroll_speaker("alice", audio[:8000]) and ref.enroll_speaker("bob", audio[:8000])
        want = served["ref_labels"](segs, audio, ref)

        calls = []

        class Fixed(diarization.SpeakerDiarizer):
            def _embed(self, audios):
                calls.append(len(audios))
                return [v for v in (vecs[:2] + [v for i, v in enumerate(vecs[2:]) if i != 7])[:len(audios)]]
        dev = Fixed(max_speakers=max_speakers, speaker_names=["alice", "bob", "carol"])
        assert dev.enroll_speaker("alice", audio[:8000]) and dev.enroll_speaker("bob", audio[:8000])
        from whisperlive_b200.rest import speaker_labels_for_segments
        got = speaker_labels_for_segments(segs, audio, dev)
        assert got == want and calls == [2 + n - 1]
        assert len(set(want.values())) > 2 and 7 not in want
