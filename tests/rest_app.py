"""The reference's own REST app (whisper_live/server.py ``TranscriptionServer.run(enable_rest=True)``), built in process for
the REST tests and tests/golden/make_golden_rest.py: ``uvicorn.run`` hands over the FastAPI app instead of serving it,
the websocket ``serve`` returns at once, and the imports this machine lacks (``faster_whisper``, ``onnxruntime``) are
stubbed while the server module loads.  Needs the reference tree (build container only)."""
import contextlib
import importlib.machinery
import io
import json
import os
import sys
import types
import wave

import numpy as np

REF = "/root/reference"
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
SR = 16000


def reference_present() -> bool:
    return os.path.isdir(os.path.join(REF, "whisper_live"))


def server_module():
    """``whisper_live.server``, imported with stubs for the modules it imports but the REST route does not use."""
    if "whisper_live.server" in sys.modules:
        return sys.modules["whisper_live.server"]
    added = []
    for name in ("faster_whisper", "onnxruntime"):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__spec__ = importlib.machinery.ModuleSpec(name, None)
            sys.modules[name] = m
            added.append(name)
    if not hasattr(sys.modules["faster_whisper"], "WhisperModel"):
        sys.modules["faster_whisper"].WhisperModel = None       # replaced by the caller before any request
    sys.path.insert(0, REF)
    try:
        import whisper_live.server as server
    finally:
        sys.path.remove(REF)
        for name in added:                                      # other tests must not see the stubs
            del sys.modules[name]
    return server


def build_app(server, **run_kwargs):
    """The FastAPI app ``TranscriptionServer.run(enable_rest=True, ...)`` builds."""
    captured = {}

    class _Uvicorn:
        @staticmethod
        def run(app, **kw):
            captured["app"] = app

    class _Serve:
        def serve_forever(self):
            pass

    @contextlib.contextmanager
    def _serve(*a, **k):
        yield _Serve()

    saved = server.uvicorn, server.serve
    server.uvicorn, server.serve = _Uvicorn, _serve
    try:
        server.TranscriptionServer().run("127.0.0.1", backend="faster_whisper", enable_rest=True, **run_kwargs)
    finally:
        server.uvicorn, server.serve = saved
    return captured["app"]


# ------------------------------------------------------------------ inputs (both sides)
def wav_bytes(pcm: np.ndarray) -> bytes:
    """16-bit mono 16 kHz WAV of float PCM in [-1, 1)."""
    buf = io.BytesIO()
    with wave.open(buf, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(SR)
        w.writeframes(np.clip(np.round(pcm * 32768.0), -32768, 32767).astype("<i2").tobytes())
    return buf.getvalue()


def read_wav(path) -> np.ndarray:
    """Mono float32 of a 16-bit 16 kHz WAV, as PyAV's ``flt`` resampler gives it for that input."""
    with wave.open(path if isinstance(path, str) else io.BytesIO(path), "rb") as w:
        assert w.getsampwidth() == 2 and w.getframerate() == SR and w.getnchannels() == 1
        raw = w.readframes(w.getnframes())
    return (np.frombuffer(raw, dtype="<i2").astype(np.float64) / 32768.0).astype(np.float32)


def audios():
    """name -> PCM of the uploads the REST cases send."""
    from whisperlive_b200 import synth
    jfk = np.load(os.path.join(ROOT, "tests", "golden", "jfk_16k_i16.npy")).astype(np.float32) / 32768.0
    return {
        "jfk": jfk,
        "long": np.concatenate([jfk, synth.speech_like(52.0, seed=21)]).astype(np.float32),   # 63 s: three windows
        "alice": synth.speech_like(3.0, seed=31),
        "bob": synth.speech_like(3.0, seed=32),
        "conversation": np.concatenate([synth.speech_like(9.0, seed=31), synth.silence(1.0),
                                        synth.speech_like(9.0, seed=33), synth.silence(1.0),
                                        synth.speech_like(9.0, seed=32)]).astype(np.float32),
    }


def cases():
    """name -> (upload, form fields, known speaker reference uploads)."""
    out = {}
    for fmt in ("json", "text", "srt", "vtt", "verbose_json"):
        out[fmt] = ("jfk", {"response_format": fmt}, [])
        out[fmt + "_words"] = ("jfk", {"response_format": fmt, "timestamp_granularities": ["word"]}, [])
    out["language_prompt_hotwords"] = ("jfk", {"response_format": "verbose_json", "language": "en",
                                               "prompt": "The president said", "hotwords": "country"}, [])
    out["multi_window"] = ("long", {"response_format": "verbose_json"}, [])
    out["stream"] = ("jfk", {"stream": "true"}, [])
    out["stream_words"] = ("long", {"stream": "true", "timestamp_granularities": ["word"]}, [])
    out["known_speakers"] = ("conversation", {"response_format": "verbose_json",
                                              "known_speaker_names": ["alice", "bob"]}, ["alice", "bob"])
    out["bad_format"] = ("jfk", {"response_format": "xml"}, [])
    out["mismatched_speakers"] = ("jfk", {"response_format": "verbose_json",
                                          "known_speaker_names": ["alice", "bob"]}, ["alice"])
    return out


def post(client, case, pcm=None, filename="upload.wav"):
    """One request of ``cases()``: ``{"status", "content_type", "body"}`` with the body as text."""
    upload, fields, refs = cases()[case]
    a = audios()
    data = wav_bytes(a[upload]) if pcm is None else pcm
    files = [("file", (filename, data, "audio/wav"))]
    files += [("known_speaker_references", (f"{r}.wav", wav_bytes(a[r]), "audio/wav")) for r in refs]
    r = client.post("/v1/audio/transcriptions", data=fields, files=files)
    return {"status": r.status_code, "content_type": r.headers.get("content-type", "").split(";")[0], "body": r.text}


def load_golden():
    with open(os.path.join(ROOT, "tests", "golden", "rest_reference.json")) as f:
        return json.load(f)
