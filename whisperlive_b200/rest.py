"""The reference's OpenAI-compatible REST route (``POST /v1/audio/transcriptions``, whisper_live/server.py:693-867, and
its streaming variant :490-537) served by the resident model's running decode loop.

The reference builds a fresh ``faster_whisper.WhisperModel`` per request -- a second model beside the resident one --
and, for ``verbose_json`` with known speakers, a pyannote ``SpeakerDiarizer`` that reads audio through PyAV and embeds
the segments one call at a time.  ``install(server_module)`` replaces exactly those model pieces and nothing else; the
route itself (FastAPI, form fields, response shapes, status codes, error texts, API key, rate limit, CORS, metrics)
stays the reference's:

* ``ScheduledWhisperModel``: the ``WhisperModel`` surface the route uses.  ``transcribe`` submits the whole file as ONE
  request to the resident model's ``RoundScheduler``: the file takes one session index beside the live connections'
  chunks, its windows decode one after another inside the running decode loop, and the segments come back window by
  window as they settle.  Closing the segment generator early (an SSE client that went away) cancels the request.
* ``load_audio``: ``audio.decode_audio`` (WAV / FLAC; other containers raise, naming the container).
* the REST diarizer: the reference's ``SpeakerDiarizer`` whose embeddings come from the same scheduler.  Enrolment is
  deferred, and ``speaker_labels_for_segments`` hands the scheduler every enrolled reference and every segment of the
  file at once -- one ``wl_spk_embed`` call at its next round boundary -- then runs the reference's own
  ``identify_speaker`` matching over them in segment order (best match, threshold, running average, new speakers,
  ``max_speakers``), since those updates depend on order.
"""
from __future__ import annotations

import collections
import threading
import weakref
from typing import List, Optional

import numpy as np

from .audio import decode_audio
from .scheduler import BatchRequest

SAMPLING_RATE = 16000
MIN_EMBED_SECONDS = 0.3        # the reference's SpeakerDiarizer embeds nothing shorter (diarization.py:112)


class _Lease:
    """The scheduler of a model as the websocket connections resolve it: the shared ``SINGLE_MODEL`` /
    ``BATCH_WORKER`` when ``single_model`` is on, else one connection of ``ServeClientB200.model_registry()``, held
    until ``release``."""

    def __init__(self, model_size_or_path: str, single_model: bool, scheduler=None):
        self.registry, self.entry = None, None
        self._lock = threading.Lock()
        if scheduler is not None:
            self.scheduler = scheduler
            return
        from .backend import ServeClientB200
        cls = ServeClientB200
        if single_model:
            _model, self.scheduler = cls.shared_model(lambda: cls.build_model(model_size_or_path))
        else:
            self.registry = cls.model_registry()
            self.entry = self.registry.acquire(model_size_or_path)
            self.scheduler = self.entry.scheduler

    def release(self) -> None:
        with self._lock:
            entry, self.entry = self.entry, None
        if entry is not None:
            self.registry.release(entry)


class ScheduledWhisperModel:
    """``faster_whisper.WhisperModel`` as the REST route uses it, served by the resident model's scheduler.
    Construction loads nothing: ``transcribe`` resolves the model as a websocket connection does (``MODEL_FACTORY``
    included).  ``SINGLE_MODEL``: serve from the shared single model (``install(..., single_model=True)``).
    ``scheduler``: serve from this ``RoundScheduler`` instead (tests, and callers that run their own)."""

    SINGLE_MODEL = False

    def __init__(self, model_size_or_path: str, device: str = "cuda", device_index=0, compute_type: str = "float16",
                 scheduler=None, **kwargs):
        self.model_size_or_path = model_size_or_path
        self.scheduler = scheduler

    def transcribe(self, audio, language: Optional[str] = None, initial_prompt=None, temperature=0.0,
                   vad_filter: bool = False, word_timestamps: bool = False, hotwords: Optional[str] = None):
        """``(segments, info)`` as faster-whisper returns them.  Blocks until the file is admitted (its language is
        resolved there); ``segments`` is a generator of each window's segments as they settle.  A float
        ``temperature`` is a one-rung ladder; a rung above 0 samples inside the running decode loop."""
        if not isinstance(audio, np.ndarray):
            audio = decode_audio(audio, sampling_rate=SAMPLING_RATE)
        lease = _Lease(self.model_size_or_path, self.SINGLE_MODEL, self.scheduler)
        try:
            request = BatchRequest(audio=audio, language=language, initial_prompt=initial_prompt, use_vad=bool(vad_filter),
                                   word_timestamps=bool(word_timestamps), hotwords=hotwords, temperature=temperature,
                                   want_segments=True)
            lease.scheduler.submit(request)
            request.admitted.wait()
            if request.error is not None:
                raise request.error
        except BaseException:
            lease.release()
            raise
        segments = _segments(request, lease)
        # a generator that is dropped before its first next() never runs its finally: cancel and release here too
        weakref.finalize(segments, _abandon, request, lease)
        return segments, request.info


def _abandon(request: BatchRequest, lease: _Lease) -> None:
    if not request.future.is_set():
        request.cancel()
    lease.release()


def _segments(request: BatchRequest, lease: _Lease):
    n = 0
    try:
        while not request.future.is_set():
            segs = request.settled.since(n)
            yield from segs
            n += len(segs)
            request.settled.event.wait()
            request.settled.event.clear()
        if request.error is not None:
            raise request.error
        yield from (request.result or [])[n:]
    finally:
        _abandon(request, lease)


def load_audio(file_path, sample_rate: int = SAMPLING_RATE) -> np.ndarray:
    """The reference's ``whisper_live.diarization.load_audio``: mono float32 PCM at ``sample_rate``."""
    return decode_audio(file_path, sampling_rate=sample_rate)


def diarizer_class(base, model_size_or_path: str = "small", single_model: bool = False):
    """The REST diarizer: the reference's ``SpeakerDiarizer`` (``base``) with the embeddings of ``model_size_or_path``'s
    scheduler, batched per request (``speaker_labels_for_segments``)."""

    class RestSpeakerDiarizer(base):
        MODEL = model_size_or_path
        SINGLE_MODEL = single_model

        def __init__(self, *args, **kwargs):
            super().__init__(*args, **kwargs)
            self._enrolled: List[tuple] = []               # (name, audio) not embedded yet, in enrolment order
            self._ready: collections.deque = collections.deque()   # embeddings for the next _compute_embedding calls

        def _load_model(self):
            pass

        def enroll_speaker(self, speaker_name, audio_np, sample_rate=SAMPLING_RATE):
            """Deferred enrolment: the reference audio is embedded with the file's segments, in one call."""
            if len(audio_np) < sample_rate * MIN_EMBED_SECONDS:
                return False
            self._check_rate(sample_rate)
            self._enrolled.append((speaker_name, np.asarray(audio_np, dtype=np.float32).reshape(-1)))
            return True

        def embed_batch(self, audios, sample_rate=SAMPLING_RATE) -> None:
            """Embed the pending enrolments and ``audios`` (those of at least 0.3 s) in one scheduler request; the
            enrolments take their place in ``speakers``, and the next ``_compute_embedding`` calls return the vectors
            of ``audios`` in order (None for the short ones)."""
            self._check_rate(sample_rate)
            enrolled, self._enrolled = self._enrolled, []
            long = [a for a in audios if len(a) >= sample_rate * MIN_EMBED_SECONDS]
            vectors = self._embed([a for _, a in enrolled] + long)
            for (name, _a), v in zip(enrolled, vectors):
                self.speakers[name] = v
            it = iter(vectors[len(enrolled):])
            self._ready.extend(next(it) if len(a) >= sample_rate * MIN_EMBED_SECONDS else None for a in audios)

        def _compute_embedding(self, audio_np, sample_rate=SAMPLING_RATE):
            if not self._ready:
                self.embed_batch([audio_np], sample_rate)
            return self._ready.popleft()

        def identify_speaker(self, audio_np, sample_rate=SAMPLING_RATE):
            if self._enrolled:
                self.embed_batch([], sample_rate)
            return super().identify_speaker(audio_np, sample_rate)

        @staticmethod
        def _check_rate(sample_rate):
            if sample_rate != SAMPLING_RATE:
                raise ValueError(f"the speaker embedding runs at {SAMPLING_RATE} Hz, not {sample_rate}")

        def _embed(self, audios) -> List[np.ndarray]:
            if not audios:
                return []
            lease = _Lease(self.MODEL, self.SINGLE_MODEL)
            try:
                requests = lease.scheduler.embed_many(audios)
                out = [r.wait(timeout=None) for r in requests]
            finally:
                lease.release()
            return [v / np.linalg.norm(v) for v in out]

    return RestSpeakerDiarizer


def speaker_labels_for_segments(segments, audio_np, diarizer, sample_rate=SAMPLING_RATE):
    """The reference's ``TranscriptionServer._speaker_labels_for_segments`` with every segment embedded in one batch
    first (a diarizer without ``embed_batch`` embeds one segment at a time, as the reference does)."""
    if diarizer is None or audio_np is None:
        return {}
    spans = []
    for index, segment in enumerate(segments):
        start = max(0, int(segment.start * sample_rate))
        end = min(len(audio_np), int(segment.end * sample_rate))
        if end > start:
            spans.append((index, audio_np[start:end]))
    if hasattr(diarizer, "embed_batch"):
        diarizer.embed_batch([a for _, a in spans], sample_rate)
    labels = {}
    for index, audio in spans:
        speaker = diarizer.identify_speaker(audio, sample_rate)
        if speaker:
            labels[index] = speaker
    return labels


def install(server_module, model: str = "small", single_model: bool = False) -> None:
    """Serve the REST route of ``server_module`` (``whisper_live.server``) on the device: its ``WhisperModel``,
    ``whisper_live.diarization.SpeakerDiarizer`` / ``load_audio`` and ``TranscriptionServer._speaker_labels_for_segments``.
    ``model``: the model the route serves (``faster_whisper_custom_model_path`` or ``"small"``, as the route picks
    it), whose scheduler embeds the speakers; ``single_model``: resolve models as ``single_model=True`` connections do."""
    import whisper_live.diarization as diarization
    ScheduledWhisperModel.SINGLE_MODEL = bool(single_model)
    server_module.WhisperModel = ScheduledWhisperModel
    base = getattr(diarization.SpeakerDiarizer, "reference_class", diarization.SpeakerDiarizer)
    cls = diarizer_class(base, model, single_model)
    cls.reference_class = base
    diarization.SpeakerDiarizer = cls
    diarization.load_audio = load_audio
    server_module.TranscriptionServer._speaker_labels_for_segments = staticmethod(speaker_labels_for_segments)
