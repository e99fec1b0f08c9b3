"""RoundScheduler: the one thread that owns the GPU engine, fed by the per-client threads.

What the reference has in this place is ``BatchInferenceWorker`` (whisper_live/batch_inference.py:87-438): collect a
batch for a time window, run it to completion, answer, repeat -- so a chunk that arrives 10 ms after a batch started
waits for the whole batch, only the first 30 s window is batched, every fallback rung re-encodes, and hotwords / word
timestamps fall back to the unbatched path.  This scheduler shares only its *request record* with it (``BatchRequest``,
the drop-in schema a client thread fills in and waits on); the control flow is different:

* there is no batch.  A ``TranscribeSession`` (transcriber.py) holds every stream that is in flight; the owner thread
  alternates ``admit`` (everything that is in the inbox RIGHT NOW, up to the stream capacity) and ``round`` (one device
  round for everything in flight: encode the next windows, one generate call per option set, align, post-process);
* a stream is answered the moment its last window settles -- it does not wait for the streams it shared rounds with;
* admission happens between rounds, and a round is at most ``step_tokens`` TOKEN STEPS of the device-side decode loop
  (``TranscribeSession.step_round`` over the engine's decode session, ``wl_session_*``): a late chunk is encoded,
  prefilled and joins the loop of the chunks that are already decoding a few token steps after it arrived, and the index
  of a finished stream is refilled immediately;
* an engine error fails the streams it touched, never the scheduler (``TranscribeSession`` isolates them);
* between step rounds the owner thread publishes interim segments for the requests that want them (one batched peek of
  the decode session) and drops cancelled requests, freeing their decode index and encoder slots;
* speaker-embedding requests (``embed``, the device diarizer's) are answered at every round boundary, all that are
  pending in one ``speaker_embeddings`` call, and right away when nothing is in flight;
* a request that wants its segments window by window (``want_segments``, the REST route's file jobs) gets the segments
  that settled published after every round: host state only, no peek of the decode session.

``linger_ms`` (default 0) optionally waits for more requests when the engine is idle and a single request arrived --
the latency / batching trade the reference hard-codes as its 50 ms window.
"""
from __future__ import annotations

import collections
import logging
import threading
import time
from dataclasses import dataclass, field
from typing import Any, Deque, Dict, List, Optional

import numpy as np

log = logging.getLogger("whisperlive_b200.scheduler")

EMBED_CALL_SAMPLES = 30 * 16000     # per stream of capacity: one 30 s segment each, the first wl_spk_embed workspace


class RequestCancelled(RuntimeError):
    """The error a request's future carries after ``BatchRequest.cancel``."""


class Partial:
    """The latest interim segments of a request that wants them: ``version`` counts publications, ``event`` is set on
    each one and when the request finishes (so a client can wait on it alone)."""

    def __init__(self):
        self._lock = threading.Lock()
        self.segments: List[Any] = []
        self.version = 0
        self.ntok = 0
        self.event = threading.Event()

    def publish(self, segments: List[Any]) -> bool:
        """Store ``segments`` as a new version when their token count differs from the last one's."""
        ntok = sum(len(s.tokens) for s in segments)
        with self._lock:
            if ntok == self.ntok:
                return False
            self.segments, self.ntok, self.version = list(segments), ntok, self.version + 1
        self.event.set()
        return True

    def latest(self):
        """``(version, segments)``"""
        with self._lock:
            return self.version, list(self.segments)


class Settled:
    """The segments of a request's settled windows, appended by the owner thread as windows settle; ``event`` is set on
    each append and when the request finishes."""

    def __init__(self):
        self._lock = threading.Lock()
        self._segments: List[Any] = []
        self.event = threading.Event()

    def __len__(self) -> int:
        with self._lock:
            return len(self._segments)

    def extend(self, segments: List[Any]) -> None:
        with self._lock:
            self._segments.extend(segments)
        self.event.set()

    def since(self, n: int) -> List[Any]:
        """The segments after the first ``n``."""
        with self._lock:
            return self._segments[n:]


@dataclass
class BatchRequest:
    """What a client thread submits and waits on (same fields as the reference's request record,
    whisper_live/batch_inference.py:51-84, so ``ServeClient*`` code can fill either).  ``want_partials``: publish interim
    segments in ``partial`` after each step round; ``cancel()``: nobody waits for the result any more.
    ``temperature``: the ladder (a float is a one-rung ladder); None keeps the transcriber's default.  ``want_segments``:
    append the segments of each window that settles to ``settled``, after the round it settled in.  ``admitted`` is set once the request is in the
    session, with ``info`` (language resolved) -- or once it failed or was cancelled before that."""
    audio: np.ndarray
    language: Optional[str] = None
    task: str = "transcribe"
    initial_prompt: Optional[str] = None
    use_vad: bool = True
    vad_parameters: Optional[Dict] = None
    word_timestamps: bool = False
    client_uid: Optional[str] = None
    hotwords: Optional[str] = None
    future: threading.Event = field(default_factory=threading.Event)
    result: Optional[Any] = None
    info: Optional[Any] = None
    error: Optional[Exception] = None
    submitted_at: float = 0.0
    finished_at: float = 0.0
    want_partials: bool = False
    partial: Partial = field(default_factory=Partial)
    cancelled: bool = False
    temperature: Optional[Any] = None
    want_segments: bool = False
    settled: Settled = field(default_factory=Settled)
    admitted: threading.Event = field(default_factory=threading.Event)

    def cancel(self) -> None:
        """The scheduler drops this request at its next round boundary (its decode index and encoder slots go back) and
        sets its future with ``RequestCancelled``; a request that already finished keeps its result."""
        self.cancelled = True

    def kwargs(self) -> dict:
        kw = dict(language=self.language, task=self.task, initial_prompt=self.initial_prompt, vad_filter=self.use_vad,
                  vad_parameters=self.vad_parameters if self.use_vad else None, hotwords=self.hotwords,
                  word_timestamps=self.word_timestamps)
        if self.temperature is not None:
            kw["temperature"] = self.temperature
        return kw


@dataclass
class FileRequest:
    """One ``BatchedInferencePipeline`` file decoded by the running loop (``BatchedInferencePipeline(model,
    scheduler=...)``): ``run`` holds its speech chunks (``transcriber._ChunkRun``).  Its chunks hold at most
    ``max_share`` of the decode indices, and none is admitted while a live request waits.  ``settled`` receives the
    segments in chunk order as chunks settle; ``future`` is set when the file is done, failed (``error``) or was
    cancelled; ``steps`` holds every chunk's token steps."""
    run: Any
    max_share: float = 0.5
    future: threading.Event = field(default_factory=threading.Event)
    error: Optional[Exception] = None
    cancelled: bool = False
    settled: Settled = field(default_factory=Settled)
    admitted: threading.Event = field(default_factory=threading.Event)
    steps: List[int] = field(default_factory=list)
    submitted_at: float = 0.0
    finished_at: float = 0.0

    def cancel(self) -> None:
        """The scheduler takes the file's chunks out of the loop at its next round boundary."""
        self.cancelled = True


class EmbeddingRequest:
    """A speaker-embedding request (``RoundScheduler.embed``): ``wait()`` returns the [256] float32 vector or raises the
    error of the call that failed it."""

    def __init__(self, audio: np.ndarray):
        self.audio = audio
        self.future = threading.Event()
        self.result: Optional[np.ndarray] = None
        self.error: Optional[Exception] = None

    def wait(self, timeout: Optional[float] = 60.0) -> np.ndarray:
        if not self.future.wait(timeout):
            raise TimeoutError(f"speaker embedding not answered within {timeout} s")
        if self.error is not None:
            raise self.error
        return self.result


class RoundScheduler:
    def __init__(self, transcriber, max_batch_size: int = 8, batch_window_ms: int = 0, linger_ms: Optional[int] = None,
                 step_tokens: Optional[int] = 16):
        """``max_batch_size``: streams in flight at once (the engine's ``max_streams``).  ``batch_window_ms`` is accepted
        for signature compatibility with the reference worker and used as ``linger_ms`` when that is not given.
        ``step_tokens``: token steps per device round (``TranscribeSession.step_round``): the inbox is looked at -- and
        a finished stream answered -- at least that often, and new streams join the decode loop already running;
        ``None`` / 0 = window-level rounds (one ``generate`` call run to completion per round)."""
        self.transcriber = transcriber
        self.step_tokens = int(step_tokens or 0)
        self.capacity = max(1, int(max_batch_size))
        self.linger_s = (batch_window_ms if linger_ms is None else linger_ms) / 1000.0
        self._inbox: Deque[BatchRequest] = collections.deque()
        self._embeds: List[EmbeddingRequest] = []
        self._files: List[FileRequest] = []
        self._cv = threading.Condition()
        self._stop = False
        self._thread: Optional[threading.Thread] = None
        # statistics (tests, metrics)
        self.rounds_run = 0
        self.streams_done = 0
        self.max_in_flight = 0
        self.admitted_mid_flight = 0   # streams that joined while others were already decoding
        self.embedding_calls = 0
        self.files_in_flight = 0       # batched files the owner thread holds (admitted, not yet finished or dropped)
        self.rule_admissions = 0       # streams that joined the decode loop with logits rules of their own

    # ------------------------------------------------------------------ client side
    def submit(self, request) -> None:
        """Queue a ``BatchRequest`` (a live chunk or an upload) or a ``FileRequest`` (a batched file's chunks)."""
        request.submitted_at = time.monotonic()
        with self._cv:
            (self._files if isinstance(request, FileRequest) else self._inbox).append(request)
            self._cv.notify()

    def embed(self, audio: np.ndarray) -> EmbeddingRequest:
        """Queue one segment for a speaker embedding; the owner thread answers it with every other pending one at the
        next round boundary, or at once when the engine is idle."""
        return self.embed_many([audio])[0]

    def embed_many(self, audios) -> List[EmbeddingRequest]:
        """Queue several segments at once: they are answered together, by one ``speaker_embeddings`` call."""
        requests = [EmbeddingRequest(np.asarray(a, dtype=np.float32).reshape(-1)) for a in audios]
        with self._cv:
            self._embeds.extend(requests)
            self._cv.notify()
        return requests

    def start(self) -> None:
        self._thread = threading.Thread(target=self._owner_loop, daemon=True, name="wlb200-rounds")
        self._thread.start()

    def stop(self) -> None:
        with self._cv:
            self._stop = True
            self._cv.notify()
        if self._thread is not None:
            self._thread.join(timeout=10)

    # ------------------------------------------------------------------ owner thread
    def _take(self, room: int, block: bool) -> List[BatchRequest]:
        with self._cv:
            if block:
                while not self._inbox and not self._embeds and not self._files and not self._stop:
                    self._cv.wait(timeout=0.5)
                if self.linger_s > 0 and self._inbox and len(self._inbox) < room and not self._stop:
                    end = time.monotonic() + self.linger_s      # idle engine, first request: optionally wait for company
                    while len(self._inbox) < room and not self._embeds and not self._stop:
                        left = end - time.monotonic()
                        if left <= 0:
                            break
                        self._cv.wait(timeout=left)
            out = []
            while self._inbox and len(out) < room:
                out.append(self._inbox.popleft())
            return out

    def _owner_loop(self) -> None:
        session = self.transcriber.open_session() if hasattr(self.transcriber, "open_session") else _OneShotSession(self.transcriber)
        in_flight: Dict[int, BatchRequest] = {}
        files: Dict[int, FileRequest] = {}
        self._rules_before = 0         # rule admissions of sessions replaced after a failed round
        while True:
            with self._cv:
                if self._stop and not in_flight and not files and not self._inbox and not self._embeds and not self._files:
                    close = getattr(session, "close", None)
                    if close is not None:
                        close()             # hands the engine's decode session back
                    return
            # a file's chunks take indices (and encoder slots) from the same capacity as the live streams
            room = self.capacity - len(in_flight) - (session.file_streams() if files else 0)
            new = self._take(room, block=not in_flight and not files) if room > 0 else []
            self._admit_files(session, files)
            if hasattr(session, "live_waiting"):
                session.live_waiting = len(self._inbox) > 0     # live requests first: no new chunk while one waits
            for r in [r for r in new if r.cancelled]:
                new.remove(r)
                self._finish(r, None, None, RequestCancelled("request cancelled before admission"))
            if new:
                if in_flight:
                    self.admitted_mid_flight += len(new)
                try:
                    handles = session.add_streams([r.audio for r in new], [r.kwargs() for r in new])
                    for h, r in zip(handles, new):
                        in_flight[h] = r
                except Exception as e:      # admission (VAD / mel / language id) failed: only these requests
                    log.error("admission failed: %s", e)
                    for r in new:
                        self._finish(r, None, None, e)
                else:
                    self._announce_admitted(session, zip(handles, new))
            self._answer_embeddings()
            self.max_in_flight = max(self.max_in_flight, len(in_flight))
            self._drop_cancelled(session, in_flight)
            self._drop_cancelled_files(session, files)
            self.files_in_flight = len(files)
            if not in_flight and not files:
                continue
            step = self.step_tokens > 0 and hasattr(session, "step_round")
            try:
                if step:
                    session.step_round(self.step_tokens)
                else:
                    session.round()
                self.rounds_run += 1
            except Exception as e:          # the session isolates per-stream errors; anything else fails what is in flight
                log.error("round failed: %s", e)
                for h, r in list(in_flight.items()):
                    self._finish(r, None, None, e)
                in_flight.clear()
                for r in files.values():
                    self._finish_file(r, e)
                files.clear()
                self.files_in_flight = 0
                self._rules_before += getattr(session, "rule_admissions", 0)
                session = self.transcriber.open_session() if hasattr(self.transcriber, "open_session") else _OneShotSession(self.transcriber)
                continue
            for entry in session.pop_finished():
                r = in_flight.pop(entry.handle, None)
                if r is None:
                    continue
                try:
                    segments, info = session.result_of(entry)
                    self._finish(r, segments, info, None)
                except Exception as e:
                    self._finish(r, None, None, e)
            if step:
                self._publish_partials(session, in_flight)
            self._publish_settled(session, in_flight)
            self._publish_files(session, files)
            self.files_in_flight = len(files)
            self.rule_admissions = self._rules_before + getattr(session, "rule_admissions", 0)

    # ------------------------------------------------------------------ batched files
    def _admit_files(self, session, files: Dict[int, FileRequest]) -> None:
        with self._cv:
            new, self._files = self._files, []
        for r in new:
            if r.cancelled:
                self._finish_file(r, RequestCancelled("request cancelled before admission"))
            elif not hasattr(session, "add_file"):
                self._finish_file(r, NotImplementedError("this transcriber cannot decode batched files in its loop"))
            else:
                files[session.add_file(r.run, r.max_share, capacity=self.capacity)] = r
                r.admitted.set()

    def _drop_cancelled_files(self, session, files: Dict[int, FileRequest]) -> None:
        for h, r in [(h, r) for h, r in files.items() if r.cancelled]:
            del files[h]
            try:
                session.drop_file(h)
            except Exception as e:
                log.error("cancel of a file failed: %s", e)
            self._finish_file(r, RequestCancelled("request cancelled"))

    def _publish_files(self, session, files: Dict[int, FileRequest]) -> None:
        for h, r in list(files.items()):
            segs = session.file_segments(h, len(r.settled))
            if segs:
                r.settled.extend(segs)
            if session.file_done(h):
                r.steps = list(session.files[h].steps)
                err = session.file_error(h)
                session.drop_file(h)
                del files[h]
                self._finish_file(r, err)

    def _finish_file(self, r: FileRequest, error) -> None:
        r.error = error
        r.finished_at = time.monotonic()
        r.future.set()
        r.settled.event.set()
        r.admitted.set()

    def _announce_admitted(self, session, admitted) -> None:
        """``info`` (language resolved) for the admitted requests that want segments, then their ``admitted`` event.  A
        failing ``info`` leaves ``info`` unset; the stream keeps decoding and its result carries the info."""
        for h, r in admitted:
            if r.want_segments:
                try:
                    r.info = session.info(h)
                except Exception as e:
                    log.error("info of an admitted request failed: %s", e)
            r.admitted.set()

    def _answer_embeddings(self) -> None:
        """Every pending embedding request, in calls of at most ``capacity`` x 30 s of audio -- the workspace
        ``footprint_estimate`` budgets for the speaker embedding -- so a long file's segments cannot grow it further
        (a longer segment goes alone); an error fails only the requests of its call."""
        with self._cv:
            batch, self._embeds = self._embeds, []
        limit = self.capacity * EMBED_CALL_SAMPLES
        group, samples = [], 0
        for r in batch:
            if group and samples + len(r.audio) > limit:
                self._embed_call(group)
                group, samples = [], 0
            group.append(r)
            samples += len(r.audio)
        if group:
            self._embed_call(group)

    def _embed_call(self, batch: List[EmbeddingRequest]) -> None:
        try:
            out = self.transcriber.speaker_embeddings([r.audio for r in batch])
            self.embedding_calls += 1
            for r, v in zip(batch, out):
                r.result = np.asarray(v, dtype=np.float32)
        except Exception as e:
            log.error("speaker embeddings failed: %s", e)
            for r in batch:
                r.error = e
        for r in batch:
            r.future.set()

    def _drop_cancelled(self, session, in_flight: Dict[int, BatchRequest]) -> None:
        """Take the cancelled requests out of the session (index and encoder slots back) and answer them."""
        for h, r in [(h, r) for h, r in in_flight.items() if r.cancelled]:
            del in_flight[h]
            try:
                session.cancel(h)
            except Exception as e:          # the stream stays in the session; its result is dropped when it finishes
                log.error("cancel failed: %s", e)
            self._finish(r, None, None, RequestCancelled("request cancelled"))

    def _publish_partials(self, session, in_flight: Dict[int, BatchRequest]) -> None:
        """One batched ``partials`` call for the in-flight requests that want interim text (none: no peek at all)."""
        want = [h for h, r in in_flight.items() if r.want_partials and not r.cancelled]
        if not want or not hasattr(session, "partials"):
            return
        try:
            got = session.partials(want)
        except Exception as e:              # interim text is best effort: the final result is unaffected
            log.error("partials failed: %s", e)
            return
        for h, segs in got.items():
            in_flight[h].partial.publish(segs)

    def _publish_settled(self, session, in_flight: Dict[int, BatchRequest]) -> None:
        """Append the newly settled segments of the in-flight requests that want them (host state of the session, read
        past each request's cursor only); an error here loses interim segments, never the final result."""
        want = {h: len(r.settled) for h, r in in_flight.items() if r.want_segments and not r.cancelled}
        if not want:
            return
        try:
            got = session.settled(want)
        except Exception as e:
            log.error("settled segments failed: %s", e)
            return
        for h, segs in got.items():
            in_flight[h].settled.extend(segs)

    def _finish(self, r: BatchRequest, segments, info, error) -> None:
        r.result = list(segments) if segments is not None else None
        r.info = info
        r.error = error
        r.finished_at = time.monotonic()
        self.streams_done += 1
        r.future.set()
        r.partial.event.set()
        r.settled.event.set()
        r.admitted.set()


class _OneShotSession:
    """Adapter for transcribers without ``open_session`` (only ``transcribe_batch``): every round is one call."""

    def __init__(self, transcriber):
        self.t = transcriber
        self._pending: List[Any] = []
        self._done: List[Any] = []
        self._n = 0

    def add_streams(self, audios, kws):
        hs = []
        for a, k in zip(audios, kws):
            self._pending.append((self._n, a, k))
            hs.append(self._n)
            self._n += 1
        return hs

    def round(self):
        batch, self._pending = self._pending, []
        try:
            out = self.t.transcribe_batch([a for _, a, _ in batch], [k for _, _, k in batch])
            for (h, _, _), res in zip(batch, out):
                self._done.append(_Done(h, res, None))
        except Exception as e:
            for h, _, _ in batch:
                self._done.append(_Done(h, None, e))

    def cancel(self, handle):
        self._pending = [p for p in self._pending if p[0] != handle]
        self._done = [d for d in self._done if d.handle != handle]

    def pop_finished(self):
        d, self._done = self._done, []
        return d

    def info(self, handle):
        return None                 # known once the call returns

    def settled(self, cursors):
        return {}

    def result_of(self, entry):
        if entry.error is not None:
            raise entry.error
        return entry.res


class _Done:
    def __init__(self, handle, res, error):
        self.handle, self.res, self.error = handle, res, error


# the name the backend plugin and round-1 tests import
StreamScheduler = RoundScheduler
