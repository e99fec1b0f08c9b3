"""ServeClientB200: the WhisperLive backend plugin (Boundary A, SURVEY.md §8b).

Subclass of the reference's own ``whisper_live.backend.base.ServeClientBase`` (audio ring buffer,
``speech_to_text`` loop, segment commit logic and the WebSocket JSON are the reference's, unchanged);
mirrors ``ServeClientFasterWhisper`` (whisper_live/backend/faster_whisper_backend.py): same ctor
signature :19-40, ``SINGLE_MODEL`` / ``BATCH_WORKER`` class attributes :15-17, ``set_language``
:180-194, ``transcribe_audio`` :196-250, ``handle_transcription_output`` :252-267, SERVER_READY with
``"backend": "faster_whisper"`` :123-131 (the stock client only collects transcripts for that backend
name: whisper_live/client.py:182).

Differences that are the point of the port: one engine per model shared by all clients, driven by a
single scheduler thread that batches the chunks of all live connections per decode step
(whisperlive_b200.scheduler.StreamScheduler); no CPU device / compute-type probing -- construction
fails loudly without the CUDA engine.

``single_model=True`` (the constructor default): the first connection's model serves every connection, as the
reference's ``SINGLE_MODEL``.  ``single_model=False`` (the reference server's default): each connection is served by the
model it asked for, from a ``models.ModelRegistry`` shared by the process -- loaded once, kept resident while idle,
evicted least recently used first when a new model needs the memory.
"""
from __future__ import annotations

import json
import logging
import os
import threading
import time

try:  # the reference package must be importable: this module is a plugin for it
    from whisper_live.backend.base import ServeClientBase
except Exception as _e:  # pragma: no cover
    ServeClientBase = None
    _IMPORT_ERROR = _e

from .models import ModelRegistry, engine_footprint
from .scheduler import BatchRequest, StreamScheduler


def vad_from_env():
    """``WLB200_VAD=device``: Silero probabilities on the model's GPU context (``vad.DeviceVad``); unset or ``cpu``:
    faster-whisper's CPU module, as the reference."""
    v = os.environ.get("WLB200_VAD", "cpu").strip().lower()
    if v not in ("cpu", "device"):
        raise ValueError(f"WLB200_VAD={v!r}: 'cpu' (default) or 'device'")
    return "device" if v == "device" else None


def diarize_from_env() -> str:
    """``WLB200_DIARIZE=device``: speaker embeddings on the model's GPU context (``speaker.DeviceSpeakerDiarizer``);
    unset or ``cpu``: the diarizer the reference passes in, untouched."""
    v = os.environ.get("WLB200_DIARIZE", "cpu").strip().lower()
    if v not in ("cpu", "device"):
        raise ValueError(f"WLB200_DIARIZE={v!r}: 'cpu' (default) or 'device'")
    return v


if ServeClientBase is not None:

    class ServeClientB200(ServeClientBase):
        SINGLE_MODEL = None
        SINGLE_MODEL_LOCK = threading.Lock()
        BATCH_WORKER = None
        REGISTRY = None          # models.ModelRegistry of the single_model=False connections (built on first use)
        MAX_STREAMS = 8          # streams batched per decode step on this GPU
        BATCH_WINDOW_MS = 20
        MODEL_FACTORY = None     # tests inject a callable(model_name) -> transcriber
        PARTIALS = os.environ.get("WLB200_PARTIALS", "0") == "1"   # interim text of the chunk in flight
        REQUEST_TIMEOUT_S = 30
        MEMORY_RESERVE_BYTES = 1 << 30   # kept free beyond a new model's footprint (CUDA graphs, allocator rounding)
        WAIT_SLICE_S = 0.05      # how often a waiting client thread looks at exit / new interim text

        def __init__(self, websocket, task="transcribe", device=None, language=None, client_uid=None, model="small.en",
                     initial_prompt=None, vad_parameters=None, use_vad=True, single_model=True, send_last_n_segments=10,
                     no_speech_thresh=0.45, clip_audio=False, same_output_threshold=7, cache_path="~/.cache/whisper-live/",
                     translation_queue=None, hotwords=None, diarization=None, word_timestamps=False):
            super().__init__(client_uid, websocket, send_last_n_segments, no_speech_thresh, clip_audio,
                             same_output_threshold, translation_queue, diarization, word_timestamps)
            self.cache_path = cache_path
            self.model_size_or_path = model
            self.language = "en" if (model or "").endswith("en") else language
            self.task = task
            self.initial_prompt = initial_prompt
            self.vad_parameters = vad_parameters or {"threshold": 0.5}
            self.hotwords = hotwords
            self.compute_type = "float16"
            self.model_entry = None
            self.registry = None
            self.scheduler = None    # the registry entry's scheduler; kept after cleanup() so a chunk in flight finds it
            if self.model_size_or_path is None:
                return
            try:
                cls = ServeClientB200
                if single_model:
                    self.transcriber, _worker = cls.shared_model(self.create_model)
                else:
                    self.registry = cls.model_registry()
                    self.model_entry = self.registry.acquire(self.model_size_or_path)
                    self.transcriber = self.model_entry.transcriber
                    self.scheduler = self.model_entry.scheduler
            except Exception as e:
                logging.error(f"Failed to load model: {e}")
                self.websocket.send(json.dumps({"uid": self.client_uid, "status": "ERROR",
                                                "message": f"Failed to load model: {str(self.model_size_or_path)}"}))
                self.websocket.close()
                return
            self.use_vad = use_vad
            if self.diarization is not None and diarize_from_env() == "device":
                from .speaker import DeviceSpeakerDiarizer
                worker = self.scheduler if self.registry is not None else ServeClientB200.BATCH_WORKER
                self.diarization = DeviceSpeakerDiarizer.replacing(self.diarization, worker)
            self.trans_thread = threading.Thread(target=self.speech_to_text)
            self.trans_thread.start()
            self.websocket.send(json.dumps({"uid": self.client_uid, "message": self.SERVER_READY, "backend": "faster_whisper"}))

        def create_model(self):
            """Build the shared transcriber (CUDA engine). Raises when no H100 / library is available."""
            return ServeClientB200.build_model(self.model_size_or_path, self.compute_type)

        @staticmethod
        def build_model(model_size_or_path, compute_type="float16"):
            if ServeClientB200.MODEL_FACTORY is not None:
                return ServeClientB200.MODEL_FACTORY(model_size_or_path)
            from .parallel import MultiDeviceWhisperModel, devices_from_env
            from .transcriber import B200WhisperModel
            devices = devices_from_env()     # WLB200_DEVICES=0,1,...: one engine context per GPU, streams placed i mod G
            vad = vad_from_env()
            if len(devices) > 1:
                return MultiDeviceWhisperModel(model_size_or_path, device_index=devices, device="cuda",
                                               compute_type=compute_type, max_streams=ServeClientB200.MAX_STREAMS, vad=vad)
            return B200WhisperModel(model_size_or_path, device="cuda", device_index=devices[0],
                                    compute_type=compute_type, max_streams=ServeClientB200.MAX_STREAMS, vad=vad)

        @classmethod
        def shared_model(cls, create):
            """``(SINGLE_MODEL, BATCH_WORKER)``, the model every ``single_model=True`` connection shares and its
            scheduler; ``create()`` builds the model on first use."""
            with cls.SINGLE_MODEL_LOCK:
                if cls.SINGLE_MODEL is None:
                    cls.SINGLE_MODEL = create()
                    cls.BATCH_WORKER = StreamScheduler(cls.SINGLE_MODEL, max_batch_size=cls.MAX_STREAMS,
                                                       batch_window_ms=cls.BATCH_WINDOW_MS)
                    cls.BATCH_WORKER.start()
                return cls.SINGLE_MODEL, cls.BATCH_WORKER

        @classmethod
        def model_registry(cls) -> ModelRegistry:
            """The process's registry of per-connection models.  With the CUDA engine an entry is keyed by the checkpoint
            directory a name resolves to (``weights.resolve_model_dir``, local snapshots only, as ``B200WhisperModel``
            loads them) and a load is checked against the free memory of every configured device; a ``MODEL_FACTORY``
            model is keyed by its name and loaded without a check."""
            with cls.SINGLE_MODEL_LOCK:
                if cls.REGISTRY is None:
                    kw = {}
                    if cls.MODEL_FACTORY is None:
                        from .parallel import devices_from_env
                        from .weights import resolve_model_dir
                        resolve = lambda name: resolve_model_dir(name, local_files_only=True)
                        kw = dict(resolve=resolve, devices=devices_from_env(), reserve_bytes=cls.MEMORY_RESERVE_BYTES,
                                  footprint=lambda name: engine_footprint(name, cls.MAX_STREAMS, resolve=resolve,
                                                                         vad=vad_from_env() == "device",
                                                                         diarize=diarize_from_env() == "device"))
                    cls.REGISTRY = ModelRegistry(cls.build_model, max_streams=cls.MAX_STREAMS,
                                                 batch_window_ms=cls.BATCH_WINDOW_MS, **kw)
                return cls.REGISTRY

        def cleanup(self):
            """The connection ended (the server calls this on disconnect): its model loses a connection, then the
            reference's cleanup stops the transcription thread.  A chunk the thread submits in between still goes to
            this model's scheduler (``self.scheduler`` stays set) and is cancelled once ``exit`` is set."""
            entry, self.model_entry = getattr(self, "model_entry", None), None
            if entry is not None:
                self.registry.release(entry)
            super().cleanup()

        def set_language(self, info):
            if info.language_probability > 0.5:
                self.language = info.language
                logging.info(f"Detected language {self.language} with probability {info.language_probability}")
                self.websocket.send(json.dumps({"uid": self.client_uid, "language": self.language,
                                                "language_prob": info.language_probability}))

        def transcribe_audio(self, input_sample):
            """Submit the chunk and wait for it in short slices: interim text goes out while it decodes (``PARTIALS``),
            and a timeout or a disconnect (``self.exit``) cancels the request so it stops using the engine."""
            request = BatchRequest(audio=input_sample, language=self.language, task=self.task,
                                   initial_prompt=self.initial_prompt, use_vad=self.use_vad,
                                   vad_parameters=self.vad_parameters if self.use_vad else None,
                                   word_timestamps=self.word_timestamps, client_uid=self.client_uid, hotwords=self.hotwords,
                                   want_partials=self.PARTIALS)
            worker = self.scheduler if self.registry is not None else ServeClientB200.BATCH_WORKER
            worker.submit(request)
            duration = input_sample.shape[0] / self.RATE
            deadline = time.monotonic() + self.REQUEST_TIMEOUT_S
            sent = 0
            while not request.future.is_set():
                if self.exit:
                    request.cancel()
                    return None
                left = deadline - time.monotonic()
                if left <= 0:
                    request.cancel()
                    raise TimeoutError(f"transcription request timed out after {self.REQUEST_TIMEOUT_S} s")
                request.partial.event.wait(timeout=min(self.WAIT_SLICE_S, left))
                request.partial.event.clear()
                version, segs = request.partial.latest()
                if version != sent and not request.future.is_set():
                    sent = version
                    self.send_interim(segs, duration)
            if request.error:
                raise request.error
            if self.language is None and request.info is not None:
                self.set_language(request.info)
            return request.result

        def send_interim(self, segments, duration):
            """The unfinished text of the chunk in flight as the reference's incomplete line: the recent transcript plus
            one ``completed: False`` segment (``prepare_segments(last)``).  Segments over ``no_speech_thresh`` are left
            out as ``update_segments`` does; the transcript, ``timestamp_offset`` and the rest of the commit state stay
            as they are."""
            kept = [s for s in segments if self.get_segment_no_speech_prob(s) <= self.no_speech_thresh]
            if not kept:
                return
            with self.lock:
                offset = self.timestamp_offset
            last = self.format_segment(offset + self.get_segment_start(kept[0]),
                                       offset + min(duration, self.get_segment_end(kept[-1])),
                                       "".join(s.text for s in kept), completed=False)
            self.send_transcription_to_client(self.prepare_segments(last))

        def handle_transcription_output(self, result, duration):
            segments = []
            if len(result):
                self.t_start = None
                last_segment = self.update_segments(result, duration)
                segments = self.prepare_segments(last_segment)
            if len(segments):
                self.send_transcription_to_client(segments)

        @classmethod
        def shutdown(cls):
            if cls.BATCH_WORKER is not None:
                cls.BATCH_WORKER.stop()
            cls.BATCH_WORKER = None
            cls.SINGLE_MODEL = None
            if cls.REGISTRY is not None:
                cls.REGISTRY.shutdown()
            cls.REGISTRY = None

else:

    class ServeClientB200:  # type: ignore
        def __init__(self, *a, **k):
            raise ImportError("whisper_live (the reference package) is not importable: ServeClientB200 is a plugin "
                              f"for whisper_live.backend.base.ServeClientBase ({_IMPORT_ERROR})")
