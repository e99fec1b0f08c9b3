"""ModelRegistry: several Whisper models resident on the GPU, each served by its own ``RoundScheduler``.

The reference lets every connection choose its model (the ``model`` of its first message): with ``single_model`` off,
``ServeClientFasterWhisper`` builds the model each client asks for (whisper_live/backend/faster_whisper_backend.py:99-107).
The backend plugin does the same with ``single_model=False``, through this registry, without building a model per
connection:

* an entry is keyed by the resolved checkpoint (the model directory, or the name itself when there is nothing to
  resolve), so ``"large-v3"`` and the path of the same snapshot share one entry;
* an entry holds the transcriber, its own ``RoundScheduler`` (thread + CUDA stream), a connection count and the time
  it was last acquired or released;
* ``acquire(name)`` loads a model once: concurrent requests for it wait for that one load, and a load holds no lock
  the schedulers or the acquisitions of loaded models need;
* ``release(entry)`` drops a connection; an entry without connections stays loaded for the next client;
* before a load, the model's footprint (``engine.footprint_estimate``) is compared with the free memory of every device
  it will live on (``wl_mem_info``), less what the resident models will still allocate: an engine allocates its decode
  session and its first-round workspaces lazily, so each resident entry's footprint minus the bytes it holds now
  (``device_bytes``) is spoken for.  Idle entries are evicted, least recently used first, until it fits; an entry with
  connections is never evicted.  When it still does not fit the load fails before anything is allocated.  Evicting
  stops the entry's scheduler and destroys its engine contexts; an entry whose scheduler does not stop stays listed
  (``evicting()``) and is destroyed at a later load or at ``shutdown`` once its thread has exited.

The per-model schedulers run side by side: their decode loops share the GPU, which interleaves their kernels.
"""
from __future__ import annotations

import logging
import os
import threading
import time
from typing import Callable, Dict, List, Optional, Sequence

from .scheduler import RoundScheduler

log = logging.getLogger("whisperlive_b200.models")

GiB = 1 << 30


class ModelEntry:
    """One resident model: ``transcriber``, its ``scheduler``, ``connections`` and ``last_used`` (monotonic seconds)."""

    def __init__(self, key: str, name: str, transcriber, scheduler: RoundScheduler, footprint: Optional[int]):
        self.key, self.name = key, name
        self.transcriber = transcriber
        self.scheduler = scheduler
        self.footprint = footprint
        self.connections = 0
        self.last_used = 0.0


class _Load:
    """A load in progress: the other requesters of the same model wait on ``done``."""

    def __init__(self):
        self.done = threading.Event()
        self.error: Optional[BaseException] = None


class ModelRegistry:
    def __init__(self, factory: Callable[[str], object], *, max_streams: int = 8, batch_window_ms: int = 20,
                 resolve: Optional[Callable[[str], str]] = None, footprint: Optional[Callable[[str], Optional[int]]] = None,
                 mem_probe: Optional[Callable[[int], int]] = None, devices: Sequence[int] = (0,),
                 reserve_bytes: int = 0, clock: Callable[[], float] = time.monotonic,
                 translator_pending: Optional[Callable[[int], int]] = None):
        """``factory(name)`` builds a transcriber.  ``resolve(name)`` gives the key of a name (default: the name).
        ``footprint(name)`` the device bytes one copy of the model needs (None: unknown, loaded without a check).
        ``mem_probe(device)`` the free bytes of a device (default ``wl_mem_info``).  ``devices``: where every model is
        placed (one copy per device).  ``reserve_bytes``: kept free beyond the footprint.  ``translator_pending(device)``:
        the bytes the process-wide translator will still allocate there (default: its footprint while
        ``WLB200_TRANSLATE=device`` and it is not loaded yet)."""
        self.factory = factory
        self.max_streams = int(max_streams)
        self.batch_window_ms = batch_window_ms
        self.resolve = resolve or (lambda name: str(name))
        self.footprint = footprint
        self.mem_probe = mem_probe
        self.devices = [int(d) for d in devices] or [0]
        self.reserve_bytes = int(reserve_bytes)
        self.clock = clock
        if translator_pending is None:
            from .translation import pending_translator_bytes as translator_pending
        self.translator_pending = translator_pending
        self._lock = threading.Lock()          # entries, loads in progress, connection counts
        self._load_lock = threading.Lock()     # one check-evict-load at a time: two loads never count the same free bytes
        self._entries: Dict[str, ModelEntry] = {}
        self._loading: Dict[str, _Load] = {}
        self._evicting: List[ModelEntry] = []   # evicted, but the scheduler thread had not exited: not yet destroyed
        self.loads = 0
        self.evictions = 0

    # ------------------------------------------------------------------ connections
    def acquire(self, name: str) -> ModelEntry:
        """The entry serving ``name`` with one more connection; loads the model (once) when it is not resident.
        Raises what the load raised, ``MemoryError`` when the model does not fit."""
        key = self.resolve(name)
        while True:
            with self._lock:
                e = self._entries.get(key)
                if e is not None:
                    e.connections += 1
                    e.last_used = self.clock()
                    return e
                pending = self._loading.get(key)
                owner = pending is None
                if owner:
                    pending = self._loading[key] = _Load()
            if not owner:
                pending.done.wait()
                if pending.error is not None:
                    raise pending.error
                continue
            try:
                e = self._load(key, name)
            except BaseException as err:
                with self._lock:
                    del self._loading[key]
                pending.error = err
                pending.done.set()
                raise
            with self._lock:
                e.connections = 1
                e.last_used = self.clock()
                self._entries[key] = e
                del self._loading[key]
            pending.done.set()
            return e

    def release(self, entry: ModelEntry) -> None:
        """One connection of ``entry`` ended; the model stays resident."""
        with self._lock:
            entry.connections = max(0, entry.connections - 1)
            entry.last_used = self.clock()

    def entries(self) -> Dict[str, ModelEntry]:
        with self._lock:
            return dict(self._entries)

    def evicting(self) -> List[ModelEntry]:
        """Evicted entries whose scheduler thread had not exited, so their contexts are not destroyed yet."""
        with self._lock:
            return list(self._evicting)

    def shutdown(self) -> None:
        """Stop every scheduler and forget the entries (destroying those whose eviction was still pending)."""
        with self._lock:
            entries, self._entries = list(self._entries.values()), {}
        for e in entries:
            e.scheduler.stop()
        self._finish_evictions()

    # ------------------------------------------------------------------ loading and eviction
    def _load(self, key: str, name: str) -> ModelEntry:
        with self._load_lock:
            need = self.footprint(name) if self.footprint is not None else None
            if need is not None:
                self._make_room(name, int(need))
            transcriber = self.factory(name)
            try:
                scheduler = RoundScheduler(transcriber, max_batch_size=self.max_streams, batch_window_ms=self.batch_window_ms)
                scheduler.start()
            except BaseException:
                _destroy(transcriber)
                raise
            self.loads += 1
            return ModelEntry(key, name, transcriber, scheduler, need)

    def _pending_bytes(self, device: int) -> int:
        """What the resident models will still allocate on ``device``: footprint minus the bytes each holds now, and
        the translator's footprint until it is loaded."""
        with self._lock:
            entries = list(self._entries.values())
        pending = int(self.translator_pending(device))
        for e in entries:
            if e.footprint is None:
                continue
            held = _held_bytes(e.transcriber, device)
            if held is not None:
                pending += max(0, int(e.footprint) - held)
        return pending

    def _short_devices(self, need: int) -> Dict[int, int]:
        probe = self.mem_probe or _wl_free_bytes
        free = {d: int(probe(d)) - self._pending_bytes(d) for d in self.devices}
        return {d: f for d, f in free.items() if f < need + self.reserve_bytes}

    def _make_room(self, name: str, need: int) -> None:
        self._finish_evictions()
        while True:
            short = self._short_devices(need)
            if not short:
                return
            with self._lock:
                idle = [e for e in self._entries.values() if e.connections == 0]
                victim = min(idle, key=lambda e: e.last_used) if idle else None
                if victim is not None:
                    del self._entries[victim.key]      # no acquire can take it from here on
            if victim is None:
                d, f = next(iter(short.items()))
                raise MemoryError(f"model {name!r} needs {need / GiB:.2f} GiB (+{self.reserve_bytes / GiB:.2f} GiB reserve) "
                                  f"on device {d}, {f / GiB:.2f} GiB free after what the resident models will still "
                                  f"allocate, and every resident model has connections")
            log.info("evicting idle model %r to load %r", victim.name, name)
            self._evict(victim)

    def _evict(self, e: ModelEntry) -> None:
        e.scheduler.stop()
        if _running(e.scheduler):
            # the owner thread still drives the engine: freeing its contexts under it would fault.  The entry stays
            # listed until its thread has exited, and is destroyed then (_finish_evictions).
            log.error("scheduler of %r did not stop; its contexts are destroyed once it has", e.name)
            with self._lock:
                self._evicting.append(e)
            return
        _destroy(e.transcriber)
        self.evictions += 1

    def _finish_evictions(self) -> None:
        """Destroy the evicted entries whose scheduler thread has exited since."""
        with self._lock:
            done = [e for e in self._evicting if not _running(e.scheduler)]
            self._evicting = [e for e in self._evicting if e not in done]
        for e in done:
            _destroy(e.transcriber)
            self.evictions += 1


def _running(scheduler) -> bool:
    thread = getattr(scheduler, "_thread", None)
    return thread is not None and thread.is_alive()


def _held_bytes(transcriber, device: int) -> Optional[int]:
    """Device bytes ``transcriber`` holds on ``device`` now (``device_bytes``: an int for a single-device model, a
    per-device dict for ``MultiDeviceWhisperModel``); None when it does not report them."""
    held = getattr(transcriber, "device_bytes", None)
    if held is None:
        return None
    if isinstance(held, dict):
        return int(held.get(int(device), 0))
    return int(held)


def _destroy(transcriber) -> None:
    fn = getattr(transcriber, "destroy", None) or getattr(transcriber, "close", None)
    if fn is not None:
        fn()


def _wl_free_bytes(device: int) -> int:
    from .engine import mem_info
    return mem_info(device)[0]


def engine_footprint(name: str, max_streams: int = 8, max_beam: int = 5, resolve: Optional[Callable[[str], str]] = None,
                     vad: bool = False, diarize: bool = False) -> Optional[int]:
    """``footprint_estimate`` of the CUDA engine for a size name, or for a model directory whose HF ``config.json``
    or weight headers (safetensors header or index, ``pytorch_model.bin``, CTranslate2 ``model.bin`` table) give the
    shapes; None only for a directory with no readable header.  ``vad``: the model runs the
    Silero VAD on its context (``vad="device"``); ``diarize``: it computes speaker embeddings there
    (``WLB200_DIARIZE=device``)."""
    from .config import WhisperDims, dims_for
    from .engine import footprint_estimate
    try:
        dims = dims_for(name)
    except KeyError:
        dims = None
        path = resolve(name) if resolve is not None else name
        cfg_path = os.path.join(path, "config.json") if isinstance(path, str) else ""
        if os.path.isfile(cfg_path):
            import json
            with open(cfg_path, "r", encoding="utf-8") as f:
                cfg = json.load(f)
            if "d_model" in cfg:
                dims = WhisperDims(str(name), int(cfg["d_model"]), int(cfg["d_model"]) // 64, int(cfg["encoder_layers"]),
                                   int(cfg["decoder_layers"]), int(cfg["num_mel_bins"]), int(cfg["vocab_size"]))
        if dims is None and isinstance(path, str) and os.path.isdir(path):
            from .weights import checkpoint_dims
            dims = checkpoint_dims(path, str(name))
        if dims is None:
            return None
    return footprint_estimate(dims, max_streams=max_streams, max_beam=max_beam, vad=vad, diarize=diarize)
