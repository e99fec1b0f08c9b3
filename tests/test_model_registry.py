"""Several models per process: the model registry (acquire / release / eviction), the backend plugin's
``single_model=False`` path, the device-memory accounting of the C ABI and the distil / turbo model names."""
import json
import os
import sys
import threading
import time
from types import SimpleNamespace

import numpy as np
import pytest

REF = "/root/reference"


# ------------------------------------------------------------------ fixtures (CPU)
class FakeModel:
    """A transcriber whose every segment names the model that produced it; ``transcribe_batch`` only, so
    RoundScheduler drives it through its one-shot adapter.  It holds ``up_front`` bytes once built (default: its whole
    footprint) and the rest of its footprint from its first chunk on, as the engine allocates its decode session and
    first-round workspaces lazily."""

    def __init__(self, name, footprint=0, gate=None, up_front=None):
        self.name, self.footprint, self.gate = name, footprint, gate
        self.held = footprint if up_front is None else up_front
        self.destroyed = False
        self.calls = 0

    @property
    def device_bytes(self):
        return 0 if self.destroyed else self.held

    def transcribe_batch(self, audios, kws):
        self.calls += 1
        self.held = max(self.held, self.footprint)
        if self.gate is not None:
            self.gate.wait(30)
        seg = lambda a: SimpleNamespace(id=1, start=0.0, end=len(a) / 16000, text=self.name, tokens=[1], no_speech_prob=0.0,
                                        words=None)
        return [([seg(a)], None) for a in audios]

    def destroy(self):
        self.destroyed = True


class Factory:
    def __init__(self, footprint=None, delay=0.0, block=None, up_front=None):
        self.footprint = footprint or {}
        self.up_front = up_front or {}
        self.delay, self.block = delay, block or {}
        self.built = []
        self._lock = threading.Lock()

    def __call__(self, name):
        if name in self.block:
            self.block[name].wait(30)
        if self.delay:
            time.sleep(self.delay)
        m = FakeModel(name, self.footprint.get(name, 0), up_front=self.up_front.get(name))
        with self._lock:
            self.built.append(m)
        return m


class Memory:
    """Injected probe: ``capacity`` minus the bytes the models built so far hold now."""

    def __init__(self, factory, capacity):
        self.factory, self.capacity = factory, capacity

    def __call__(self, device):
        return self.capacity - sum(m.device_bytes for m in self.factory.built)


def _registry(factory, **kw):
    from whisperlive_b200.models import ModelRegistry
    return ModelRegistry(factory, max_streams=2, batch_window_ms=0, **kw)


def _run(entry, seconds=1.0):
    from whisperlive_b200.scheduler import BatchRequest
    r = BatchRequest(audio=np.zeros(int(16000 * seconds), dtype=np.float32), use_vad=False)
    entry.scheduler.submit(r)
    return r


def _round_threads():
    return [t for t in threading.enumerate() if t.name == "wlb200-rounds" and t.is_alive()]


# ------------------------------------------------------------------ registry (CPU)
def test_eight_concurrent_acquires_load_once():
    f = Factory(delay=0.3)
    reg = _registry(f)
    got, errs = [], []
    go = threading.Barrier(8)

    def worker():
        go.wait()
        try:
            got.append(reg.acquire("tiny.en"))
        except Exception as e:   # pragma: no cover
            errs.append(e)
    ts = [threading.Thread(target=worker) for _ in range(8)]
    try:
        for t in ts:
            t.start()
        for t in ts:
            t.join(30)
        assert not errs and len(got) == 8
        assert len(f.built) == 1 and reg.loads == 1
        assert all(e is got[0] for e in got) and got[0].connections == 8
    finally:
        reg.shutdown()


def test_same_model_shares_entry_and_key_is_the_resolved_checkpoint():
    f = Factory()
    reg = _registry(f, resolve=lambda n: "/snapshots/large-v3" if n in ("large-v3", "/snapshots/large-v3") else n)
    try:
        a = reg.acquire("large-v3")
        b = reg.acquire("/snapshots/large-v3")
        assert a is b and a.scheduler is b.scheduler and a.connections == 2 and len(f.built) == 1
        reg.release(a)
        reg.release(b)
        assert a.connections == 0 and reg.entries()["/snapshots/large-v3"] is a    # idle, still resident
        assert reg.acquire("large-v3") is a and len(f.built) == 1
    finally:
        reg.shutdown()


def test_a_blocked_load_does_not_hold_up_a_loaded_model():
    gate = threading.Event()
    f = Factory(block={"small": gate})
    reg = _registry(f)
    try:
        a = reg.acquire("tiny.en")
        loader = threading.Thread(target=lambda: reg.acquire("small"))
        loader.start()
        time.sleep(0.2)
        assert loader.is_alive()                     # model B's factory is blocked ...
        r = _run(a)
        assert r.future.wait(10), "a request on model A waited for model B's load"
        assert r.error is None and r.result[0].text == "tiny.en"
        assert reg.acquire("tiny.en") is a           # ... and so is neither acquiring A
        gate.set()
        loader.join(30)
        assert not loader.is_alive() and "small" in reg.entries()
    finally:
        gate.set()
        reg.shutdown()


def test_eviction_takes_the_least_recently_used_idle_entry():
    now = [0.0]
    f = Factory(footprint={"a": 40, "b": 40, "c": 40})
    reg = _registry(f, footprint=lambda n: 40, mem_probe=Memory(f, 100), clock=lambda: now[0])
    try:
        ea = reg.acquire("a")
        now[0] = 1.0
        eb = reg.acquire("b")
        now[0] = 2.0
        reg.release(eb)              # b idle since t = 2
        now[0] = 3.0
        reg.release(ea)              # a idle since t = 3: b is the least recently used
        now[0] = 4.0
        ec = reg.acquire("c")        # 20 free, needs 40: one eviction
        assert set(reg.entries()) == {"a", "c"} and reg.evictions == 1
        mb = next(m for m in f.built if m.name == "b")
        assert mb.destroyed and not any(m.destroyed for m in f.built if m.name != "b")
        assert eb.scheduler._thread is not None and not eb.scheduler._thread.is_alive()
        assert ea.scheduler._thread.is_alive() and ec.scheduler._thread.is_alive()
        r = _run(ec)
        assert r.future.wait(10) and r.result[0].text == "c"
    finally:
        reg.shutdown()


def test_an_entry_with_connections_is_never_evicted():
    f = Factory(footprint={"a": 40, "b": 40, "c": 40, "d": 40})
    reg = _registry(f, footprint=lambda n: 40, mem_probe=Memory(f, 100))
    try:
        ea = reg.acquire("a")        # keeps its connection throughout
        eb = reg.acquire("b")
        reg.release(eb)
        ec = reg.acquire("c")        # evicts idle b, not connected a
        assert set(reg.entries()) == {"a", "c"}
        threads = len(_round_threads())
        with pytest.raises(MemoryError, match="every resident model has connections"):
            reg.acquire("d")         # a and c both have connections
        assert set(reg.entries()) == {"a", "c"} and not any(m.destroyed for m in f.built if m.name in ("a", "c"))
        assert [m.name for m in f.built].count("d") == 0          # nothing was built for d
        assert len(_round_threads()) == threads
        reg.release(ec)
        assert reg.acquire("d").connections == 1 and set(reg.entries()) == {"a", "d"}
        assert ea.connections == 1
    finally:
        reg.shutdown()


def test_what_resident_models_will_still_allocate_is_spoken_for():
    """A resident model holds only part of its footprint until its first chunk; that rest is not free memory."""
    f = Factory(footprint={"a": 40, "b": 40, "c": 40}, up_front={"a": 10, "b": 10, "c": 10})
    reg = _registry(f, footprint=lambda n: 40, mem_probe=Memory(f, 100))
    try:
        ea = reg.acquire("a")                        # holds 10 of 40
        eb = reg.acquire("b")                        # 90 free, 30 spoken for by a: fits
        assert Memory(f, 100)(0) == 80
        with pytest.raises(MemoryError, match="every resident model has connections"):
            reg.acquire("c")                         # 80 free, but a and b will still take 60 of it
        assert [m.name for m in f.built] == ["a", "b"]
        for e, name in ((ea, "a"), (eb, "b")):       # their first chunks: both grow to their footprint, no overrun
            r = _run(e)
            assert r.future.wait(10) and r.result[0].text == name
        assert Memory(f, 100)(0) == 20
        reg.release(eb)
        assert reg.acquire("c").connections == 1 and set(reg.entries()) == {"a", "c"}
    finally:
        reg.shutdown()


def test_an_eviction_whose_scheduler_does_not_stop_stays_tracked():
    f = Factory(footprint={"a": 40, "b": 40})
    reg = _registry(f, footprint=lambda n: 40, mem_probe=Memory(f, 60))
    ea = reg.acquire("a")
    reg.release(ea)
    real = ea.scheduler
    busy = threading.Event()
    stuck = SimpleNamespace(stop=lambda: None, _thread=threading.Thread(target=busy.wait, args=(30,)))
    stuck._thread.start()
    ea.scheduler = stuck                             # a scheduler whose owner thread outlives stop()
    try:
        with pytest.raises(MemoryError):
            reg.acquire("b")                         # a is evicted but cannot be destroyed yet: b does not fit
        ma = f.built[0]
        assert not ma.destroyed and reg.evicting() == [ea] and reg.entries() == {}
        busy.set()
        stuck._thread.join(10)
        assert reg.acquire("b").connections == 1     # the next load destroys a first
        assert ma.destroyed and reg.evicting() == [] and reg.evictions == 1
    finally:
        busy.set()
        real.stop()
        reg.shutdown()


def test_a_failed_load_is_raised_to_every_waiter_and_leaves_no_entry():
    class Boom(Factory):
        def __call__(self, name):
            time.sleep(0.2)
            raise FileNotFoundError(f"no checkpoint for {name!r}")
    reg = _registry(Boom())
    errs = []

    def worker():
        try:
            reg.acquire("nope")
        except FileNotFoundError as e:
            errs.append(e)
    ts = [threading.Thread(target=worker) for _ in range(3)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(30)
    assert len(errs) == 3 and reg.entries() == {} and reg.loads == 0


# ------------------------------------------------------------------ model names (CPU)
@pytest.mark.parametrize("name", ["distil-small.en", "distil-medium.en", "distil-large-v2", "distil-large-v3",
                                  "large-v3-turbo", "turbo"])
def test_distil_and_turbo_dims_match_their_weights(name):
    from whisperlive_b200.config import dims_for
    from whisperlive_b200.weights import infer_dims, random_init
    d = dims_for(name)
    w = random_init(d, seed=0)
    got = infer_dims(w, name)
    key = lambda x: (x.d_model, x.n_heads, x.enc_layers, x.dec_layers, x.n_mels, x.vocab)
    assert key(got) == key(d)


def test_hub_repositories():
    from whisperlive_b200.weights import hub_repo
    assert hub_repo("distil-small.en") == "Systran/faster-distil-whisper-small.en"
    assert hub_repo("distil-medium.en") == "Systran/faster-distil-whisper-medium.en"
    assert hub_repo("distil-large-v2") == "Systran/faster-distil-whisper-large-v2"
    assert hub_repo("distil-large-v3") == "Systran/faster-distil-whisper-large-v3"
    assert hub_repo("large-v3-turbo") == "mobiuslabsgmbh/faster-whisper-large-v3-turbo"
    assert hub_repo("turbo") == "mobiuslabsgmbh/faster-whisper-large-v3-turbo"
    assert hub_repo("small.en") == "Systran/faster-whisper-small.en"
    assert hub_repo("large-v3") == "Systran/faster-whisper-large-v3"
    assert hub_repo("someone/custom-whisper") == "someone/custom-whisper"


def test_footprint_estimate_grows_with_the_shapes():
    from whisperlive_b200.config import dims_for
    from whisperlive_b200.engine import footprint_estimate
    t = footprint_estimate(dims_for("tiny.en"), 8, 5)
    assert footprint_estimate(dims_for("small"), 8, 5) > t > 0
    assert footprint_estimate(dims_for("tiny.en"), 16, 5) > t
    assert footprint_estimate(dims_for("tiny.en"), 8, 5, enc_slots=32) > t


# ------------------------------------------------------------------ backend plugin (CPU)
class WS:
    def __init__(self):
        self.sent, self.closed = [], False

    def send(self, msg):
        self.sent.append(json.loads(msg))

    def close(self):
        self.closed = True


@pytest.fixture
def plugin():
    if not os.path.isdir(REF):
        pytest.skip("reference tree not present")
    sys.path.insert(0, REF)
    try:
        from whisperlive_b200.backend import ServeClientB200
    finally:
        sys.path.remove(REF)
    factory = Factory()
    ServeClientB200.MODEL_FACTORY = factory
    clients = []

    def connect(model, **kw):
        c = ServeClientB200(WS(), client_uid=f"u{len(clients)}", model=model, use_vad=False, **kw)
        clients.append(c)
        return c
    try:
        yield ServeClientB200, factory, connect
    finally:
        for c in clients:
            c.cleanup()
            t = getattr(c, "trans_thread", None)
            if t is not None:
                t.join(timeout=10)
        ServeClientB200.shutdown()
        ServeClientB200.MODEL_FACTORY = None


def _transcribe(client):
    return client.transcribe_audio(np.zeros(16000, dtype=np.float32))


def test_single_model_serves_every_connection_with_the_first_model(plugin):
    cls, factory, connect = plugin
    a = connect("small.en")
    b = connect("large-v3")
    assert len(factory.built) == 1 and factory.built[0].name == "small.en"
    assert a.transcriber is b.transcriber is cls.SINGLE_MODEL and cls.REGISTRY is None
    assert _transcribe(b)[0].text == "small.en"
    assert a.websocket.sent[0]["message"] == "SERVER_READY"


def test_each_connection_gets_its_own_model(plugin):
    cls, factory, connect = plugin
    a = connect("small.en", single_model=False)
    b = connect("large-v3", single_model=False)
    c = connect("small.en", single_model=False)
    assert sorted(m.name for m in factory.built) == ["large-v3", "small.en"] and cls.SINGLE_MODEL is None
    assert _transcribe(a)[0].text == "small.en" and _transcribe(b)[0].text == "large-v3"
    assert a.model_entry is c.model_entry and a.model_entry.scheduler is c.model_entry.scheduler
    assert a.model_entry.connections == 2 and b.model_entry is not a.model_entry
    assert a.language == "en" and b.language is None            # the latch keys on each connection's own model
    entry = a.model_entry
    a.cleanup()
    assert entry.connections == 1 and a.model_entry is None
    c.cleanup()
    assert entry.connections == 0 and "small.en" in cls.REGISTRY.entries()   # idle, still resident


def test_a_chunk_after_disconnect_is_dropped_quietly(plugin):
    """cleanup() releases the model before the reference's cleanup sets ``exit``: a chunk the transcription thread
    submits in between still reaches the connection's scheduler and is cancelled, with no error."""
    cls, factory, connect = plugin
    a = connect("small.en", single_model=False)
    a.cleanup()
    assert a.model_entry is None and a.exit
    assert _transcribe(a) is None


def test_a_model_that_does_not_fit_is_refused(plugin):
    cls, factory, connect = plugin
    from whisperlive_b200.models import ModelRegistry
    factory.footprint = {"small.en": 60, "large-v3": 60}
    cls.REGISTRY = ModelRegistry(factory, max_streams=2, footprint=lambda n: 60, mem_probe=Memory(factory, 100))
    a = connect("small.en", single_model=False)
    threads = len(_round_threads())
    b = connect("large-v3", single_model=False)
    assert b.websocket.sent == [{"uid": "u1", "status": "ERROR", "message": "Failed to load model: large-v3"}]
    assert b.websocket.closed and b.model_entry is None and not hasattr(b, "trans_thread")
    assert [m.name for m in factory.built] == ["small.en"] and set(cls.REGISTRY.entries()) == {"small.en"}
    assert len(_round_threads()) == threads
    assert _transcribe(a)[0].text == "small.en"


# ------------------------------------------------------------------ GPU
def _gpu_model(name, max_streams=4, seed=0):
    from whisperlive_b200.transcriber import B200WhisperModel
    return B200WhisperModel(name, weights="random", seed=seed, hf_tokenizer="synthetic", max_streams=max_streams)


def _chunks():
    from whisperlive_b200 import synth
    return [synth.speech_like(d, seed=50 + i) for i, d in enumerate((4.0, 7.5, 11.0))]


_KW = dict(language="en", use_vad=False)


def _submit(sch, wave):
    from whisperlive_b200.scheduler import BatchRequest
    r = BatchRequest(audio=wave, **_KW)
    sch.submit(r)
    return r


def _key(r):
    assert r.future.wait(300) and r.error is None, r.error
    return [(list(s.tokens), s.start, s.end, s.text) for s in r.result]


@pytest.mark.gpu
def test_two_models_side_by_side_match_each_alone():
    """tiny.en and small resident in one process, each with its own RoundScheduler; chunks submitted to both
    interleaved give the tokens and segments each model gives alone."""
    from whisperlive_b200.scheduler import RoundScheduler
    names = ("tiny.en", "small")
    waves = _chunks()
    alone = {}
    for n in names:
        m = _gpu_model(n)
        sch = RoundScheduler(m, max_batch_size=4)
        sch.start()
        try:
            alone[n] = [_key(_submit(sch, w)) for w in waves]
        finally:
            sch.stop()
            m.destroy()
    models = {n: _gpu_model(n) for n in names}
    schs = {n: RoundScheduler(models[n], max_batch_size=4) for n in names}
    for s in schs.values():
        s.start()
    try:
        for i, w in enumerate(waves):
            rs = {n: _submit(schs[n], w) for n in names}     # both models decode this chunk at once
            for n in names:
                assert _key(rs[n]) == alone[n][i], (n, i)
    finally:
        for n in names:
            schs[n].stop()
            models[n].destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny.en", "small", "large-v3"])
def test_device_bytes_and_footprint_estimate(name):
    from whisperlive_b200.engine import footprint_estimate
    from whisperlive_b200 import synth
    m = _gpu_model(name, max_streams=8)
    eng = m.model
    try:
        loaded = eng.device_bytes
        assert loaded > 0
        ds = eng.open_decode_session(beam_size=5)
        opened = eng.device_bytes
        assert opened > loaded                      # the session's decode state and self-attention cache
        ds.close()
        sess = m.open_session()
        waves = [synth.speech_like(6.0 + i, seed=80 + i) for i in range(8)]
        sess.add_streams(waves, [dict(language="en", vad_filter=False) for _ in waves])
        sess.step_round(16)
        measured = eng.device_bytes
        sess.close()
        est = footprint_estimate(m.model.dims, max_streams=8, max_beam=5)
        assert measured >= opened
        assert measured <= est <= 1.10 * measured, (name, est, measured, est / measured)
    finally:
        m.destroy()
    assert eng.device_bytes == 0


@pytest.mark.gpu
def test_mem_info_reports_the_device():
    from whisperlive_b200.engine import mem_info
    free, total = mem_info(0)
    assert 0 <= free <= total and total > 0
