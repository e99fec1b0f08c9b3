"""Speaker embeddings on the device (whisperlive_b200/speaker.py, csrc/spk.cu): the fbank protocol against torchaudio,
the checkpoint reader and BN folding, the random weights' activation range, the diarizer's clustering against the
reference's own, the scheduler's batched embedding requests, the backend switch, and on the GPU every conv launch,
wl_spk_embed and the diarizer against the float64 oracle (tests/spk_oracle.py)."""
import importlib.util
import os
import sys
import threading
import time

import numpy as np
import pytest

from tests import spk_oracle as O
from whisperlive_b200 import speaker as S
from whisperlive_b200 import synth
from whisperlive_b200.scheduler import BatchRequest, RoundScheduler

REF = "/root/reference"
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _golden_waveforms():
    spec = importlib.util.spec_from_file_location("make_golden_spk_fbank", os.path.join(GOLDEN, "make_golden_spk_fbank.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.waveforms()


def _golden_fbank():
    """name -> (torchaudio's frame count, the kept frame indices, the fbank at those frames)"""
    gold = np.load(os.path.join(GOLDEN, "spk_fbank_reference.npz"))
    names = [k[len("fbank_"):] for k in gold.files if k.startswith("fbank_")]
    return {n: (int(gold["frames_" + n]), gold["index_" + n], gold["fbank_" + n]) for n in names}


def _fbank_tol(value: np.ndarray) -> np.ndarray:
    """1e-4, widened by the conditioning of fp32 power sums: torchaudio (fp32) loses ~1e-7 of a frame's total energy in
    every bin, which is a large share of the log of a bin far below the frame's energy (a pure tone's far bins)."""
    lse = np.log(np.exp(value.astype(np.float64)).sum(axis=1, keepdims=True))
    return 1e-4 + 2e-6 * np.exp(lse - value)


# ------------------------------------------------------------------ fbank protocol
def test_oracle_fbank_equals_torchaudio_golden():
    gold = _golden_fbank()
    waves = _golden_waveforms()
    assert sorted(waves) == sorted(gold)
    for name, w in waves.items():
        frames, idx, g = gold[name]
        o = O.fbank(w)
        assert o.shape == (frames, 80) and frames == S.n_frames(w.shape[0]), name
        o = o[idx]
        assert np.all(np.abs(o - g) <= _fbank_tol(o)), (name, float(np.abs(o - g).max()))


def test_frame_counts():
    assert [S.n_frames(n) for n in (0, 399, 400, 401, 559, 560, 4800, 480000)] == [0, 0, 1, 1, 1, 2, 28, 2998]


# ------------------------------------------------------------------ checkpoint reader
def _save(tmp_path, sd, nested):
    import torch
    state = {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}
    path = tmp_path / ("nested.bin" if nested else "flat.bin")
    torch.save({"state_dict": state, "hyper_parameters": {"sample_rate": 16000}} if nested else state, path)
    return path


@pytest.mark.parametrize("nested", [True, False])
def test_checkpoint_round_trip_and_folding(tmp_path, nested):
    sd = S.random_checkpoint(3)
    assert "resnet.layer2.0.shortcut.1.num_batches_tracked" in sd
    got = S.read_wespeaker_checkpoint(_save(tmp_path, sd, nested))
    assert set(got) == set(S.TENSOR_SHAPES)
    for k, v in got.items():
        assert v.dtype == np.float32 and v.shape == S.TENSOR_SHAPES[k]
    want = S.random_weights(3)
    for k in want:
        assert np.array_equal(got[k], want[k]), k
    # folding BN leaves the network unchanged (float64; the folded weights re-expanded to float64 from the fold's own
    # float64 values, so only the fold's arithmetic is compared)
    x = O.features(synth.speech_like(0.6, seed=5))
    folded64 = {}
    for name, conv, bn in S._checkpoint_convs():
        scale = sd[bn + ".weight"].astype(np.float64) / np.sqrt(sd[bn + ".running_var"].astype(np.float64) + S.BN_EPS)
        folded64[name + ".weight"] = sd[conv + ".weight"].astype(np.float64) * scale[:, None, None, None]
        folded64[name + ".bias"] = sd[bn + ".bias"].astype(np.float64) - sd[bn + ".running_mean"].astype(np.float64) * scale
    folded64["spk.seg_1.weight"] = sd["resnet.seg_1.weight"].astype(np.float64)
    folded64["spk.seg_1.bias"] = sd["resnet.seg_1.bias"].astype(np.float64)
    a, b = O.network(x, sd), O.network(x, folded64)
    assert np.abs(a - b).max() <= 1e-10 * max(1.0, np.abs(a).max())


def test_safetensors_checkpoint(tmp_path):
    from safetensors.numpy import save_file
    sd = {k: np.ascontiguousarray(v) for k, v in S.random_checkpoint(4).items()}
    save_file(sd, str(tmp_path / "m.safetensors"))
    got = S.read_wespeaker_checkpoint(tmp_path / "m.safetensors")
    assert all(np.array_equal(got[k], v) for k, v in S.random_weights(4).items())


def test_checkpoint_rejects_missing_wrong_shape_and_int(tmp_path):
    sd = S.random_checkpoint(1)
    bad = dict(sd)
    del bad["resnet.layer3.5.bn2.running_var"]
    with pytest.raises(S.CheckpointError, match="layer3.5.bn2.running_var"):
        S.read_wespeaker_checkpoint(_save(tmp_path, bad, True))
    bad = dict(sd)
    bad["resnet.layer4.0.shortcut.0.weight"] = np.zeros((256, 128, 3, 3), np.float32)
    with pytest.raises(S.CheckpointError, match="layer4.0.shortcut.0.weight"):
        S.read_wespeaker_checkpoint(_save(tmp_path, bad, False))
    bad = dict(sd)
    bad["resnet.seg_1.bias"] = np.zeros(256, np.int32)
    with pytest.raises(S.CheckpointError, match="seg_1.bias"):
        S.read_wespeaker_checkpoint(_save(tmp_path, bad, False))


def test_resolve_weights_never_falls_back(monkeypatch, tmp_path):
    monkeypatch.delenv("WLB200_SPK_MODEL", raising=False)
    monkeypatch.setenv("HF_HUB_CACHE", str(tmp_path))
    monkeypatch.setenv("HF_HUB_OFFLINE", "1")
    with pytest.raises(RuntimeError, match="WLB200_SPK_MODEL"):
        S.resolve_weights(None)
    path = _save(tmp_path, S.random_checkpoint(2), True)
    monkeypatch.setenv("WLB200_SPK_MODEL", str(path))
    got = S.resolve_weights(None)
    assert all(np.array_equal(got[k], v) for k, v in S.random_weights(2).items())


def test_random_weights_keep_every_stage_in_range():
    w = S.random_weights(0)
    for seed in (1, 2):
        stages = []
        O.network(O.features(synth.speech_like(3.0, seed=seed)), w, stages)
        rms = [float(np.sqrt(np.mean(h ** 2))) for h in stages]
        assert all(0.1 <= r <= 10 for r in rms), rms


# ------------------------------------------------------------------ clustering: the reference's own
def _ref_diarization():
    if not os.path.isdir(REF):
        pytest.skip("reference tree not present")
    sys.path.insert(0, REF)
    try:
        import whisper_live.diarization as D
        import whisperlive_b200.speaker as SP
        if SP._RefDiarizer is None:
            import importlib
            SP = importlib.reload(SP)
    finally:
        sys.path.remove(REF)
    return D, SP


class _FixedScheduler:
    """``embed`` answers with the next injected vector."""

    def __init__(self, vectors):
        self.vectors = list(vectors)
        self.calls = 0

    def embed(self, audio):
        from whisperlive_b200.scheduler import EmbeddingRequest
        r = EmbeddingRequest(audio)
        r.result = self.vectors[self.calls]
        self.calls += 1
        r.future.set()
        return r


def _vectors(n, seed, centres=4, spread=0.35):
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((centres, 256))
    return [(c[rng.integers(centres)] + spread * rng.standard_normal(256)).astype(np.float32) for _ in range(n)]


@pytest.mark.parametrize("max_speakers,names", [(10, None), (2, ["alice", "bob", "carol"])])
def test_device_diarizer_labels_equal_the_reference(max_speakers, names):
    D, SP = _ref_diarization()
    vecs = _vectors(40, seed=max_speakers)
    enrol = _vectors(1, seed=99)[0]
    audio = np.zeros(8000, np.float32)
    ref = D.SpeakerDiarizer(similarity_threshold=0.6, max_speakers=max_speakers, speaker_names=names)
    feed = iter([enrol] + vecs)
    ref._load_model = lambda: None
    ref._model = lambda wf: next(feed)
    dev = SP.DeviceSpeakerDiarizer(_FixedScheduler([enrol] + vecs), similarity_threshold=0.6, max_speakers=max_speakers,
                                   speaker_names=names)
    assert ref.enroll_speaker("host", audio) and dev.enroll_speaker("host", audio)
    want = [ref.identify_speaker(audio) for _ in vecs]
    got = [dev.identify_speaker(audio) for _ in vecs]
    assert got == want and len(set(want)) > 1
    assert ref.identify_speaker(audio[:4000]) is None and dev.identify_speaker(audio[:4000]) is None   # the 0.3 s rule


# ------------------------------------------------------------------ scheduler
class _Transcriber:
    """transcribe_batch blocks until ``release`` is set; speaker_embeddings counts its calls."""

    def __init__(self, fail_marker=None):
        self.release = threading.Event()
        self.entered = threading.Event()
        self.calls = []
        self.fail_marker = fail_marker

    def transcribe_batch(self, audios, kws):
        self.entered.set()
        self.release.wait(10)
        return [([], None) for _ in audios]

    def speaker_embeddings(self, audios):
        self.calls.append(len(audios))
        if self.fail_marker is not None and any(a[0] == self.fail_marker for a in audios):
            raise RuntimeError("embedding failed")
        return np.stack([np.full(256, a[0], np.float32) for a in audios])


def test_scheduler_answers_a_round_of_requests_with_one_call():
    t = _Transcriber()
    sch = RoundScheduler(t, max_batch_size=2, step_tokens=None)
    sch.start()
    try:
        sch.submit(BatchRequest(audio=np.zeros(16000, np.float32), use_vad=False))
        assert t.entered.wait(5)
        got = {}

        def client(i):
            got[i] = sch.embed(np.full(4800, float(i), np.float32)).wait(10)
        threads = [threading.Thread(target=client, args=(i,)) for i in range(5)]
        for th in threads:
            th.start()
        deadline = time.monotonic() + 5
        while len(sch._embeds) < 5 and time.monotonic() < deadline:
            time.sleep(0.01)
        assert len(sch._embeds) == 5 and t.calls == []
        t.release.set()
        for th in threads:
            th.join(10)
        assert t.calls == [5] and sch.embedding_calls == 1
        assert all(np.all(got[i] == i) for i in range(5))
    finally:
        t.release.set()
        sch.stop()


def test_scheduler_answers_an_idle_request_and_isolates_errors():
    t = _Transcriber(fail_marker=-1.0)
    sch = RoundScheduler(t, max_batch_size=2, step_tokens=None)
    sch.start()
    try:
        assert np.all(sch.embed(np.full(4800, 3.0, np.float32)).wait(5) == 3.0)
        bad = sch.embed(np.full(4800, -1.0, np.float32))
        with pytest.raises(RuntimeError, match="embedding failed"):
            bad.wait(5)
        assert np.all(sch.embed(np.full(4800, 4.0, np.float32)).wait(5) == 4.0)
    finally:
        sch.stop()


# ------------------------------------------------------------------ backend switch
class _WS:
    def __init__(self):
        self.sent, self.closed = [], False

    def send(self, msg):
        self.sent.append(msg)

    def close(self):
        self.closed = True


@pytest.mark.parametrize("mode", ["device", None])
def test_backend_swaps_the_diarizer_only_when_asked(monkeypatch, mode):
    D, SP = _ref_diarization()
    sys.path.insert(0, REF)
    try:
        from whisperlive_b200.backend import ServeClientB200
    finally:
        sys.path.remove(REF)
    if mode:
        monkeypatch.setenv("WLB200_DIARIZE", mode)
    else:
        monkeypatch.delenv("WLB200_DIARIZE", raising=False)
    ServeClientB200.MODEL_FACTORY = lambda name: _Transcriber()
    ref = D.SpeakerDiarizer(similarity_threshold=0.42, max_speakers=3, speaker_names=["a", "b"])
    ref.speakers["host"] = np.ones(256, np.float32) / 16
    ref._speaker_count = 1
    client = None
    try:
        client = ServeClientB200(_WS(), client_uid="u0", model="tiny", use_vad=False, diarization=ref)
        got = client.diarization
        if mode is None:
            assert got is ref
        else:
            assert isinstance(got, SP.DeviceSpeakerDiarizer) and isinstance(got, D.SpeakerDiarizer)
            assert got.scheduler is ServeClientB200.BATCH_WORKER
            assert (got.similarity_threshold, got.max_speakers, got.speaker_names) == (0.42, 3, ["a", "b"])
            assert list(got.speakers) == ["host"] and got._speaker_count == 1
    finally:
        if client is not None:
            client.exit = True
            client.trans_thread.join(5)
        ServeClientB200.shutdown()
        ServeClientB200.MODEL_FACTORY = None


# ------------------------------------------------------------------ GPU
def _engine(max_streams=4):
    from whisperlive_b200.config import dims_for
    from whisperlive_b200.engine import B200Whisper
    from whisperlive_b200.weights import random_init
    dims = dims_for("micro.en")
    return B200Whisper(dims, random_init(dims, seed=0), max_streams=max_streams, max_beam=1)


@pytest.fixture(scope="module")
def gpu_engine():
    eng = _engine()
    yield eng
    eng.destroy()


def _conv_ref(x16, frames, H, w16, bias, stride, res16, relu):
    """float64 over the exact fp16 inputs, per stream: out [positions, C_out] and sum |terms| per element."""
    k = int(round(w16.shape[1] ** 0.5))
    W = w16.astype(np.float64).reshape(w16.shape[0], k, k, -1).transpose(0, 3, 1, 2)
    outs, mags, p = [], [], 0
    for T in frames:
        xs = x16[p:p + T * H].astype(np.float64).reshape(T, H, -1).transpose(2, 1, 0)   # [C, H, T]
        p += T * H
        y = O.conv2d(xs, W, bias.astype(np.float64), stride)
        mag = O.conv2d(np.abs(xs), np.abs(W), np.abs(bias.astype(np.float64)), stride)
        outs.append(y.transpose(2, 1, 0).reshape(-1, W.shape[0]))
        mags.append(mag.transpose(2, 1, 0).reshape(-1, W.shape[0]))
    out, mag = np.concatenate(outs), np.concatenate(mags)
    if res16 is not None:
        out = out + res16.astype(np.float64)
        mag = mag + np.abs(res16.astype(np.float64))
    return (np.maximum(out, 0) if relu else out), mag


# every conv shape of the network: (C_in, C_out, k, stride, H_in)
_CONVS = [(32, 32, 3, 1, 80), (32, 64, 3, 2, 80), (32, 64, 1, 2, 80), (64, 64, 3, 1, 40), (64, 128, 3, 2, 40),
          (64, 128, 1, 2, 40), (128, 128, 3, 1, 20), (128, 256, 3, 2, 20), (128, 256, 1, 2, 20), (256, 256, 3, 1, 10)]


def _conv_inputs(kind, frames, H, C, rng):
    n = int(sum(frames)) * H
    if kind == "normal":
        return rng.standard_normal((n, C)).astype(np.float16)
    x = np.zeros((n, C), np.float16)
    if kind == "impulse":
        p = 0
        for T in frames:      # frequency rows 0 and H - 1 of the first and last frame of every stream
            for t in {0, T - 1}:
                x[p + t * H + 0] = 1.0
                x[p + t * H + H - 1] = -2.0
            p += T * H
        return x
    # "fence": stream 1 holds N(0, 1), its neighbours 1e4 -- any read across a stream boundary shows
    p = 0
    for b, T in enumerate(frames):
        x[p:p + T * H] = rng.standard_normal((T * H, C)).astype(np.float16) if b == 1 else np.float16(1e4)
        p += T * H
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("shape", _CONVS, ids=[f"{a}-{b}-k{k}-s{s}-H{h}" for a, b, k, s, h in _CONVS])
def test_spk_conv_every_shape(gpu_engine, shape):
    C_in, C_out, k, stride, H = shape
    rng = np.random.default_rng(C_in * 7 + C_out + k + stride)
    worst = 0.0
    for B, kind in [(1, "normal"), (3, "fence"), (7, "impulse"), (40, "normal")]:
        frames = [1, 2, 3][:B] if B <= 3 else list(rng.integers(1, 12 if B > 7 else 40, size=B))
        if kind == "fence":
            frames = [5, 1, 4]
        x = _conv_inputs(kind, frames, H, C_in, rng)
        w = (rng.standard_normal((C_out, k * k, C_in)) / np.sqrt(k * k * C_in)).astype(np.float16)
        bias = (0.1 * rng.standard_normal(C_out)).astype(np.float32)
        Ho = (H + 1) // 2 if stride == 2 else H
        To = [(t + 1) // 2 if stride == 2 else t for t in frames]
        M = Ho * sum(To)
        for res in (None, rng.standard_normal((M, C_out)).astype(np.float16)):
            got = gpu_engine.test_spk_conv(x, frames, H, w, bias, stride, res=res, relu=True)
            want, mag = _conv_ref(x, frames, H, w, bias, stride, res, True)
            err = np.abs(got.astype(np.float64) - want)
            tol = 2.0 ** -11 * np.abs(want) + 2e-6 * mag + 6e-8
            assert np.all(err <= tol), (B, kind, res is None, float((err / tol).max()))
            worst = max(worst, float((err / tol).max()))
            if B > 1:   # each stream alone is bit-identical to the same stream in the batch
                p = q = 0
                for b, T in enumerate(frames):
                    if b in (0, B // 2, B - 1):
                        alone = gpu_engine.test_spk_conv(x[p:p + T * H], [T], H, w, bias, stride,
                                                         res=None if res is None else res[q:q + Ho * To[b]], relu=True)
                        assert np.array_equal(alone.view(np.uint16), got[q:q + Ho * To[b]].view(np.uint16)), (b, kind)
                    p += T * H
                    q += Ho * To[b]
    print(f"spk_conv {shape}: worst error / tolerance {worst:.3f}")


@pytest.mark.gpu
def test_device_fbank_matches_the_golden_fixture(gpu_engine):
    gold = _golden_fbank()
    waves = _golden_waveforms()
    names = sorted(waves)
    got = gpu_engine.test_spk_fbank([waves[n] for n in names])
    for n, g in zip(names, got):
        frames, idx, want = gold[n]
        assert g.shape == (frames, 80), n
        g = g[idx]
        assert np.all(np.abs(g - want) <= 2 * _fbank_tol(want)), (n, float(np.abs(g - want).max()))


def _cos(a, b):
    return float(np.dot(a, b) / (np.linalg.norm(a) * np.linalg.norm(b)))


# fp16 activations through 36 convs: the embedding keeps a cosine above 0.9999 with float64, and no element moves by
# more than 0.2 % of the vector's largest one (measured on an H100 80GB HBM3 at 700 W: cosine 0.9999999, 4.4e-4)
EMB_REL_MAX = 2e-3


@pytest.mark.gpu
def test_spk_embed_against_the_oracle(gpu_engine):
    w = S.random_weights(0)
    gpu_engine.spk_load(w)
    rng = np.random.default_rng(0)
    secs = [0.3, 45.0] + list(rng.uniform(0.3, 45.0, size=30))
    waves = [synth.speech_like(s, seed=i) if i % 3 else synth.white_noise(s, seed=i, sigma=0.05) for i, s in enumerate(secs)]
    got = gpu_engine.spk_embeddings(waves)
    assert got.shape == (32, 256) and np.all(np.isfinite(got))
    check = [0, 1, 2, 7, 19, 31]
    worst_cos, worst_rel = 1.0, 0.0
    for i in check:
        if secs[i] > 12:     # the float64 oracle over 45 s takes minutes: compare the first 12 s through a second call
            continue
        want = O.embed(waves[i], w)
        worst_cos = min(worst_cos, _cos(got[i], want))
        worst_rel = max(worst_rel, float(np.abs(got[i] - want).max() / np.abs(want).max()))
        alone = gpu_engine.spk_embeddings([waves[i]])[0]
        assert np.array_equal(alone.view(np.uint32), got[i].view(np.uint32)), i
    long_alone = gpu_engine.spk_embeddings([waves[1]])[0]
    assert np.array_equal(long_alone.view(np.uint32), got[1].view(np.uint32))
    cut = waves[1][:12 * 16000]
    g12, want12 = gpu_engine.spk_embeddings([cut])[0], O.embed(cut, w)
    worst_cos = min(worst_cos, _cos(g12, want12))
    worst_rel = max(worst_rel, float(np.abs(g12 - want12).max() / np.abs(want12).max()))
    # one stream and 64 streams (more than max_streams: the workspace grows)
    one = gpu_engine.spk_embeddings([waves[0]])
    assert np.array_equal(one[0].view(np.uint32), got[0].view(np.uint32))
    short = [synth.speech_like(float(s), seed=100 + i) for i, s in enumerate(rng.uniform(0.3, 2.0, size=64))]
    g64 = gpu_engine.spk_embeddings(short)
    for i in (0, 31, 63):
        want = O.embed(short[i], w)
        worst_cos = min(worst_cos, _cos(g64[i], want))
        worst_rel = max(worst_rel, float(np.abs(g64[i] - want).max() / np.abs(want).max()))
    print(f"spk_embed: worst cosine {worst_cos:.7f}, worst max|delta| / max|ref| {worst_rel:.2e}")
    assert worst_cos >= 0.9999 and worst_rel <= EMB_REL_MAX


def _cluster(vectors, threshold, max_speakers=10):
    """SpeakerDiarizer.identify_speaker's rule on given vectors (the CPU test shows DeviceSpeakerDiarizer runs exactly
    the reference's code; the reference package is not installed beside the GPU)."""
    speakers, count, labels = {}, 0, []
    for e in vectors:
        e = e / np.linalg.norm(e)
        best, best_sim = None, -1.0
        for sid, s in speakers.items():
            sim = float(np.dot(e, s))
            if sim > best_sim:
                best, best_sim = sid, sim
        if best_sim >= threshold:
            speakers[best] = speakers[best] * 0.9 + e * 0.1
            speakers[best] /= np.linalg.norm(speakers[best])
            labels.append(best)
        elif len(speakers) >= max_speakers:
            labels.append(best)
        else:
            sid = f"SPEAKER_{count:02d}"
            count += 1
            speakers[sid] = e
            labels.append(sid)
    return labels


@pytest.mark.gpu
def test_diarization_labels_from_device_embeddings_equal_oracle_labels(gpu_engine):
    w = S.random_weights(0)
    gpu_engine.spk_load(w)
    jfk = np.load(os.path.join(GOLDEN, "jfk_16k_i16.npy")).astype(np.float32) / 32768.0
    segs = [jfk[int(a * 16000):int(b * 16000)] for a, b in [(0, 2.5), (2.5, 4.2), (4.2, 7.0), (7.0, 11.0)]]
    for i in range(6):
        segs.append(synth.speech_like(1.0 + 0.4 * i, seed=200 + i % 3))
    dev = gpu_engine.spk_embeddings(segs)
    ora = np.stack([O.embed(s, w) for s in segs])
    dn = dev / np.linalg.norm(dev, axis=1, keepdims=True)
    on = ora / np.linalg.norm(ora, axis=1, keepdims=True)
    sims = np.sort((on @ on.T)[np.triu_indices(len(segs), 1)])
    dev_err = float(np.abs(dn @ dn.T - on @ on.T).max())
    gaps = np.diff(sims)
    j = int(np.argmax(gaps))
    threshold = float((sims[j] + sims[j + 1]) / 2)
    margin = float(gaps[j] / 2)
    print(f"diarization: threshold {threshold:.4f}, margin {margin:.4f}, device similarity error {dev_err:.2e}")
    assert margin > 20 * dev_err
    assert _cluster(list(dev), threshold) == _cluster(list(ora), threshold)


@pytest.mark.gpu
def test_footprint_and_refusals():
    from whisperlive_b200.engine import spk_footprint
    eng = _engine(max_streams=4)
    try:
        before = eng.device_bytes
        launches = eng.kernel_launches()
        with pytest.raises(Exception, match="not loaded"):
            eng.spk_embeddings([synth.speech_like(1.0, seed=1)])
        w = S.random_weights(1)
        eng.spk_load(w)
        with pytest.raises(Exception, match="at least 400"):
            eng.spk_embeddings([synth.speech_like(1.0, seed=1), np.zeros(399, np.float32)])
        assert eng.kernel_launches() == launches
        eng.spk_embeddings([synth.speech_like(2.0, seed=i) for i in range(4)])
        used = eng.device_bytes - before
        est = spk_footprint(4)
        print(f"speaker footprint: estimate {est} B, allocated {used} B")
        assert used <= est <= 1.10 * used
        with pytest.raises(Exception, match="unknown"):
            eng.spk_load({"spk.nope": np.zeros(3, np.float32)})
        with pytest.raises(Exception, match="must have shape"):
            eng.spk_load({"spk.seg_1.bias": np.zeros(255, np.float32)})
    finally:
        eng.destroy()
