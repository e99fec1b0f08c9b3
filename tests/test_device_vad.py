"""Silero VAD on the device (whisperlive_b200/vad.py, csrc/vad.cu): the ONNX reader, the float64 oracle's frame protocol,
the host gating restatement, the transcriber's batched VAD call, and on the GPU wl_vad against the oracle."""
import ctypes as C

import numpy as np
import pytest

from tests import vad_oracle
from whisperlive_b200 import synth
from whisperlive_b200.vad import (TENSOR_SHAPES, DeviceVad, OnnxError, VadOptions, n_frames, random_weights,
                                  read_silero_onnx, speech_timestamps_from_probs)


# ------------------------------------------------------------------ a test-side ONNX writer (protobuf wire format)
def _varint(v):
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _ld(field, payload):
    return _varint(field << 3 | 2) + _varint(len(payload)) + payload


def _vi(field, v):
    return _varint(field << 3) + _varint(v)


def _tensor(name, a, enc="raw", dtype=1):
    b = b"".join(_vi(1, d) for d in a.shape) + _vi(2, dtype) + _ld(8, name.encode())
    if dtype == 7:
        return b + _ld(9, np.asarray(a, "<i8").tobytes())
    if enc == "raw":
        return b + _ld(9, np.asarray(a, "<f4").tobytes())
    return b + _ld(4, np.asarray(a, "<f4").tobytes())      # packed float_data


def _node(op, inputs, outputs, attrs=b""):
    return b"".join(_ld(1, i.encode()) for i in inputs) + b"".join(_ld(2, o.encode()) for o in outputs) + \
        _ld(4, op.encode()) + attrs


def _attr_tensor(name, t):
    return _ld(5, _ld(1, name.encode()) + _ld(5, t) + _vi(20, 4))


def _attr_graph(name, g):
    return _ld(5, _ld(1, name.encode()) + _ld(6, g) + _vi(20, 5))


def _graph(nodes, inits):
    return b"".join(_ld(1, n) for n in nodes) + b"".join(_ld(5, t) for t in inits)


def _model(graph):
    return _vi(1, 8) + _ld(7, graph)


_ONNX_GATES = [0, 3, 1, 2]     # PyTorch blocks i, f, g, o -> ONNX i, o, f, c


def _to_onnx_gates(a):
    blocks = np.split(a, 4, axis=0)
    return np.concatenate([blocks[k] for k in _ONNX_GATES], axis=0)


def _network(w, prefix="", enc="raw", as_constants=False, lstm="named", dtype_override=None, drop=(), shape_override=None,
             part="all"):
    """(nodes, initializers) of a Silero-shaped graph over the weights w (vad.* names); part = "encoder" (the STFT and
    the convs), "decoder" (the LSTM and the output conv) or "all"."""
    tensors = {}
    convs = [("stft", "vad.stft.basis", None), ("c0", "vad.conv0.weight", "vad.conv0.bias"),
             ("c1", "vad.conv1.weight", "vad.conv1.bias"), ("c2", "vad.conv2.weight", "vad.conv2.bias"),
             ("c3", "vad.conv3.weight", "vad.conv3.bias")]
    nodes, x = [], prefix + "input"
    for tag, wn, bn in convs:
        ins = [x, prefix + wn]
        tensors[prefix + wn] = w[wn]
        if bn:
            ins.append(prefix + bn)
            tensors[prefix + bn] = w[bn]
        nodes.append(_node("Conv", ins, [prefix + tag]))
        x = prefix + tag
    if lstm == "named":
        for k in ("weight_ih", "bias_ih", "weight_hh", "bias_hh"):
            tensors[f"{prefix}decoder.rnn.{k}"] = w[f"vad.lstm.{k}"]
        nodes.append(_node("Gemm", [x, prefix + "decoder.rnn.weight_ih", prefix + "decoder.rnn.bias_ih"], [prefix + "gi"]))
        nodes.append(_node("Gemm", ["h", prefix + "decoder.rnn.weight_hh", prefix + "decoder.rnn.bias_hh"], [prefix + "gh"]))
        x = prefix + "h_new"
    elif lstm == "anonymous":     # no telling names: the graph consumes W_ih / b_ih first
        tensors[prefix + "m1"] = w["vad.lstm.weight_ih"]
        tensors[prefix + "b1"] = w["vad.lstm.bias_ih"]
        tensors[prefix + "m2"] = w["vad.lstm.weight_hh"]
        tensors[prefix + "b2"] = w["vad.lstm.bias_hh"]
        nodes.append(_node("Gemm", [x, prefix + "m1", prefix + "b1"], [prefix + "gi"]))
        nodes.append(_node("Gemm", ["h", prefix + "m2", prefix + "b2"], [prefix + "gh"]))
        x = prefix + "h_new"
    else:                         # the ONNX LSTM op: W / R / B in its own gate order
        tensors[prefix + "W"] = _to_onnx_gates(w["vad.lstm.weight_ih"])[None]
        tensors[prefix + "R"] = _to_onnx_gates(w["vad.lstm.weight_hh"])[None]
        tensors[prefix + "B"] = np.concatenate([_to_onnx_gates(w["vad.lstm.bias_ih"]),
                                                _to_onnx_gates(w["vad.lstm.bias_hh"])])[None]
        nodes.append(_node("LSTM", [x, prefix + "W", prefix + "R", prefix + "B"], [prefix + "y"]))
        x = prefix + "y"
    tensors[prefix + "out.w"] = w["vad.out.weight"]
    tensors[prefix + "out.b"] = w["vad.out.bias"]
    nodes.append(_node("Conv", [x, prefix + "out.w", prefix + "out.b"], [prefix + "logit"]))
    if part != "all":
        enc_names = {prefix + k for k in ("vad.stft.basis", "vad.conv0.weight", "vad.conv0.bias", "vad.conv1.weight",
                                          "vad.conv1.bias", "vad.conv2.weight", "vad.conv2.bias", "vad.conv3.weight",
                                          "vad.conv3.bias")}
        keep = (lambda k: k in enc_names) if part == "encoder" else (lambda k: k not in enc_names)
        tensors = {k: v for k, v in tensors.items() if keep(k)}
        nodes = nodes[:5] if part == "encoder" else nodes[5:]
    tensors = {k: v for k, v in tensors.items() if k[len(prefix):] not in drop}
    nodes = [n for n in nodes if not any(d.encode() in n for d in drop)]
    if shape_override:
        for k, shape in shape_override.items():
            tensors[prefix + k] = np.zeros(shape, np.float32)
    inits = []
    for k, v in tensors.items():
        dt = (dtype_override or {}).get(k[len(prefix):], 1)
        t = _tensor(k, np.asarray(v), enc=enc, dtype=dt)
        if as_constants:
            nodes.insert(0, _node("Constant", [], [k], _attr_tensor("value", t)))
        else:
            inits.append(t)
    return nodes, inits


def _weights_8k(seed=7):
    rng = np.random.default_rng(seed)
    return {"basis8": rng.standard_normal((130, 1, 128)).astype(np.float32),
            "conv0_8": rng.standard_normal((128, 65, 3)).astype(np.float32),
            "conv1_8": rng.standard_normal((64, 128, 3)).astype(np.float32),
            "conv1_8b": rng.standard_normal(64).astype(np.float32)}


def _graph_8k():
    w = _weights_8k()
    nodes = [_node("Conv", ["input", "basis8"], ["s8"]), _node("Conv", ["s8", "conv0_8"], ["a8"]),
             _node("Conv", ["a8", "conv1_8", "conv1_8b"], ["b8"])]
    return _graph(nodes, [_tensor(k, v) for k, v in w.items()])


def _write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


def _same(got, want):
    assert set(got) == set(TENSOR_SHAPES)
    for k in TENSOR_SHAPES:
        assert got[k].shape == TENSOR_SHAPES[k], k
        np.testing.assert_array_equal(got[k], want[k].astype(np.float32), err_msg=k)


# ------------------------------------------------------------------ CPU: ONNX reader
@pytest.mark.parametrize("enc", ["raw", "float_data"])
@pytest.mark.parametrize("lstm", ["named", "anonymous", "onnx_op"])
def test_onnx_reader_top_level_initializers(tmp_path, enc, lstm):
    w = random_weights(seed=1)
    nodes, inits = _network(w, enc=enc, lstm=lstm)
    _same(read_silero_onnx(_write(tmp_path, "m.onnx", _model(_graph(nodes, inits)))), w)


@pytest.mark.parametrize("enc", ["raw", "float_data"])
def test_onnx_reader_if_branches_skip_the_8k_network(tmp_path, enc):
    """The 16 kHz network inside one If branch, the 8 kHz one (its [130, 1, 128] basis, conv shapes shared with the
    16 kHz network) inside the other: only the 16 kHz tensors are taken."""
    w = random_weights(seed=2)
    nodes, inits = _network(w, prefix="b16/", enc=enc)
    then_g = _graph(nodes, inits)
    top = _graph([_node("If", ["is_16k"], ["out"], _attr_graph("then_branch", then_g) + _attr_graph("else_branch", _graph_8k()))],
                 [])
    _same(read_silero_onnx(_write(tmp_path, "m.onnx", _model(top))), w)


def test_onnx_reader_constant_nodes_and_two_files(tmp_path):
    """Weights as Constant node values, split over an encoder file and a decoder file (as faster-whisper ships them)."""
    w = random_weights(seed=3, basis="random")
    p1 = _write(tmp_path, "enc.onnx", _model(_graph(*_network(w, as_constants=True, part="encoder"))))
    p2 = _write(tmp_path, "dec.onnx", _model(_graph(*_network(w, as_constants=True, lstm="onnx_op", part="decoder"))))
    _same(read_silero_onnx([p1, p2]), w)


def test_onnx_reader_rejects_a_missing_tensor(tmp_path):
    w = random_weights(seed=4)
    nodes, inits = _network(w, drop=("out.w", "out.b"))
    with pytest.raises(OnnxError, match=r"missing vad\.out\.weight, vad\.out\.bias; tensors found: .*\[258, 1, 256\]"):
        read_silero_onnx(_write(tmp_path, "m.onnx", _model(_graph(nodes, inits))))


def test_onnx_reader_rejects_a_wrong_shape(tmp_path):
    w = random_weights(seed=5)
    nodes, inits = _network(w, shape_override={"vad.conv0.weight": (128, 129, 2)})
    with pytest.raises(OnnxError, match=r"Conv weight 'vad\.conv0\.weight' has shape \[128, 129, 2\], which no role"):
        read_silero_onnx(_write(tmp_path, "m.onnx", _model(_graph(nodes, inits))))


def test_onnx_reader_rejects_a_non_float_dtype(tmp_path):
    w = random_weights(seed=6)
    w["vad.conv0.bias"] = np.arange(128)
    nodes, inits = _network(w, dtype_override={"vad.conv0.bias": 7})
    with pytest.raises(OnnxError, match=r"'vad\.conv0\.bias' \[128\] has dtype int64"):
        read_silero_onnx(_write(tmp_path, "m.onnx", _model(_graph(nodes, inits))))


def test_onnx_reader_rejects_a_truncated_file(tmp_path):
    w = random_weights(seed=7)
    data = _model(_graph(*_network(w)))
    with pytest.raises(OnnxError, match="truncated ONNX data"):
        read_silero_onnx(_write(tmp_path, "m.onnx", data[:len(data) // 2]))


# ------------------------------------------------------------------ CPU: the oracle's frame protocol
def test_frame_counts_and_the_extra_frame():
    assert [n_frames(n) for n in (0, 1, 511, 512, 513, 1023, 1024, 1025)] == [0, 1, 1, 2, 2, 2, 3, 3]
    x = vad_oracle.frame_inputs(np.ones(1024, np.float32))
    assert x.shape == (3, 576)
    np.testing.assert_array_equal(x[2, 64:], 0.0)       # the whole frame of zeros after an aligned length,
    np.testing.assert_array_equal(x[2, :64], 1.0)       # behind the real context of the last full frame


def test_first_frame_context_is_zeros():
    a = synth.speech_like(0.2, seed=3)
    x = vad_oracle.frame_inputs(a)
    np.testing.assert_array_equal(x[0, :64], 0.0)
    np.testing.assert_array_equal(x[0, 64:], a[:512])
    np.testing.assert_array_equal(x[1, :64], a[448:512])


@pytest.mark.parametrize("n", [511, 512, 513, 4000])
def test_whole_stream_equals_the_frame_loop(n):
    """One call over the stream equals 512 samples at a time with h, c and the context carried between calls, as
    whisper_live/vad.py:74-86 feeds the model."""
    w = random_weights(seed=8)
    a = synth.speech_like(n / 16000, seed=n)
    whole = vad_oracle.probs(a, w)
    loop = vad_oracle.FrameLoop(w)
    padded = np.zeros(n_frames(n) * 512)
    padded[:n] = a
    step = np.array([loop(padded[i:i + 512]) for i in range(0, padded.shape[0], 512)])
    assert whole.shape == (n_frames(n),)
    np.testing.assert_allclose(whole, step, rtol=0, atol=1e-12)


# ------------------------------------------------------------------ CPU: the gating restatement
def _gate(probs, frames_total, **opts):
    return speech_timestamps_from_probs(np.asarray(probs, np.float64), frames_total * 512, VadOptions(**opts))


def test_gating_threshold_and_neg_threshold_hysteresis():
    p = [0.1, 0.6, 0.4, 0.4, 0.2, 0.2, 0.2, 0.2, 0.2, 0.2]
    base = dict(min_silence_duration_ms=0, speech_pad_ms=0)
    # neg_threshold defaults to threshold - 0.15: the 0.4 frames stay speech
    assert _gate(p, 10, threshold=0.5, **base) == [{"start": 512, "end": 2048}]
    assert _gate(p, 10, threshold=0.5, neg_threshold=0.45, **base) == [{"start": 512, "end": 1024}]


def test_gating_min_speech_duration():
    p = [0.9, 0.9, 0.1, 0.1, 0.1, 0.1]    # 1024 samples of speech = 64 ms
    base = dict(min_silence_duration_ms=0, speech_pad_ms=0)
    assert _gate(p, 6, min_speech_duration_ms=100, **base) == []
    assert _gate(p, 6, min_speech_duration_ms=50, **base) == [{"start": 0, "end": 1024}]


_TWO_BURSTS = [0.9, 0.9, 0.9, 0.1, 0.1, 0.9, 0.9, 0.9] + [0.1] * 8


def test_gating_min_silence_duration():
    # 2 frames (64 ms) of silence: bridged at 100 ms, a boundary at 30 ms
    assert _gate(_TWO_BURSTS, 16, min_silence_duration_ms=100, speech_pad_ms=0) == [{"start": 0, "end": 4096}]
    assert _gate(_TWO_BURSTS, 16, min_silence_duration_ms=30, speech_pad_ms=0) == [{"start": 0, "end": 1536},
                                                                                  {"start": 2560, "end": 4096}]


def test_gating_speech_pad():
    # gap 1024 >= 2 x 320: each side padded by 320; gap 1024 < 2 x 640: split in the middle, the ends padded by 640
    assert _gate(_TWO_BURSTS, 16, min_silence_duration_ms=30, speech_pad_ms=20) == [{"start": 0, "end": 1856},
                                                                                   {"start": 2240, "end": 4416}]
    assert _gate(_TWO_BURSTS, 16, min_silence_duration_ms=30, speech_pad_ms=40) == [{"start": 0, "end": 2048},
                                                                                   {"start": 2048, "end": 4736}]


def test_gating_max_speech_duration_cuts_where_the_limit_is_reached():
    # max_speech_samples = 0.352 s x 16000 - 512 = 10 frames: no silence to split at, so cut at frames 11 and 23
    p = [0.9] * 30 + [0.1] * 4
    got = _gate(p, 34, max_speech_duration_s=11 * 512 / 16000, min_silence_duration_ms=0, speech_pad_ms=0)
    assert got == [{"start": 0, "end": 5632}, {"start": 6144, "end": 11776}, {"start": 12288, "end": 15360}]


def test_gating_max_speech_duration_splits_at_the_last_long_silence():
    # 5 silent frames (160 ms > 98 ms) inside speech: the chunk that reaches 20 frames ends where that silence began,
    # and the next one starts where speech resumed; the second chunk then reaches the limit with no silence and is cut
    p = [0.9] * 5 + [0.1] * 5 + [0.9] * 20 + [0.1] * 20
    got = _gate(p, 50, max_speech_duration_s=21 * 512 / 16000, min_silence_duration_ms=2000, speech_pad_ms=0)
    assert got == [{"start": 0, "end": 2560}, {"start": 5120, "end": 15872}]


# ------------------------------------------------------------------ CPU: the transcriber's batched call
def _gapped(seconds, seed):
    a = synth.speech_like(seconds, seed=seed)
    a[int(0.35 * a.shape[0]):int(0.6 * a.shape[0])] = 0.0
    return a


def _clear(probs, target):
    """A threshold near ``target`` as far as the probabilities near it allow from every frame's probability: the middle
    of the widest gap among the 20 sorted values around ``target``."""
    p = np.sort(np.asarray(probs, np.float64))
    i = int(np.searchsorted(p, target))
    lo, hi = max(0, i - 10), min(p.size - 1, i + 10)
    j = lo + int(np.argmax(np.diff(p[lo:hi + 1])))
    return float((p[j] + p[j + 1]) / 2)


def _median_kw(w, audio):
    """Gating at the stream's median probability (chunks that depend on the probabilities), with both thresholds
    clear of every frame's probability so that fp32 and float64 probabilities take the same side."""
    p = vad_oracle.probs(audio, w)
    thr = _clear(p, float(np.median(p)))
    neg = _clear(p, float(np.quantile(p, 0.3)))     # random weights keep the probabilities in a narrow band
    return dict(language="en", vad_filter=True, temperature=0.0,
                vad_parameters=dict(threshold=thr, neg_threshold=min(neg, thr), min_silence_duration_ms=200,
                                    speech_pad_ms=100))


class _PerStreamModule:
    """The ``faster_whisper.vad`` interface without ``speech_timestamps_batch``: the transcriber's per-stream path."""

    def __init__(self, dv):
        self.dv = dv
        self.VadOptions, self.collect_chunks, self.SpeechTimestampsMap = dv.VadOptions, dv.collect_chunks, dv.SpeechTimestampsMap

    def get_speech_timestamps(self, audio, vad_options=None, sampling_rate=16000, **kw):
        return self.dv.get_speech_timestamps(audio, vad_options, sampling_rate, **kw)


def test_transcriber_batches_the_vad_and_matches_the_per_stream_module():
    from tests.test_boundary_cpu import _oracle_model
    w = random_weights(seed=9)
    audios = [_gapped(4.0, 11), _gapped(5.5, 12), synth.silence(1.0), _gapped(3.0, 13)]
    kws = [_median_kw(w, a) for a in audios]
    kws[2] = dict(language="en", vad_filter=True, temperature=0.0)
    kws[3]["vad_filter"] = False                  # not gated: never reaches the VAD

    eng = vad_oracle.OracleVadEngine()
    batched = _oracle_model()
    batched._vad = DeviceVad(eng, weights=w)
    eng_ref = vad_oracle.OracleVadEngine()
    single = _oracle_model()
    single._vad = _PerStreamModule(DeviceVad(eng_ref, weights=w))

    got = batched.transcribe_batch(audios, [dict(k) for k in kws])
    ref = single.transcribe_batch(audios, [dict(k) for k in kws])
    assert eng.calls == [3]                       # one probability call for the three gated streams
    assert eng_ref.calls == [1, 1, 1]
    for (gs, gi), (rs, ri) in zip(got, ref):
        if ri is None:
            assert gi is None
            continue
        assert gi.vad_options == ri.vad_options
        assert gi.duration_after_vad == ri.duration_after_vad
        assert [(s.start, s.end, s.text, list(s.tokens)) for s in gs] == [(s.start, s.end, s.text, list(s.tokens)) for s in rs]
    assert got[0][1].duration_after_vad < got[0][1].duration     # the gating removed audio


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


# fp32 against float64: every sum of the front end and the recurrence runs in fp32 with its own summation order (the
# STFT's 256 terms, conv sums of up to 387 terms, 128-term gate dot products accumulated in four partial sums), which
# leaves the gates within ~1e-6 relative; through the sigmoid (slope <= 1/4) that is well under 1e-5 in probability.
TOL = 1e-5
_LENGTHS = [0, 1, 511, 512, 513, 5 * 16000, 30 * 16000, 45 * 16000]


def _wave(n, seed):
    if n == 0:
        return np.zeros(0, np.float32)
    kind = seed % 3
    if kind == 0:
        return synth.speech_like(n / 16000, seed=seed)
    if kind == 1:
        return synth.white_noise(n / 16000, seed=seed, sigma=0.05)
    a = synth.speech_like(n / 16000, seed=seed)
    a[: n // 3] = 0.0
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("basis", ["dft", "random"])
def test_wl_vad_matches_the_float64_oracle(gpu_engine, basis):
    w = random_weights(seed=21, basis=basis)
    gpu_engine.vad_load(w)
    waves = [_wave(n, seed=i) for i, n in enumerate(_LENGTHS)]
    got = gpu_engine.vad_probs(waves)
    worst = 0.0
    for a, g in zip(waves, got):
        ref = vad_oracle.probs(a, w)
        assert g.shape == ref.shape == (n_frames(a.shape[0]),)
        if ref.size:
            worst = max(worst, float(np.abs(g - ref).max()))
    print(f"basis={basis}: max |dp| = {worst:.2e}")
    assert worst <= TOL


@pytest.mark.gpu
def test_wl_vad_32_mixed_streams_one_call(gpu_engine):
    """32 streams of ragged lengths in one call: every frame within the tolerance of the oracle, every frame written and
    nothing past the last one, and each stream bit-identical to the same stream alone."""
    from whisperlive_b200 import _lib
    w = random_weights(seed=22)
    gpu_engine.vad_load(w)
    rng = np.random.default_rng(5)
    lens = [int(x) for x in rng.integers(0, 30 * 16000, 32)]
    lens[:6] = [0, 1, 511, 512, 513, 30 * 16000]
    waves = [_wave(n, seed=100 + i) for i, n in enumerate(lens)]
    off = np.zeros(33, np.int64)
    off[1:] = np.cumsum(lens)
    poff = np.zeros(33, np.int64)
    poff[1:] = np.cumsum([n_frames(n) for n in lens])
    pcm = np.concatenate(waves).astype(np.float32)
    out = np.full(int(poff[-1]) + 64, np.nan, np.float32)
    lib = gpu_engine.lib
    rc = lib.wl_vad(gpu_engine.ctx, _lib.ptr(pcm, C.c_float), _lib.ptr(off, C.c_int64), 32, _lib.ptr(out, C.c_float),
                    _lib.ptr(poff, C.c_int64))
    _lib.check(lib, gpu_engine.ctx, rc, "wl_vad")
    assert not np.isnan(out[:poff[-1]]).any()
    assert np.isnan(out[poff[-1]:]).all()
    worst = 0.0
    for i, a in enumerate(waves):
        g = out[poff[i]:poff[i + 1]]
        alone = gpu_engine.vad_probs([a])[0]
        assert g.tobytes() == alone.tobytes(), i
        if g.size:
            worst = max(worst, float(np.abs(g - vad_oracle.probs(a, w)).max()))
    print(f"32 streams: max |dp| = {worst:.2e}")
    assert worst <= TOL


@pytest.mark.gpu
def test_wl_vad_refuses_missing_weights_and_wrong_shapes():
    from whisperlive_b200._lib import WlError
    eng = _engine()
    try:
        with pytest.raises(WlError, match=r"VAD weights not loaded: 'vad\.stft\.basis' is missing"):
            eng.vad_probs([np.zeros(1000, np.float32)])
        with pytest.raises(WlError, match=r"'vad\.conv0\.weight' must have shape \[128, 129, 3\]"):
            eng.vad_load({"vad.conv0.weight": np.zeros((128, 129, 2), np.float32)})
        with pytest.raises(WlError, match="unknown VAD tensor"):
            eng.vad_load({"vad.conv9.weight": np.zeros((1,), np.float32)})
    finally:
        eng.destroy()


def _first_diff(a, b):
    return next((i for i, (x, y) in enumerate(zip(a, b)) if x != y), None)


@pytest.mark.gpu
def test_gating_on_device_probabilities_equals_gating_on_oracle_probabilities(gpu_engine):
    """At threshold 0.5 and at each stream's median probability (many frames near the threshold).  A boundary may
    differ only where the deciding frame's oracle probability lies within the tolerance of a threshold."""
    w = random_weights(seed=23)
    gpu_engine.vad_load(w)
    waves = [_wave(n, seed=200 + i) for i, n in enumerate([5 * 16000, 12 * 16000, 30 * 16000, 45 * 16000])]
    got = gpu_engine.vad_probs(waves)
    for a, g in zip(waves, got):
        ref = vad_oracle.probs(a, w)
        for thr in (0.5, float(np.median(ref))):
            opts = VadOptions(threshold=thr, min_silence_duration_ms=100, speech_pad_ms=30)
            neg = max(thr - 0.15, 0.01)
            cg = speech_timestamps_from_probs(g, a.shape[0], opts)
            cr = speech_timestamps_from_probs(ref, a.shape[0], opts)
            if cg == cr:
                continue
            # the first frame where the two sequences take different sides of a threshold decides it
            sides_g = [(p >= thr, p < neg) for p in g]
            sides_r = [(p >= thr, p < neg) for p in ref]
            i = _first_diff(sides_g, sides_r)
            assert i is not None, "different chunks from identical threshold decisions"
            margin = min(abs(ref[i] - thr), abs(ref[i] - neg))
            print(f"boundary differs at frame {i}: oracle p={ref[i]:.7f} device p={g[i]:.7f} threshold={thr:.7f}")
            assert margin <= TOL


@pytest.mark.gpu
def test_transcribe_batch_with_device_vad_matches_the_oracle_module():
    from whisperlive_b200.transcriber import B200WhisperModel
    m = B200WhisperModel("tiny.en", weights="random", seed=0, hf_tokenizer="synthetic", max_streams=4, vad="device")
    try:
        w = random_weights(seed=0)     # what vad="device" loads with weights="random", seed=0
        audios = [_gapped(6.0, 31), _gapped(9.0, 32), _gapped(4.0, 33)]
        kws = [_median_kw(w, a) for a in audios]
        got = m.transcribe_batch(audios, [dict(k) for k in kws])
        dv = m._vad
        m._vad = DeviceVad(vad_oracle.OracleVadEngine(), weights=w)
        ref = m.transcribe_batch(audios, [dict(k) for k in kws])
        m._vad = dv
        for (gs, gi), (rs, ri) in zip(got, ref):
            assert (gi is None) == (ri is None)
            if gi is None:
                continue
            assert gi.duration_after_vad == ri.duration_after_vad
            assert [(s.start, s.end, list(s.tokens)) for s in gs] == [(s.start, s.end, list(s.tokens)) for s in rs]
        assert any(gi is not None and gi.duration_after_vad < gi.duration for _gs, gi in got)
    finally:
        m.destroy()


@pytest.mark.gpu
def test_footprint_estimate_with_vad():
    from whisperlive_b200.engine import footprint_estimate
    from whisperlive_b200.transcriber import B200WhisperModel
    m = B200WhisperModel("tiny.en", weights="random", seed=0, hf_tokenizer="synthetic", max_streams=8, vad="device")
    eng = m.model
    try:
        sess = m.open_session()
        waves = [synth.speech_like(6.0 + i, seed=80 + i) for i in range(8)]
        sess.add_streams(waves, [dict(language="en", vad_filter=True, vad_parameters=dict(threshold=0.0)) for _ in waves])
        sess.step_round(16)
        measured = eng.device_bytes
        sess.close()
        est = footprint_estimate(eng.dims, max_streams=8, max_beam=5, vad=True)
        assert measured <= est <= 1.10 * measured, (est, measured, est / measured)
        assert est - footprint_estimate(eng.dims, max_streams=8, max_beam=5) > 8 * 30 * 16000 * 4
    finally:
        m.destroy()
