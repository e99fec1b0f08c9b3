"""Silero VAD on the device behind the ``faster_whisper.vad`` interface.

The reference gates every default chunk with faster-whisper's CPU Silero model, once per stream
(transcriber_faster_whisper.py:830-838).  ``DeviceVad`` computes the same network's per-frame speech probabilities with
``wl_vad`` (csrc/vad.cu, fp32) for all streams of a round in one call, and turns them into speech chunks with a host
restatement of faster-whisper 1.2.0's ``get_speech_timestamps`` state machine: the options and the gating rules are
unchanged, only the probabilities move to the GPU.

Weights come from the ONNX file(s) of the model (a hand-written reader: ``onnx`` is not a dependency), from
``WLB200_VAD_MODEL=<path>[:<path>...]``, or from faster-whisper's bundled asset when ``faster_whisper`` is importable.
Nothing is downloaded.  ``weights="random"`` is the explicit opt-in for tests and tools.

The frame protocol is recalled from upstream (neither the network nor faster-whisper's wrapper is in the reference
tree; whisper_live/vad.py:56-91 shows the 576-sample input with 64 samples of context and the [2, B, 128] state).  Every
recalled detail is named below, once; the kernel restates them and tests/golden/capture_silero_vad.py records the
reference's own outputs to check them against."""
from __future__ import annotations

import bisect
import glob
import os
import struct
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np

# ---------------------------------------------------------------------------------------------- the recalled protocol
SAMPLING_RATE = 16000
FRAME_SAMPLES = 512                 # new samples per frame
CONTEXT_SAMPLES = 64                # the previous frame's last samples in front of each frame (zeros for frame 0)
STFT_REFLECT_PAD = ("right", 64)    # reflection pad of the 576-sample input before the STFT conv (basis [258, 1, 256], stride 128)
EXTRA_FRAME_WHEN_ALIGNED = True     # faster-whisper pads by 512 - n % 512: a whole frame of zeros when n % 512 == 0
LSTM_GATE_ORDER = "ifgo"            # PyTorch LSTMCell; an ONNX LSTM op stores i, o, f, c and is permuted on load
HIDDEN = 128

# name -> shape of every tensor wl_vad_load_tensor takes
TENSOR_SHAPES: Dict[str, Tuple[int, ...]] = {
    "vad.stft.basis": (258, 1, 256),
    "vad.conv0.weight": (128, 129, 3), "vad.conv0.bias": (128,),
    "vad.conv1.weight": (64, 128, 3), "vad.conv1.bias": (64,),
    "vad.conv2.weight": (64, 64, 3), "vad.conv2.bias": (64,),
    "vad.conv3.weight": (128, 64, 3), "vad.conv3.bias": (128,),
    "vad.lstm.weight_ih": (512, 128), "vad.lstm.weight_hh": (512, 128),
    "vad.lstm.bias_ih": (512,), "vad.lstm.bias_hh": (512,),
    "vad.out.weight": (1, 128, 1), "vad.out.bias": (1,),
}
_CONV_ROLES = {(258, 1, 256): "vad.stft", (128, 129, 3): "vad.conv0", (64, 128, 3): "vad.conv1", (64, 64, 3): "vad.conv2",
               (128, 64, 3): "vad.conv3", (1, 128, 1): "vad.out"}
_BASIS_8K = (130, 1, 128)


def n_frames(n_samples: int) -> int:
    """Frames the model sees for ``n_samples`` of audio (0 for empty audio)."""
    if n_samples <= 0:
        return 0
    if n_samples % FRAME_SAMPLES == 0:
        return n_samples // FRAME_SAMPLES + (1 if EXTRA_FRAME_WHEN_ALIGNED else 0)
    return n_samples // FRAME_SAMPLES + 1


# ---------------------------------------------------------------------------------------------- ONNX reader
class OnnxError(ValueError):
    pass


_ONNX_FLOAT, _ONNX_DOUBLE = 1, 11
_ONNX_TYPES = {1: "float", 2: "uint8", 3: "int8", 5: "int16", 6: "int32", 7: "int64", 9: "bool", 10: "float16",
               11: "double", 16: "bfloat16"}


def _fields(buf: bytes, what: str):
    """Protobuf wire format: yields (field number, wire type, value); value is an int or a bytes slice."""
    i, n = 0, len(buf)

    def varint():
        nonlocal i
        v, shift = 0, 0
        while True:
            if i >= n:
                raise OnnxError(f"truncated ONNX data inside {what}")
            b = buf[i]
            i += 1
            v |= (b & 0x7F) << shift
            if b < 0x80:
                return v
            shift += 7
            if shift > 63:
                raise OnnxError(f"malformed varint inside {what}")

    while i < n:
        key = varint()
        fno, wt = key >> 3, key & 7
        if wt == 0:
            yield fno, wt, varint()
        elif wt == 1 or wt == 5:
            size = 8 if wt == 1 else 4
            if i + size > n:
                raise OnnxError(f"truncated ONNX data inside {what}")
            yield fno, wt, buf[i:i + size]
            i += size
        elif wt == 2:
            size = varint()
            if i + size > n:
                raise OnnxError(f"truncated ONNX data inside {what}")
            yield fno, wt, buf[i:i + size]
            i += size
        else:
            raise OnnxError(f"unsupported protobuf wire type {wt} inside {what}")


@dataclass
class _Tensor:
    name: str
    dims: Tuple[int, ...]
    dtype: int
    raw: Optional[bytes]
    floats: List[float]

    def array(self) -> np.ndarray:
        if self.dtype not in (_ONNX_FLOAT, _ONNX_DOUBLE):
            raise OnnxError(f"tensor {self.name!r} {list(self.dims)} has dtype {_ONNX_TYPES.get(self.dtype, self.dtype)}; "
                            "the VAD weights must be float")
        count = int(np.prod(self.dims)) if self.dims else 1
        if self.raw is not None:
            dt = np.float32 if self.dtype == _ONNX_FLOAT else np.float64
            if len(self.raw) != count * np.dtype(dt).itemsize:
                raise OnnxError(f"tensor {self.name!r}: raw_data holds {len(self.raw)} bytes for shape {list(self.dims)}")
            a = np.frombuffer(self.raw, dtype="<" + np.dtype(dt).str[1:])
        else:
            if len(self.floats) != count:
                raise OnnxError(f"tensor {self.name!r}: {len(self.floats)} values for shape {list(self.dims)}")
            a = np.asarray(self.floats, dtype=np.float64)
        return a.astype(np.float32).reshape(self.dims)


def _tensor(buf: bytes) -> _Tensor:
    name, dims, dtype, raw, floats = "", [], 0, None, []
    for f, wt, v in _fields(buf, "a TensorProto"):
        if f == 1:
            if wt == 2:
                dims.extend(_packed_varints(v))
            else:
                dims.append(v)
        elif f == 2:
            dtype = v
        elif f == 4:      # float_data, packed or not
            floats.extend(struct.unpack(f"<{len(v) // 4}f", v) if wt == 2 else struct.unpack("<f", v))
        elif f == 10:     # double_data
            floats.extend(struct.unpack(f"<{len(v) // 8}d", v) if wt == 2 else struct.unpack("<d", v))
        elif f == 8:
            name = bytes(v).decode()
        elif f == 9:
            raw = bytes(v)
    return _Tensor(name, tuple(int(d) for d in dims), dtype, raw, floats)


def _packed_varints(buf: bytes) -> List[int]:
    out, i, n = [], 0, len(buf)
    while i < n:
        v, shift = 0, 0
        while True:
            if i >= n:
                raise OnnxError("truncated packed varint")
            b = buf[i]
            i += 1
            v |= (b & 0x7F) << shift
            if b < 0x80:
                break
            shift += 7
        out.append(v)
    return out


@dataclass
class _Node:
    op: str
    inputs: List[str]
    outputs: List[str]


@dataclass
class _Graph:
    tensors: Dict[str, _Tensor]     # initializers and Constant node values defined in this graph
    nodes: List[_Node]
    children: List["_Graph"]        # If / Loop / Scan bodies

    def subtree_dims(self) -> set:
        s = {t.dims for t in self.tensors.values()}
        for c in self.children:
            s |= c.subtree_dims()
        return s


def _graph(buf: bytes) -> _Graph:
    g = _Graph({}, [], [])
    for f, _wt, v in _fields(buf, "a GraphProto"):
        if f == 5:
            t = _tensor(v)
            g.tensors[t.name] = t
        elif f == 1:
            op, ins, outs, value = "", [], [], None
            for nf, _nwt, nv in _fields(v, "a NodeProto"):
                if nf == 1:
                    ins.append(bytes(nv).decode())
                elif nf == 2:
                    outs.append(bytes(nv).decode())
                elif nf == 4:
                    op = bytes(nv).decode()
                elif nf == 5:
                    for af, _awt, av in _fields(nv, "an AttributeProto"):
                        if af == 5:
                            value = _tensor(av)
                        elif af == 6:
                            g.children.append(_graph(av))
                        elif af == 11:
                            g.children.append(_graph(av))
            if op == "Constant" and value is not None and outs:
                value.name = outs[0]
                g.tensors[outs[0]] = value
            g.nodes.append(_Node(op, ins, outs))
    return g


def _model_graph(buf: bytes, what: str) -> _Graph:
    graph = None
    for f, _wt, v in _fields(buf, what):
        if f == 7:
            graph = _graph(v)
    if graph is None:
        raise OnnxError(f"{what}: no graph (not an ONNX model, or truncated)")
    return graph


def _keep_16k(g: _Graph) -> List[_Graph]:
    """The graph and its subgraphs minus every subtree that holds the 8 kHz STFT basis and not the 16 kHz one."""
    out = [g]
    for c in g.children:
        dims = c.subtree_dims()
        if _BASIS_8K in dims and TENSOR_SHAPES["vad.stft.basis"] not in dims:
            continue
        out.extend(_keep_16k(c))
    return out


_ONNX_TO_TORCH_GATES = [0, 2, 3, 1]    # ONNX LSTM blocks i, o, f, c -> PyTorch i, f, g, o


def _permute_gates(a: np.ndarray) -> np.ndarray:
    blocks = np.split(a, 4, axis=0)
    return np.concatenate([blocks[k] for k in _ONNX_TO_TORCH_GATES], axis=0)


def read_silero_onnx(paths: Union[str, os.PathLike, Sequence[Union[str, os.PathLike]]]) -> Dict[str, np.ndarray]:
    """The 16 kHz Silero network from one ONNX file or several whose tensors together form it (faster-whisper ships an
    encoder and a decoder file).  Returns the ``vad.*`` tensors; raises ``OnnxError`` listing what it found otherwise."""
    if isinstance(paths, (str, os.PathLike)):
        paths = [paths]
    graphs: List[_Graph] = []
    for p in paths:
        with open(p, "rb") as fh:
            data = fh.read()
        graphs.extend(_keep_16k(_model_graph(data, f"ONNX file {os.fspath(p)!r}")))
    return _assign_roles(graphs)


def _assign_roles(graphs: List[_Graph]) -> Dict[str, np.ndarray]:
    tensors: Dict[str, _Tensor] = {}
    for g in graphs:
        tensors.update(g.tensors)
    nodes = [n for g in graphs for n in g.nodes]
    alias = {n.outputs[0]: n.inputs[0] for n in nodes if n.op in ("Identity", "Cast") and n.inputs and n.outputs}

    def find(name: str) -> Optional[_Tensor]:
        seen = 0
        while name not in tensors and name in alias and seen < 64:
            name, seen = alias[name], seen + 1
        return tensors.get(name)

    def found() -> str:
        return ", ".join(f"{t.name or '?'} {list(t.dims)}" for t in tensors.values() if t.dims) or "none"

    out: Dict[str, np.ndarray] = {}

    def put(role: str, t: _Tensor, a: Optional[np.ndarray] = None):
        if role in out:
            raise OnnxError(f"two tensors fill {role} ({list(t.dims)}): ambiguous network; tensors found: {found()}")
        out[role] = t.array() if a is None else a

    first_use: Dict[str, int] = {}
    for i, n in enumerate(nodes):
        for x in n.inputs:
            first_use.setdefault(x, i)
        if n.op == "Conv" and len(n.inputs) >= 2:
            w = find(n.inputs[1])
            if w is None:
                continue
            role = _CONV_ROLES.get(w.dims)
            if role is None:
                raise OnnxError(f"Conv weight {w.name!r} has shape {list(w.dims)}, which no role of the 16 kHz Silero "
                                f"network has; tensors found: {found()}")
            put("vad.stft.basis" if role == "vad.stft" else role + ".weight", w)
            if len(n.inputs) >= 3 and n.inputs[2]:
                b = find(n.inputs[2])
                if b is None:
                    raise OnnxError(f"bias {n.inputs[2]!r} of Conv {w.name!r} is not a constant tensor")
                put(role + ".bias", b)
        elif n.op == "LSTM" and len(n.inputs) >= 4:
            W, R, Bt = find(n.inputs[1]), find(n.inputs[2]), find(n.inputs[3])
            if W is None or R is None or Bt is None:
                raise OnnxError("LSTM node whose W / R / B are not constant tensors")
            if W.dims != (1, 4 * HIDDEN, HIDDEN) or R.dims != (1, 4 * HIDDEN, HIDDEN) or Bt.dims != (1, 8 * HIDDEN):
                raise OnnxError(f"LSTM with W {list(W.dims)}, R {list(R.dims)}, B {list(Bt.dims)}; expected "
                                f"[1, 512, 128] twice and [1, 1024]")
            b = Bt.array()[0]
            put("vad.lstm.weight_ih", W, _permute_gates(W.array()[0]))
            put("vad.lstm.weight_hh", R, _permute_gates(R.array()[0]))
            put("vad.lstm.bias_ih", Bt, _permute_gates(b[:4 * HIDDEN]))
            put("vad.lstm.bias_hh", Bt, _permute_gates(b[4 * HIDDEN:]))
    if "vad.lstm.weight_ih" not in out:
        # an LSTMCell exported as MatMul / Gemm: W_ih and W_hh (and the two biases) share a shape, so they are told
        # apart by name, else by which one the graph consumes first (the input projection comes before the recurrence)
        for kind, dims in (("weight", (4 * HIDDEN, HIDDEN)), ("bias", (4 * HIDDEN,))):
            cand = [t for t in tensors.values() if t.dims == dims]
            if len(cand) != 2:
                continue
            by_name = {k: [t for t in cand if k in t.name.lower()] for k in ("ih", "hh")}
            if len(by_name["ih"]) == 1 and len(by_name["hh"]) == 1 and by_name["ih"][0] is not by_name["hh"][0]:
                ih, hh = by_name["ih"][0], by_name["hh"][0]
            else:
                ih, hh = sorted(cand, key=lambda t: first_use.get(t.name, len(nodes)))
            put(f"vad.lstm.{kind}_ih", ih)
            put(f"vad.lstm.{kind}_hh", hh)
    missing = [k for k in TENSOR_SHAPES if k not in out]
    if missing:
        raise OnnxError(f"not a 16 kHz Silero VAD network: missing {', '.join(missing)}; tensors found: {found()}")
    for k, shape in TENSOR_SHAPES.items():
        if tuple(out[k].shape) != shape:
            raise OnnxError(f"{k} has shape {list(out[k].shape)}, expected {list(shape)}")
    return out


# ---------------------------------------------------------------------------------------------- weights
def random_weights(seed: int = 0, basis: str = "dft") -> Dict[str, np.ndarray]:
    """Seeded weights of the real shapes (tests and tools).  ``basis="dft"``: the windowed DFT an STFT front end uses
    (Hann window, 129 real rows then 129 imaginary rows); ``"random"``: Gaussian rows."""
    rng = np.random.default_rng(seed)
    out: Dict[str, np.ndarray] = {}
    if basis == "dft":
        n = np.arange(256)
        k = np.arange(129)[:, None]
        win = 0.5 - 0.5 * np.cos(2 * np.pi * n / 256)
        ang = 2 * np.pi * k * n / 256
        out["vad.stft.basis"] = np.concatenate([np.cos(ang) * win, -np.sin(ang) * win])[:, None, :].astype(np.float32)
    elif basis == "random":
        out["vad.stft.basis"] = (rng.standard_normal((258, 1, 256)) / 16).astype(np.float32)
    else:
        raise ValueError(f"basis={basis!r}: 'dft' or 'random'")
    for name, shape in TENSOR_SHAPES.items():
        if name == "vad.stft.basis":
            continue
        # the output head unscaled: with 1/sqrt(fan_in) there too the probabilities of a random network stay within
        # about 1e-3 of each other, and gating on them would test nothing
        fan_in = 1 if name == "vad.out.weight" else int(np.prod(shape[1:])) if len(shape) > 1 else 128
        out[name] = (rng.uniform(-1.0, 1.0, shape) / np.sqrt(fan_in)).astype(np.float32)
    return out


def _bundled_model_files() -> List[str]:
    import faster_whisper  # noqa: F401  (ImportError when absent)
    assets = os.path.join(os.path.dirname(faster_whisper.__file__), "assets")
    enc = sorted(glob.glob(os.path.join(assets, "silero_encoder*.onnx")))
    dec = sorted(glob.glob(os.path.join(assets, "silero_decoder*.onnx")))
    if enc and dec:
        return [enc[-1], dec[-1]]
    single = sorted(glob.glob(os.path.join(assets, "silero_vad*.onnx")))
    if single:
        return [single[-1]]
    raise FileNotFoundError(f"no Silero VAD model under {assets}")


def resolve_weights(weights=None, seed: int = 0) -> Dict[str, np.ndarray]:
    """A tensor dict, ``"random"`` (seeded), an ONNX path or list of paths, or None: ``WLB200_VAD_MODEL`` (paths
    separated by ``os.pathsep``), else faster-whisper's bundled model.  Raises when none of these gives the weights."""
    if isinstance(weights, dict):
        return dict(weights)
    if isinstance(weights, str) and weights == "random":
        return random_weights(seed)
    if weights is not None:
        return read_silero_onnx(weights)
    env = os.environ.get("WLB200_VAD_MODEL")
    if env:
        return read_silero_onnx([p for p in env.split(os.pathsep) if p])
    try:
        files = _bundled_model_files()
    except (ImportError, FileNotFoundError) as e:
        raise RuntimeError("the device VAD needs the Silero model: set WLB200_VAD_MODEL=<silero .onnx file(s)> or "
                           f"install faster-whisper, whose bundled model it reads ({e})") from e
    return read_silero_onnx(files)


# ---------------------------------------------------------------------------------------------- gating (host)
@dataclass
class VadOptions:
    """faster-whisper 1.2.0 ``VadOptions``."""
    threshold: float = 0.5
    neg_threshold: Optional[float] = None
    min_speech_duration_ms: int = 0
    max_speech_duration_s: float = float("inf")
    min_silence_duration_ms: int = 2000
    speech_pad_ms: int = 400


def speech_timestamps_from_probs(speech_probs: Sequence[float], audio_length_samples: int,
                                 vad_options: Optional[VadOptions] = None, sampling_rate: int = SAMPLING_RATE) -> List[dict]:
    """faster-whisper 1.2.0 ``get_speech_timestamps`` after its model call, restated: hysteresis between ``threshold``
    and ``neg_threshold``, ``min_silence_duration_ms`` before a chunk ends, ``max_speech_duration_s`` (split at the last
    silence of at least 98 ms, else cut where the limit is reached), ``min_speech_duration_ms``, then ``speech_pad_ms``
    on both sides (half the gap when two chunks are closer than twice the pad)."""
    o = vad_options or VadOptions()
    window = FRAME_SAMPLES
    threshold = o.threshold
    neg_threshold = o.neg_threshold if o.neg_threshold is not None else max(threshold - 0.15, 0.01)
    min_speech_samples = sampling_rate * o.min_speech_duration_ms / 1000
    speech_pad_samples = sampling_rate * o.speech_pad_ms / 1000
    max_speech_samples = sampling_rate * o.max_speech_duration_s - window - 2 * speech_pad_samples
    min_silence_samples = sampling_rate * o.min_silence_duration_ms / 1000
    min_silence_samples_at_max_speech = sampling_rate * 98 / 1000

    triggered = False
    speeches: List[dict] = []
    current: dict = {}
    temp_end = 0
    prev_end = next_start = 0
    for i, p in enumerate(speech_probs):
        if p >= threshold and temp_end:
            temp_end = 0
            if next_start < prev_end:
                next_start = window * i
        if p >= threshold and not triggered:
            triggered = True
            current["start"] = window * i
            continue
        if triggered and window * i - current["start"] > max_speech_samples:
            if prev_end:
                current["end"] = prev_end
                speeches.append(current)
                current = {}
                if next_start < prev_end:
                    triggered = False
                else:
                    current["start"] = next_start
                prev_end = next_start = temp_end = 0
            else:
                current["end"] = window * i
                speeches.append(current)
                current = {}
                prev_end = next_start = temp_end = 0
                triggered = False
                continue
        if p < neg_threshold and triggered:
            if not temp_end:
                temp_end = window * i
            if window * i - temp_end > min_silence_samples_at_max_speech:
                prev_end = temp_end
            if window * i - temp_end < min_silence_samples:
                continue
            current["end"] = temp_end
            if current["end"] - current["start"] > min_speech_samples:
                speeches.append(current)
            current = {}
            prev_end = next_start = temp_end = 0
            triggered = False
            continue
    if current and audio_length_samples - current["start"] > min_speech_samples:
        current["end"] = audio_length_samples
        speeches.append(current)

    for i, s in enumerate(speeches):
        if i == 0:
            s["start"] = int(max(0, s["start"] - speech_pad_samples))
        if i != len(speeches) - 1:
            silence = speeches[i + 1]["start"] - s["end"]
            if silence < 2 * speech_pad_samples:
                s["end"] += int(silence // 2)
                speeches[i + 1]["start"] = int(max(0, speeches[i + 1]["start"] - silence // 2))
            else:
                s["end"] = int(min(audio_length_samples, s["end"] + speech_pad_samples))
                speeches[i + 1]["start"] = int(max(0, speeches[i + 1]["start"] - speech_pad_samples))
        else:
            s["end"] = int(min(audio_length_samples, s["end"] + speech_pad_samples))
    return speeches


def collect_chunks(audio: np.ndarray, chunks: List[dict], sampling_rate: int = SAMPLING_RATE,
                   max_duration: float = float("inf")) -> Tuple[List[np.ndarray], List[dict]]:
    """faster-whisper 1.2.0 ``collect_chunks``: the speech chunks concatenated, in groups of at most ``max_duration``."""
    if not chunks:
        return [np.array([], dtype=np.float32)], [{"offset": 0, "duration": 0, "segments": []}]
    audio_chunks, metadata = [], []
    segments: List[dict] = []
    current_duration = total_duration = 0
    current = np.array([], dtype=np.float32)
    for c in chunks:
        if current_duration + c["end"] - c["start"] > max_duration * sampling_rate:
            audio_chunks.append(current)
            metadata.append({"offset": total_duration / sampling_rate, "duration": current_duration / sampling_rate,
                             "segments": segments})
            total_duration += current_duration
            segments = [c]
            current = audio[c["start"]:c["end"]]
            current_duration = c["end"] - c["start"]
        else:
            segments.append(c)
            current = np.concatenate((current, audio[c["start"]:c["end"]]))
            current_duration += c["end"] - c["start"]
    audio_chunks.append(current)
    metadata.append({"offset": total_duration / sampling_rate, "duration": current_duration / sampling_rate,
                     "segments": segments})
    return audio_chunks, metadata


class SpeechTimestampsMap:
    """Maps times on the silence-free axis back to the original audio (faster-whisper ``vad.py``)."""

    def __init__(self, chunks: List[dict], sampling_rate: int, time_precision: int = 2):
        self.sampling_rate = sampling_rate
        self.time_precision = time_precision
        self.chunk_end_sample: List[int] = []
        self.total_silence_before: List[float] = []
        previous_end = 0
        silent_samples = 0
        for chunk in chunks:
            silent_samples += chunk["start"] - previous_end
            previous_end = chunk["end"]
            self.chunk_end_sample.append(chunk["end"] - silent_samples)
            self.total_silence_before.append(silent_samples / sampling_rate)

    def get_original_time(self, time: float, chunk_index: Optional[int] = None, is_end: bool = False) -> float:
        if chunk_index is None:
            chunk_index = self.get_chunk_index(time, is_end)
        return round(self.total_silence_before[chunk_index] + time, self.time_precision)

    def get_chunk_index(self, time: float, is_end: bool = False) -> int:
        sample = int(time * self.sampling_rate)
        if sample in self.chunk_end_sample and is_end:
            return self.chunk_end_sample.index(sample)
        return min(bisect.bisect(self.chunk_end_sample, sample), len(self.chunk_end_sample) - 1)


# ---------------------------------------------------------------------------------------------- the module object
class DeviceVad:
    """``faster_whisper.vad`` interface (``VadOptions``, ``get_speech_timestamps``, ``collect_chunks``,
    ``SpeechTimestampsMap``) with the probabilities computed by ``engine`` (``vad_load`` / ``vad_probs``: a
    ``B200Whisper`` context), plus ``speech_timestamps_batch``, which answers many streams with one device call."""

    VadOptions = VadOptions
    SpeechTimestampsMap = SpeechTimestampsMap

    def __init__(self, engine, weights=None, seed: int = 0):
        self.engine = engine
        engine.vad_load(resolve_weights(weights, seed))

    @staticmethod
    def collect_chunks(audio, chunks, sampling_rate: int = SAMPLING_RATE, max_duration: float = float("inf")):
        return collect_chunks(audio, chunks, sampling_rate, max_duration)

    def get_speech_timestamps(self, audio: np.ndarray, vad_options: Optional[VadOptions] = None,
                              sampling_rate: int = SAMPLING_RATE, **kwargs) -> List[dict]:
        return self.speech_timestamps_batch([audio], [vad_options or VadOptions(**kwargs)], sampling_rate)[0]

    def speech_timestamps_batch(self, audios: Sequence[np.ndarray],
                                vad_options: Union[None, VadOptions, Sequence[Optional[VadOptions]]] = None,
                                sampling_rate: int = SAMPLING_RATE) -> List[List[dict]]:
        """Speech chunks of every waveform, from one ``wl_vad`` call.  ``vad_options``: one for all, or one per stream."""
        if sampling_rate != SAMPLING_RATE:
            raise ValueError(f"the Silero VAD runs at {SAMPLING_RATE} Hz, not {sampling_rate}")
        if vad_options is None or isinstance(vad_options, VadOptions):
            vad_options = [vad_options] * len(audios)
        if len(vad_options) != len(audios):
            raise ValueError(f"{len(vad_options)} VadOptions for {len(audios)} streams")
        waves = [np.asarray(a, dtype=np.float32).reshape(-1) for a in audios]
        probs = self.engine.vad_probs(waves)
        return [speech_timestamps_from_probs(p, w.shape[0], o, sampling_rate) for p, w, o in zip(probs, waves, vad_options)]
