"""B200Whisper: the CUDA engine with the ``ctranslate2.models.Whisper`` call surface (Boundary C).

Reference call sites it is a drop-in for (whisper_live/transcriber/transcriber_faster_whisper.py):
ctor :634-643, ``encode`` :1348, ``generate`` :1394-1407, ``detect_language`` :1140 / :1771,
``align`` :1657-1663, properties ``is_multilingual`` :652, ``n_mels`` :446, ``device`` /
``device_index`` :1342; and whisper_live/batch_inference.py:271, :283, :355.  All arithmetic runs in
libwlb200.so through the C ABI (include/wlb200.h); numpy arrays are only the host-side containers.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
import weakref
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np

from . import _lib
from .config import WhisperDims, dims_for
from .tokenizer import LANGUAGE_CODES

T_MAX = 448


@dataclass
class WhisperGenerationResult:
    sequences_ids: List[List[int]]
    scores: List[float]
    no_speech_prob: float
    steps: int = 0


@dataclass
class WhisperAlignmentResult:
    alignments: List[Tuple[int, int]]
    text_token_probs: List[float]


class _SlotRef:
    """Reference-counted ownership of encoder slots in the library's pool."""

    def __init__(self, engine: "B200Whisper", slots: List[int]):
        self.engine = engine
        self.slots = list(slots)
        self._fin = weakref.finalize(self, B200Whisper._release_slots, weakref.ref(engine), list(slots))

    def release(self) -> None:
        """Give the slots back now (idempotent); every view sharing this owner becomes invalid."""
        self._fin()
        self.slots = []


class _Borrowed:
    """Owner stand-in of a joined handle: holds references to the real owners, releases nothing."""

    def __init__(self, owners, engine):
        self.owners, self.engine, self.slots = owners, engine, []

    def release(self) -> None:
        return


class EncoderOutput:
    """Opaque handle playing the role of the ``ctranslate2.StorageView`` returned by encode():
    a list of pool slots (encoder output + cross-attention K/V resident in HBM)."""

    def __init__(self, owner: _SlotRef, slots: List[int], d_model: int):
        self._owner = owner
        self.slots = list(slots)
        self._d = d_model

    @property
    def shape(self):
        return (len(self.slots), 1500, self._d)

    def select(self, indices: Sequence[int]) -> "EncoderOutput":
        return EncoderOutput(self._owner, [self.slots[i] for i in indices], self._d)

    def join(self, views: Sequence["EncoderOutput"]) -> "EncoderOutput":
        """One batch handle over the slots of several views (of this or other encode calls).  Borrowed: the result
        keeps its parents alive but never releases their slots itself."""
        return EncoderOutput(_Borrowed([v._owner for v in views], self._owner.engine), [s_ for v in views for s_ in v.slots], self._d)

    def release(self) -> None:
        """Explicit end of life of the encoder output and ALL its views (the transcriber calls this at the end of
        every window instead of relying on reference counting)."""
        self._owner.release()
        self.slots = []

    def __len__(self):
        return len(self.slots)

    def __array__(self, dtype=None, copy=None):
        eng = self._owner.engine
        out = np.stack([eng._encoder_output(s) for s in self.slots])
        return out.astype(dtype) if dtype is not None else out


# stored dtype -> WL_DT_* of wl_load_tensor_typed (uint16 is bfloat16 bits: weights.BF16)
_WL_DT = {np.dtype(np.float32): 0, np.dtype(np.float16): 1, np.dtype(np.uint16): 2, np.dtype(np.int8): 3}


def footprint_estimate(dims: WhisperDims, max_streams: int = 8, max_beam: int = 5, enc_slots: Optional[int] = None,
                       n_align_heads: Optional[int] = None, vad: bool = False, diarize: bool = False) -> int:
    """Device bytes a context of these shapes allocates through ``wl_init``, the weight load and one open decode session
    (csrc/engine.cu: ``wl_load_tensor``, ``finalize_impl``, ``alloc_decode_state``, ``wl_session_open``), plus the
    workspaces its first step round grows: the log-mel of ``max_streams`` 30-second chunks (``wl_mel``) and the batched
    prefill at its first size of 1024 rows (``prefill_reserve``).  What a model registry compares with the free memory
    before a load.  ``vad=True`` adds the Silero VAD weights and the VAD workspace of ``max_streams`` 30-second chunks
    (``wl_vad_load_tensor``, ``wl_vad``); ``diarize=True`` the speaker-embedding weights and the workspace of its first
    call, ``max_streams`` segments of 30 s (``wl_spk_load_tensor``, ``wl_spk_embed``).  Not included: the CUDA context of the process, CUDA graph executables, workspaces grown later (longer
    chunks, more prompt rows, the word-alignment buffers; a grown workspace replaces the one before it, so it adds only
    the difference) and the allocator's rounding."""
    B, K = int(max_streams), int(max_beam)
    NS = int(enc_slots) if enc_slots is not None else 2 * B
    d, H, Le, Ld, nm, V = dims.d_model, dims.n_heads, dims.enc_layers, dims.dec_layers, dims.n_mels, dims.vocab
    ff, dd, S, S_PAD, T = 4 * d, d * d, 1500, 1536, T_MAX
    MAX_HYPS, MAX_CAND, MAX_ROWS = 24, 16, 8          # csrc/kernels.cuh
    PEEK_STRIDE = 8 + 2 * MAX_HYPS + T_MAX
    if n_align_heads is None:
        n_align_heads = len(dims.default_alignment_heads())
    f32 = i32 = 4
    f16 = 2
    # weights as uploaded: fp16 for matrices, fp32 for vectors, the encoder position table and the mel filters
    enc_layer = 4 * dd * f16 + 3 * d * f32 + 2 * d * f32 + 2 * ff * d * f16 + (ff + d) * f32 + 2 * d * f32
    dec_layer = 8 * dd * f16 + 6 * d * f32 + 3 * 2 * d * f32 + 2 * ff * d * f16 + (ff + d) * f32
    weights = (d * nm * 3 * f16 + d * f32 + d * d * 3 * f16 + d * f32 + S * d * f32 + Le * enc_layer + 2 * d * f32
               + V * d * f16 + T * d * f16 + Ld * dec_layer + 2 * d * f32 + nm * 201 * f32)
    # fused copies finalize makes: encoder Q|K, decoder Q|K|V (weights and biases)
    fused = Le * (2 * dd * f16 + 2 * d * f32) + Ld * (3 * dd * f16 + 3 * d * f32)
    mel_tables = (400 + 800) * f32 + 2 * nm * i32 + B * 4 + 4 * (B + 1) * 8 + B * i32 + 3 * B * i32
    EB = min(B, max(1, int(os.environ.get("WLB200_ENC_BATCH") or 16)))
    AB = min(EB, 2 if d >= 1024 else 4)
    M = EB * S
    encoder = (B * nm * 3000 * f32 + (EB * 3002 * nm + 4096) * f16 + (EB * 3002 * d + 4096) * f16 + M * d * f32
               + M * d * f16 + M * 2 * d * f16 + EB * d * S_PAD * f16 + AB * H * S * S_PAD * (f32 + f16) + M * d * f16
               + M * ff * f16 + B * i32)
    pool = NS * S * d * f16 + Ld * 2 * NS * S * d * f16
    R = B * K
    Rp = (R + 15) // 16 * 16
    mask = ((V + 31) // 32 + 1) * 4
    caches = 2 * Ld * R * H * T * 64 * f16
    decoder = (R * d * f32 + (R * 16 * d + R * 4 * ff) * f32 + R * 16 * d * f32 + R * ((V + 3) // 4 * 4) * f32
               + 2 * Rp * d * f16 + Rp * ff * f16 + caches + B * H * 12 * MAX_ROWS * 66 * f32 + mask
               + (2 * n_align_heads * i32 if n_align_heads else 0))
    state = (8 * R * 4 + R * T * i32 + R * T * 2 + 2 * R * MAX_CAND * 4 + 22 * B * 4 + B * T * i32
             + 2 * B * MAX_HYPS * 4 + B * MAX_HYPS * T * i32 + B * T * f32 + 4 * 4)
    session = state + caches + mask + B * i32 + B * PEEK_STRIDE * i32
    pcm = B * 30 * 16000
    frames = B * (30 * 16000 // 160 + 1) * nm
    mel = (pcm + pcm // 4) * f32 + (frames + frames // 4) * f32
    cap = 1024
    prefill = (4 * cap * i32 + 2 * (cap // 8 + 128) * i32 + (3 * R + 16) * i32 + cap * T * 2 + 5 * cap * d * f32
               + 2 * cap * d * f16 + cap * ff * f16 + 128 * H * 12 * MAX_ROWS * 66 * f32)
    total = weights + fused + mel_tables + encoder + pool + decoder + state + session + mel + prefill
    if vad:
        vad_weights = (258 * 256 + 128 * 129 * 3 + 128 + 64 * 128 * 3 + 64 + 64 * 64 * 3 + 64 + 128 * 64 * 3 + 128
                       + 2 * 512 * 128 + 2 * 512 + 128 + 1) * f32
        vad_frames = B * (pcm // B // 512 + 1)
        total += vad_weights + pcm * f32 + vad_frames * (512 + 1) * f32 + 2 * (B + 1) * 8
    if diarize:
        total += spk_footprint(B)
    return int(total)


def spk_footprint(max_streams: int) -> int:
    """Device bytes of the speaker-embedding weights as ``wl_spk_load_tensor`` stores them (fp16 tensor-core conv
    weights, fp32 stem, biases and embedding layer) plus the workspace ``wl_spk_embed`` allocates at its first call."""
    from . import speaker as S
    B, f32, f16 = int(max_streams), 4, 2
    weights = 0
    for name, co, ci, k in S.conv_names():
        weights += co * ci * k * k * (f32 if ci == 1 else f16) + co * f32
    weights += (S.POOL_DIM * S.EMBED_DIM + S.EMBED_DIM) * f32
    mel = S.MEL_BINS * (S.N_FFT // 2 + 1) * f32 + 2 * S.MEL_BINS * 4
    pcm = B * 30 * S.SAMPLING_RATE
    frames = B * S.n_frames(30 * S.SAMPLING_RATE)
    per_stream = (S.MEL_BINS + S.POOL_DIM + S.EMBED_DIM) * f32 + 6 * 8
    acts, T = [], S.n_frames(30 * S.SAMPLING_RATE)
    for L, (c, _nb, _stride) in enumerate(S.STAGES):
        if L:
            T = (T + 1) // 2
        acts.append(B * (S.MEL_BINS >> L) * T * c)
    act = max(acts[0], acts[2]) + max(acts) + max(acts[1], acts[3])
    return int(weights + mel + pcm * f32 + frames * S.MEL_BINS * f32 + B * per_stream + 6 * 8 + act * f16)


def mem_info(device: int = 0) -> Tuple[int, int]:
    """``(free, total)`` device memory of CUDA ordinal ``device`` in bytes (``wl_mem_info``; no context needed)."""
    lib = _lib.load()
    free, total = C.c_int64(0), C.c_int64(0)
    rc = lib.wl_mem_info(int(device), C.byref(free), C.byref(total))
    if rc != 0:
        raise _lib.WlError(f"wl_mem_info failed ({rc}): {lib.wl_last_error(None).decode()}")
    return int(free.value), int(total.value)


def _gen_opts(beam_size, patience, num_hypotheses, length_penalty, max_length, suppress_blank, max_initial_timestamp_index,
              sampling_topk, sampling_temperature, seed, sup: np.ndarray, use_cuda_graph, prefill) -> "_lib.WlGenOpts":
    """wl_gen_opts of a generate call (``sup`` must outlive the call; ``max_length_per_stream`` is left unset)."""
    return _lib.WlGenOpts(
        beam_size=int(beam_size), patience=float(patience), num_hypotheses=int(num_hypotheses),
        length_penalty=float(length_penalty), max_length=int(max_length), suppress_blank=int(bool(suppress_blank)),
        max_initial_timestamp_index=int(max_initial_timestamp_index), sampling_topk=int(sampling_topk),
        sampling_temperature=float(sampling_temperature), seed=int(seed) & 0xFFFFFFFF,
        suppress_tokens=_lib.ptr(sup, C.c_int32) if len(sup) else None, n_suppress=len(sup),
        use_cuda_graph=int(use_cuda_graph), max_length_per_stream=None,
        prefill=0 if prefill is None else (1 if prefill else 2))


class B200Whisper:
    def __init__(self, dims: WhisperDims, weights: Dict[str, "np.ndarray"], device_index: Union[int, List[int]] = 0,
                 compute_type: str = "float16", max_streams: int = 8, max_beam: int = 5, enc_slots: Optional[int] = None,
                 alignment_heads: Optional[List[Tuple[int, int]]] = None, use_cuda_graph: bool = True):
        if compute_type not in ("float16", "default", "auto"):
            raise ValueError(f"compute_type {compute_type!r}: the engine computes in float16 with fp32 accumulation")
        self.lib = _lib.load()
        self.dims = dims
        self.device = "cuda"
        self.device_index = [device_index] if isinstance(device_index, int) else list(device_index)
        self.compute_type = "float16"
        self.max_streams = max_streams
        self.max_beam = max_beam
        self.enc_slots = enc_slots if enc_slots is not None else 2 * max_streams
        self.use_cuda_graph = use_cuda_graph
        self._lock = threading.RLock()
        from .weights import _special_ids
        eot, ts_begin = _special_ids(dims)
        self.eot, self.sot = eot, eot + 1
        self.timestamp_begin = ts_begin
        self.no_timestamps = ts_begin - 1
        self.no_speech = ts_begin - 2
        n_lang = dims.num_languages if dims.multilingual else 0
        heads = alignment_heads if alignment_heads is not None else dims.default_alignment_heads()
        self.alignment_heads = [(int(l), int(h)) for l, h in heads]
        self._heads_arr = np.asarray(self.alignment_heads, dtype=np.int32).reshape(-1)
        cfg = _lib.WlConfig(
            abi_version=_lib.ABI_VERSION, device=self.device_index[0], d_model=dims.d_model, n_heads=dims.n_heads,
            enc_layers=dims.enc_layers, dec_layers=dims.dec_layers, n_mels=dims.n_mels, vocab=dims.vocab, eot=eot,
            sot=eot + 1, no_speech=self.no_speech, no_timestamps=self.no_timestamps, timestamp_begin=ts_begin, blank=220,
            lang_begin=eot + 2, n_lang=n_lang, max_streams=max_streams, max_beam=max_beam,
            enc_slots=enc_slots if enc_slots is not None else 2 * max_streams,
            n_align_heads=len(self.alignment_heads), align_heads=_lib.ptr(self._heads_arr, C.c_int32))
        ctx = C.c_void_p()
        rc = self.lib.wl_init(C.byref(cfg), C.byref(ctx))
        if rc != 0:
            raise _lib.WlError(f"wl_init failed ({rc}): {self.lib.wl_last_error(None).decode()}")
        self.ctx = ctx
        self._fin = weakref.finalize(self, self.lib.wl_destroy, ctx)
        try:
            self._load_weights(weights)
        except BaseException:
            self._fin()      # a failed load gives its device memory back now, not when the traceback is collected
            raise

    # ------------------------------------------------------------------ construction
    @classmethod
    def from_model(cls, model_size_or_path: str, device_index=0, compute_type="float16", weights=None, seed: int = 0,
                   max_streams: int = 8, max_beam: int = 5, download_root: Optional[str] = None,
                   local_files_only: bool = False, **kw) -> "B200Whisper":
        """Resolve ``model_size_or_path`` the way the reference does (faster_whisper_backend.py:133-178,
        transcriber_faster_whisper.py:620-656): a local directory holding HF ``model.safetensors`` or the
        CTranslate2 ``model.bin``; else a size name / hub id looked up through ``huggingface_hub``
        (``Systran/faster-whisper-<size>``, honouring ``download_root`` / ``local_files_only``).  When no
        checkpoint can be found this RAISES -- a transcriber serving random weights is never built silently.
        ``weights`` may be a tensor dict, or the explicit opt-in ``"random"`` (seeded random initialisation of
        the named architecture: bench.py and the tests, which run without network or checkpoints)."""
        import os
        from . import weights as W
        if isinstance(weights, str):
            if weights != "random":
                raise ValueError(f"weights={weights!r}: pass a tensor dict, None, or the explicit opt-in 'random'")
            dims = dims_for(model_size_or_path)
            return cls(dims, W.random_init(dims, seed=seed), device_index=device_index, compute_type=compute_type,
                       max_streams=max_streams, max_beam=max_beam, **kw)
        model_dir, metadata = None, {}
        if weights is None:
            model_dir = W.resolve_model_dir(model_size_or_path, download_root=download_root, local_files_only=local_files_only)
            weights = W.open_checkpoint(model_dir)     # streamed to the device tensor by tensor, as stored
            metadata = W.model_metadata(model_dir)
            if kw.get("alignment_heads") is None and metadata.get("alignment_heads"):
                kw["alignment_heads"] = metadata["alignment_heads"]
        shapes = weights.shapes if hasattr(weights, "tensors") else weights
        try:
            dims = dims_for(model_size_or_path)
        except KeyError:
            dims = W.infer_dims(shapes, str(model_size_or_path))
        eng = cls(dims, weights, device_index=device_index, compute_type=compute_type, max_streams=max_streams,
                  max_beam=max_beam, **kw)
        eng.model_dir = model_dir
        eng.model_metadata = metadata
        return eng

    def _load_weights(self, weights) -> None:
        """``weights``: a tensor dict (uploaded as fp32 through ``wl_load_tensor``) or a checkpoint reader
        (``weights.open_checkpoint``), whose tensors go over one at a time in their stored dtype through
        ``wl_load_tensor_typed`` and are converted on the device."""
        from .feature_extractor import mel_filters
        if hasattr(weights, "tensors"):
            for name, a, scale in weights.tensors():
                self._load_typed(name, a, scale)
            weights = {}
        items = dict(weights)
        items["mel_filters"] = mel_filters(self.dims.n_mels)
        for name, t in items.items():
            a = t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
            a = np.ascontiguousarray(a, dtype=np.float32)
            shape = np.asarray(a.shape, dtype=np.int64)
            rc = self.lib.wl_load_tensor(self.ctx, name.encode(), _lib.ptr(a, C.c_float), _lib.ptr(shape, C.c_int64), a.ndim)
            _lib.check(self.lib, self.ctx, rc, f"wl_load_tensor({name})")
        _lib.check(self.lib, self.ctx, self.lib.wl_finalize_weights(self.ctx), "wl_finalize_weights")

    def _load_typed(self, name: str, a: np.ndarray, scale: Optional[np.ndarray] = None) -> None:
        a = np.ascontiguousarray(a)
        if a.dtype not in _WL_DT:
            raise ValueError(f"{name}: dtype {a.dtype} cannot be uploaded (float32, float16, bfloat16 bits or int8)")
        shape = np.asarray(a.shape, dtype=np.int64)
        s, sdt = None, 0
        if scale is not None:
            s = np.ascontiguousarray(scale).reshape(-1)
            sdt = _WL_DT[s.dtype]
        rc = self.lib.wl_load_tensor_typed(self.ctx, name.encode(), a.ctypes.data, _WL_DT[a.dtype],
                                           _lib.ptr(shape, C.c_int64), a.ndim, None if s is None else s.ctypes.data, sdt)
        _lib.check(self.lib, self.ctx, rc, f"wl_load_tensor_typed({name})")

    # ------------------------------------------------------------------ properties (ctranslate2 names)
    @property
    def is_multilingual(self) -> bool:
        return self.dims.multilingual

    @property
    def n_mels(self) -> int:
        return self.dims.n_mels

    @property
    def num_languages(self) -> int:
        return self.dims.num_languages

    @property
    def vocab_size(self) -> int:
        return self.dims.vocab

    def kernel_launches(self) -> int:
        return int(self.lib.wl_kernel_launches(self.ctx))

    @property
    def device_bytes(self) -> int:
        """Device memory this context holds right now (``wl_device_bytes``): weights, workspaces, slot pool, caches,
        decode states and the grown workspaces at their current sizes (a grown workspace replaces the one before it);
        0 once the context is destroyed."""
        out = C.c_int64(0)
        with self._lock:     # destroy() frees the context under the same lock
            if not self._fin.alive:
                return 0
            _lib.check(self.lib, self.ctx, self.lib.wl_device_bytes(self.ctx, C.byref(out)), "wl_device_bytes")
        return int(out.value)

    def destroy(self) -> None:
        """Free the context and all its device memory now (idempotent); the engine is unusable afterwards."""
        with self._lock:
            self._fin()

    def last_device_ms(self, which: int) -> float:
        return float(self.lib.wl_last_device_ms(self.ctx, which))

    def vad_load(self, tensors: Dict[str, "np.ndarray"]) -> None:
        """Upload the Silero VAD tensors (``vad.*`` names of include/wlb200.h) as float32."""
        for name, t in tensors.items():
            a = np.ascontiguousarray(t, dtype=np.float32)
            shape = np.asarray(a.shape, dtype=np.int64)
            with self._lock:
                rc = self.lib.wl_vad_load_tensor(self.ctx, name.encode(), _lib.ptr(a, C.c_float), _lib.ptr(shape, C.c_int64),
                                                 a.ndim)
                _lib.check(self.lib, self.ctx, rc, f"wl_vad_load_tensor({name})")

    def vad_probs(self, audios: Sequence[np.ndarray]) -> List[np.ndarray]:
        """Silero speech probability of every 512-sample frame of each waveform (``wl_vad``): one upload of all of
        them, one launch of each kernel, one download."""
        from .vad import n_frames
        if not audios:
            return []
        waves = [np.ascontiguousarray(a, dtype=np.float32).reshape(-1) for a in audios]
        lens = np.asarray([w.shape[0] for w in waves], dtype=np.int64)
        off = np.zeros(len(waves) + 1, dtype=np.int64)
        off[1:] = np.cumsum(lens)
        poff = np.zeros(len(waves) + 1, dtype=np.int64)
        poff[1:] = np.cumsum([n_frames(int(n)) for n in lens])
        pcm = np.concatenate(waves) if off[-1] else np.zeros(1, np.float32)
        out = np.empty(max(int(poff[-1]), 1), dtype=np.float32)
        with self._lock:
            rc = self.lib.wl_vad(self.ctx, _lib.ptr(pcm, C.c_float), _lib.ptr(off, C.c_int64), len(waves),
                                 _lib.ptr(out, C.c_float), _lib.ptr(poff, C.c_int64))
            _lib.check(self.lib, self.ctx, rc, "wl_vad")
        return [out[poff[i]:poff[i + 1]].copy() for i in range(len(waves))]

    def spk_load(self, tensors: Dict[str, "np.ndarray"]) -> None:
        """Upload the speaker-embedding tensors (``spk.*`` names of include/wlb200.h, BN folded) as float32."""
        for name, t in tensors.items():
            a = np.ascontiguousarray(t, dtype=np.float32)
            shape = np.asarray(a.shape, dtype=np.int64)
            with self._lock:
                rc = self.lib.wl_spk_load_tensor(self.ctx, name.encode(), _lib.ptr(a, C.c_float), _lib.ptr(shape, C.c_int64),
                                                 a.ndim)
                _lib.check(self.lib, self.ctx, rc, f"wl_spk_load_tensor({name})")

    def spk_embeddings(self, audios: Sequence[np.ndarray]) -> np.ndarray:
        """Speaker embeddings [B, 256] of 16 kHz waveforms of at least 400 samples (``wl_spk_embed``): one upload of all
        of them, one pass of the network, one download."""
        if not audios:
            return np.zeros((0, 256), np.float32)
        waves = [np.ascontiguousarray(a, dtype=np.float32).reshape(-1) for a in audios]
        off = np.zeros(len(waves) + 1, dtype=np.int64)
        off[1:] = np.cumsum([w.shape[0] for w in waves])
        pcm = np.concatenate(waves)
        out = np.empty((len(waves), 256), dtype=np.float32)
        with self._lock:
            rc = self.lib.wl_spk_embed(self.ctx, _lib.ptr(pcm, C.c_float), _lib.ptr(off, C.c_int64), len(waves),
                                       _lib.ptr(out, C.c_float))
            _lib.check(self.lib, self.ctx, rc, "wl_spk_embed")
        return out

    def test_spk_fbank(self, audios: Sequence[np.ndarray]) -> List[np.ndarray]:
        """``wl_spk_embed``'s fbank of each waveform (``wl_test_spk_fbank``): [frames, 80] before CMN."""
        from .speaker import n_frames
        waves = [np.ascontiguousarray(a, dtype=np.float32).reshape(-1) for a in audios]
        off = np.zeros(len(waves) + 1, dtype=np.int64)
        off[1:] = np.cumsum([w.shape[0] for w in waves])
        foff = np.zeros(len(waves) + 1, dtype=np.int64)
        foff[1:] = np.cumsum([n_frames(w.shape[0]) for w in waves])
        pcm = np.concatenate(waves)
        out = np.empty((max(int(foff[-1]), 1), 80), dtype=np.float32)
        with self._lock:
            rc = self.lib.wl_test_spk_fbank(self.ctx, _lib.ptr(pcm, C.c_float), _lib.ptr(off, C.c_int64), len(waves),
                                            _lib.ptr(out, C.c_float))
            _lib.check(self.lib, self.ctx, rc, "wl_test_spk_fbank")
        return [out[foff[i]:foff[i + 1]].copy() for i in range(len(waves))]

    def test_spk_conv(self, x: np.ndarray, frames: Sequence[int], H_in: int, w: np.ndarray, bias: np.ndarray, stride: int,
                      res: Optional[np.ndarray] = None, relu: bool = True, out: Optional[np.ndarray] = None) -> np.ndarray:
        """One convolution launch of ``wl_spk_embed`` (``wl_test_spk_conv``): x fp16 [positions, C_in], w fp16
        [C_out, taps, C_in], res / out fp16 [out positions, C_out] (out: the buffer as it is before the launch)."""
        x16 = np.ascontiguousarray(x, dtype=np.float16)
        w16 = np.ascontiguousarray(w, dtype=np.float16)
        C_out, taps, C_in = w16.shape
        k = int(round(taps ** 0.5))
        fr = np.ascontiguousarray(frames, dtype=np.int64)
        H_out = (H_in + 1) // 2 if stride == 2 else H_in
        T_out = (fr + 1) // 2 if stride == 2 else fr
        M = int(H_out * T_out.sum())
        o16 = np.zeros((M, C_out), np.float16) if out is None else np.ascontiguousarray(out, dtype=np.float16).copy()
        b32 = np.ascontiguousarray(bias, dtype=np.float32)
        r16 = None if res is None else np.ascontiguousarray(res, dtype=np.float16)
        with self._lock:
            rc = self.lib.wl_test_spk_conv(self.ctx, _lib.ptr(x16.view(np.uint16), C.c_uint16), _lib.ptr(fr, C.c_int64), len(fr),
                                           int(H_in), C_in, C_out, k, int(stride), _lib.ptr(w16.view(np.uint16), C.c_uint16),
                                           _lib.ptr(b32, C.c_float),
                                           None if r16 is None else _lib.ptr(r16.view(np.uint16), C.c_uint16), int(relu),
                                           _lib.ptr(o16.view(np.uint16), C.c_uint16))
            _lib.check(self.lib, self.ctx, rc, "wl_test_spk_conv")
        return o16

    def profile_cross_attn(self, enable: bool) -> None:
        """Bracket every cross-attention launch of graph-less generate calls with CUDA events (bench.py roofline)."""
        _lib.check(self.lib, self.ctx, self.lib.wl_profile_cross_attn(self.ctx, int(bool(enable))), "wl_profile_cross_attn")

    @staticmethod
    def _release_slots(engine_ref, slots):
        eng = engine_ref()
        if eng is None or not eng._fin.alive:
            return
        arr = np.asarray(slots, dtype=np.int32)
        with eng._lock:
            eng.lib.wl_slots_release(eng.ctx, _lib.ptr(arr, C.c_int32), len(slots))

    def free_slots(self) -> int:
        return int(self.lib.wl_slots_free_count(self.ctx))

    def _encoder_output(self, slot: int) -> np.ndarray:
        out = np.empty((1500, self.dims.d_model), dtype=np.float32)
        with self._lock:
            _lib.check(self.lib, self.ctx, self.lib.wl_encoder_output(self.ctx, slot, _lib.ptr(out, C.c_float)), "wl_encoder_output")
        return out

    # ------------------------------------------------------------------ K1 (used by FeatureExtractor)
    def mel(self, waveforms: Sequence[np.ndarray]) -> List[np.ndarray]:
        """log-mel of each waveform: float32 [n_mels, len//160 + 1] (the last frame is the one callers drop)."""
        outs: List[Optional[np.ndarray]] = [None] * len(waveforms)
        for i0 in range(0, len(waveforms), self.max_streams):
            chunk = [np.ascontiguousarray(w, dtype=np.float32) for w in waveforms[i0:i0 + self.max_streams]]
            lens = [len(w) for w in chunk]
            if min(lens) <= 0:
                raise ValueError("mel: empty waveform")
            off = np.zeros(len(chunk) + 1, dtype=np.int64)
            off[1:] = np.cumsum(lens)
            frames = [n // 160 + 1 for n in lens]
            ooff = np.zeros(len(chunk) + 1, dtype=np.int64)
            ooff[1:] = np.cumsum([f * self.n_mels for f in frames])
            pcm = np.concatenate(chunk)
            out = np.empty(int(ooff[-1]), dtype=np.float32)
            with self._lock:
                rc = self.lib.wl_mel(self.ctx, _lib.ptr(pcm, C.c_float), _lib.ptr(off, C.c_int64), len(chunk),
                                     _lib.ptr(out, C.c_float), _lib.ptr(ooff, C.c_int64))
                _lib.check(self.lib, self.ctx, rc, "wl_mel")
            for j, f in enumerate(frames):
                outs[i0 + j] = out[ooff[j]:ooff[j + 1]].reshape(self.n_mels, f)
        return outs  # type: ignore

    # ------------------------------------------------------------------ resident features (K1 -> K2 without leaving HBM)
    def mel_device(self, waveforms: Sequence[np.ndarray]) -> List[int]:
        """log-mel of up to ``max_streams`` waveforms, kept on the device until the next call; returns the frame
        count of each (len // 160 + 1, the last frame being the one callers drop).  Pair with ``encode_windows``."""
        chunk = [np.ascontiguousarray(w, dtype=np.float32) for w in waveforms]
        if not chunk or len(chunk) > self.max_streams:
            raise ValueError(f"mel_device takes 1..{self.max_streams} waveforms, got {len(chunk)}")
        if min(len(w) for w in chunk) <= 0:
            raise ValueError("mel: empty waveform")
        off = np.zeros(len(chunk) + 1, dtype=np.int64)
        off[1:] = np.cumsum([len(w) for w in chunk])
        pcm = np.concatenate(chunk)
        frames = np.zeros(len(chunk), dtype=np.int32)
        with self._lock:
            rc = self.lib.wl_mel_device(self.ctx, _lib.ptr(pcm, C.c_float), _lib.ptr(off, C.c_int64), len(chunk), _lib.ptr(frames, C.c_int32))
            _lib.check(self.lib, self.ctx, rc, "wl_mel_device")
            self._resident_epoch = getattr(self, "_resident_epoch", 0) + 1
        return [int(f) for f in frames]

    def encode_windows(self, windows: Sequence[Tuple[int, int, int]]) -> EncoderOutput:
        """Encode windows ``(stream, seek, length)`` cut from the resident log-mel (zero-padded to 3000 frames on the
        device, what ``pad_or_trim`` does on the host in the reference, transcriber_faster_whisper.py:1127)."""
        slots_all: List[int] = []
        with self._lock:
            free = self.free_slots()
            if len(windows) > free:
                raise RuntimeError(f"encode: {len(windows)} windows requested but only {free} encoder slots are free")
            for b0 in range(0, len(windows), self.max_streams):
                part = windows[b0:b0 + self.max_streams]
                arr = np.asarray(part, dtype=np.int32).reshape(-1, 3)
                st, sk, ln = (np.ascontiguousarray(arr[:, i]) for i in range(3))
                slots = np.zeros(len(part), dtype=np.int32)
                rc = self.lib.wl_encode_windows(self.ctx, len(part), _lib.ptr(st, C.c_int32), _lib.ptr(sk, C.c_int32),
                                                _lib.ptr(ln, C.c_int32), _lib.ptr(slots, C.c_int32))
                if rc != 0 and slots_all:
                    a = np.asarray(slots_all, dtype=np.int32)
                    self.lib.wl_slots_release(self.ctx, _lib.ptr(a, C.c_int32), len(slots_all))
                _lib.check(self.lib, self.ctx, rc, "wl_encode_windows")
                slots_all.extend(int(x) for x in slots)
        return EncoderOutput(_SlotRef(self, slots_all), slots_all, self.dims.d_model)

    # ------------------------------------------------------------------ ctranslate2.models.Whisper.encode
    def encode(self, features, to_cpu: bool = False) -> EncoderOutput:
        f = np.ascontiguousarray(np.asarray(features), dtype=np.float32)
        if f.ndim == 2:
            f = f[None]
        if f.ndim != 3 or f.shape[1] != self.n_mels or f.shape[2] != 3000:
            raise ValueError(f"encode expects [batch, {self.n_mels}, 3000] features, got {f.shape}")
        slots_all: List[int] = []
        with self._lock:
            free = self.free_slots()
            if f.shape[0] > free:
                raise RuntimeError(f"encode: {f.shape[0]} windows requested but only {free} encoder slots are free "
                                   f"(pool of {self.enc_slots}; release earlier EncoderOutput handles or encode in groups "
                                   f"of at most max_streams={self.max_streams})")
            for b0 in range(0, f.shape[0], self.max_streams):
                part = f[b0:b0 + self.max_streams]
                slots = np.zeros(part.shape[0], dtype=np.int32)
                rc = self.lib.wl_encode(self.ctx, _lib.ptr(part, C.c_float), part.shape[0], _lib.ptr(slots, C.c_int32))
                if rc != 0 and slots_all:
                    arr = np.asarray(slots_all, dtype=np.int32)
                    self.lib.wl_slots_release(self.ctx, _lib.ptr(arr, C.c_int32), len(slots_all))
                _lib.check(self.lib, self.ctx, rc, "wl_encode")
                slots_all.extend(int(s) for s in slots)
        return EncoderOutput(_SlotRef(self, slots_all), slots_all, self.dims.d_model)

    def _as_encoded(self, features) -> EncoderOutput:
        return features if isinstance(features, EncoderOutput) else self.encode(features)

    # ------------------------------------------------------------------ ctranslate2.models.Whisper.generate
    def generate(self, features, prompts: Sequence[Sequence[int]], *, beam_size: int = 5, patience: float = 1,
                 num_hypotheses: int = 1, length_penalty: float = 1, repetition_penalty: float = 1,
                 no_repeat_ngram_size: int = 0, max_length: int = 448, return_scores: bool = False,
                 return_no_speech_prob: bool = False, max_initial_timestamp_index: int = 50, suppress_blank: bool = True,
                 suppress_tokens: Optional[Sequence[int]] = (-1,), sampling_topk: int = 1, sampling_temperature: float = 1,
                 seed: Optional[int] = None, max_length_per_stream: Optional[Sequence[int]] = None,
                 prefill: Optional[bool] = None) -> List[WhisperGenerationResult]:
        if repetition_penalty != 1 or no_repeat_ngram_size != 0:
            raise NotImplementedError("repetition_penalty / no_repeat_ngram_size other than the reference's 1 / 0")
        if seed is None:
            # like CT2's generator state, the noise advances from one sampling call to the next: the rungs of the
            # temperature ladder and successive windows never replay each other's draws
            if int(beam_size) == 1 and sampling_topk != 1 and sampling_temperature > 0:
                self._sampling_calls = getattr(self, "_sampling_calls", 0) + 1
            seed = getattr(self, "_sampling_calls", 0)
        enc = self._as_encoded(features)
        if len(prompts) != len(enc):
            raise ValueError(f"{len(prompts)} prompts for {len(enc)} encoded streams")
        sup = np.asarray(sorted({int(t) for t in (suppress_tokens or ()) if t >= 0}), dtype=np.int32)
        results: List[WhisperGenerationResult] = []
        NH = int(num_hypotheses)
        for b0 in range(0, len(prompts), self.max_streams):
            ps = [list(map(int, p)) for p in prompts[b0:b0 + self.max_streams]]
            B = len(ps)
            off = np.zeros(B + 1, dtype=np.int32)
            off[1:] = np.cumsum([len(p) for p in ps])
            flat = np.asarray([t for p in ps for t in p], dtype=np.int32)
            slots = np.asarray(enc.slots[b0:b0 + B], dtype=np.int32)
            opts = _gen_opts(beam_size, patience, NH, length_penalty, max_length, suppress_blank, max_initial_timestamp_index,
                             sampling_topk, sampling_temperature, seed, sup, self.use_cuda_graph, prefill)
            mlps = None
            if max_length_per_stream is not None:
                mlps = np.asarray(list(max_length_per_stream)[b0:b0 + B], dtype=np.int32)
                opts.max_length_per_stream = _lib.ptr(mlps, C.c_int32)
            ids = np.zeros((B, NH, T_MAX), dtype=np.int32)
            lens = np.zeros((B, NH), dtype=np.int32)
            score = np.zeros((B, NH), dtype=np.float32)
            nsp = np.zeros(B, dtype=np.float32)
            steps = np.zeros(B, dtype=np.int32)
            with self._lock:
                rc = self.lib.wl_generate(self.ctx, _lib.ptr(slots, C.c_int32), B, _lib.ptr(flat, C.c_int32),
                                          _lib.ptr(off, C.c_int32), C.byref(opts), _lib.ptr(ids, C.c_int32),
                                          _lib.ptr(lens, C.c_int32), _lib.ptr(score, C.c_float), _lib.ptr(nsp, C.c_float),
                                          _lib.ptr(steps, C.c_int32))
                _lib.check(self.lib, self.ctx, rc, "wl_generate")
            for b in range(B):
                seqs, scs = [], []
                for h in range(NH):
                    if lens[b, h] >= 0:
                        seqs.append(ids[b, h, :lens[b, h]].tolist())
                        scs.append(float(score[b, h]))
                results.append(WhisperGenerationResult(seqs, scs, float(nsp[b]), int(steps[b])))
        self.last_steps = max((r.steps for r in results), default=0)
        return results

    # ------------------------------------------------------------------ N2: decode session (step-level admission)
    def open_decode_session(self, capacity: Optional[int] = None, **generate_kwargs) -> "DecodeSession":
        """A decode loop whose streams come and go independently (``wl_session_*``): same keyword arguments as
        ``generate`` (``max_length`` is given per stream at admission; the session's own search does not sample, a
        stream samples when ``DecodeSession.admit`` is given a ``sampling`` spec for it)."""
        # one session per engine context: whatever an earlier owner left behind (a scheduler stopped mid-decode) is dropped
        with self._lock:
            rc = self.lib.wl_session_close(self.ctx)
            _lib.check(self.lib, self.ctx, rc, "wl_session_close")
        return DecodeSession(self, capacity or self.max_streams, **generate_kwargs)

    # ------------------------------------------------------------------ ctranslate2.models.Whisper.detect_language
    def detect_language(self, features) -> List[List[Tuple[str, float]]]:
        if not self.is_multilingual:
            raise RuntimeError("detect_language can only be called on multilingual models")
        enc = self._as_encoded(features)
        n_lang = self.num_languages
        out: List[List[Tuple[str, float]]] = []
        for b0 in range(0, len(enc), self.max_streams):
            slots = np.asarray(enc.slots[b0:b0 + self.max_streams], dtype=np.int32)
            probs = np.zeros((len(slots), n_lang), dtype=np.float32)
            with self._lock:
                rc = self.lib.wl_detect_language(self.ctx, _lib.ptr(slots, C.c_int32), len(slots), _lib.ptr(probs, C.c_float))
                _lib.check(self.lib, self.ctx, rc, "wl_detect_language")
            for p in probs:
                order = np.lexsort((np.arange(n_lang), -p))
                out.append([(f"<|{LANGUAGE_CODES[i]}|>", float(p[i])) for i in order])
        return out

    # ------------------------------------------------------------------ ctranslate2.models.Whisper.align
    def align(self, features, start_sequence: Sequence[int], text_tokens: Sequence[Sequence[int]],
              num_frames: Union[int, Sequence[int]], *, median_filter_width: int = 7) -> List[WhisperAlignmentResult]:
        enc = self._as_encoded(features)
        if len(text_tokens) != len(enc):
            raise ValueError(f"{len(text_tokens)} token lists for {len(enc)} encoded streams")
        out: List[WhisperAlignmentResult] = []
        start = np.asarray(list(start_sequence), dtype=np.int32)
        for b0 in range(0, len(enc), self.max_streams):
            tt = [list(map(int, t)) for t in text_tokens[b0:b0 + self.max_streams]]
            B = len(tt)
            slots = np.asarray(enc.slots[b0:b0 + B], dtype=np.int32)
            toff = np.zeros(B + 1, dtype=np.int32)
            toff[1:] = np.cumsum([len(t) for t in tt])
            flat = np.asarray([x for t in tt for x in t] or [0], dtype=np.int32)
            nf = np.asarray([num_frames] * B if isinstance(num_frames, (int, np.integer)) else list(num_frames)[b0:b0 + B],
                            dtype=np.int32)
            cap = int(sum(len(t) + 1 + max(1, int(f) // 2) for t, f in zip(tt, nf)) + 8)
            pairs = np.zeros((cap, 2), dtype=np.int32)
            poff = np.zeros(B + 1, dtype=np.int32)
            probs = np.zeros(max(1, int(toff[-1])), dtype=np.float32)
            with self._lock:
                rc = self.lib.wl_align(self.ctx, _lib.ptr(slots, C.c_int32), B, _lib.ptr(start, C.c_int32), len(start),
                                       _lib.ptr(flat, C.c_int32), _lib.ptr(toff, C.c_int32), _lib.ptr(nf, C.c_int32),
                                       int(median_filter_width), _lib.ptr(pairs, C.c_int32), cap, _lib.ptr(poff, C.c_int32),
                                       _lib.ptr(probs, C.c_float))
                _lib.check(self.lib, self.ctx, rc, "wl_align")
            for b in range(B):
                al = [(int(a), int(t)) for a, t in pairs[poff[b]:poff[b + 1]]]
                out.append(WhisperAlignmentResult(al, probs[toff[b]:toff[b + 1]].tolist()))
        return out

    # ------------------------------------------------------------------ parity hooks
    def decode_logits(self, features, token_lists: Sequence[Sequence[int]]) -> List[np.ndarray]:
        """Teacher-forced logits [T, vocab] per stream (test hook: wl_decode_logits)."""
        enc = self._as_encoded(features)
        tl = [list(map(int, t)) for t in token_lists]
        B = len(tl)
        off = np.zeros(B + 1, dtype=np.int32)
        off[1:] = np.cumsum([len(t) for t in tl])
        flat = np.asarray([x for t in tl for x in t], dtype=np.int32)
        slots = np.asarray(enc.slots, dtype=np.int32)
        out = np.zeros((int(off[-1]), self.dims.vocab), dtype=np.float32)
        with self._lock:
            rc = self.lib.wl_decode_logits(self.ctx, _lib.ptr(slots, C.c_int32), B, _lib.ptr(flat, C.c_int32),
                                           _lib.ptr(off, C.c_int32), _lib.ptr(out, C.c_float))
            _lib.check(self.lib, self.ctx, rc, "wl_decode_logits")
        return [out[off[b]:off[b + 1]] for b in range(B)]

    def test_search(self, prompts: Sequence[Sequence[int]], script: Tuple[int, int], *, beam_size: int = 5, patience: float = 1,
                    num_hypotheses: int = 1, length_penalty: float = 1, max_length: int = 448,
                    max_initial_timestamp_index: int = 50, suppress_blank: bool = True,
                    suppress_tokens: Optional[Sequence[int]] = (), sampling_topk: int = 1, sampling_temperature: float = 1,
                    seed: int = 0, max_length_per_stream: Optional[Sequence[int]] = None, prefill: Optional[bool] = None,
                    use_cuda_graph: Optional[bool] = None, return_logits: bool = False
                    ) -> Tuple[List[WhisperGenerationResult], List[int], Optional[np.ndarray]]:
        """``generate`` on scripted logits (wl_test_search): ``script = (seed, pattern)`` of the function that
        tests/search_script.py restates replaces the decoder; no encoder output is needed.  At most ``max_streams``
        prompts.  Returns the results, the hypothesis count of every stream and, with ``return_logits``, the logits of
        the first decode step [B * rows per stream, (vocab + 3) // 4 * 4]."""
        ps = [list(map(int, p)) for p in prompts]
        B = len(ps)
        if not 1 <= B <= self.max_streams:
            raise ValueError(f"{B} prompts for max_streams={self.max_streams}")
        NH = int(num_hypotheses)
        Kr = int(beam_size) if int(beam_size) > 1 else NH
        off = np.zeros(B + 1, dtype=np.int32)
        off[1:] = np.cumsum([len(p) for p in ps])
        flat = np.asarray([t for p in ps for t in p], dtype=np.int32)
        sup = np.asarray(sorted({int(t) for t in (suppress_tokens or ()) if t >= 0}), dtype=np.int32)
        graph = self.use_cuda_graph if use_cuda_graph is None else use_cuda_graph
        opts = _gen_opts(beam_size, patience, NH, length_penalty, max_length, suppress_blank, max_initial_timestamp_index,
                         sampling_topk, sampling_temperature, seed, sup, graph, prefill)
        mlps = None
        if max_length_per_stream is not None:
            mlps = np.asarray(list(max_length_per_stream), dtype=np.int32)
            opts.max_length_per_stream = _lib.ptr(mlps, C.c_int32)
        sc = _lib.WlSearchScript(seed=int(script[0]) & 0xFFFFFFFF, pattern=int(script[1]))
        ids = np.zeros((B, NH, T_MAX), dtype=np.int32)
        lens = np.zeros((B, NH), dtype=np.int32)
        score = np.zeros((B, NH), dtype=np.float32)
        nsp = np.zeros(B, dtype=np.float32)
        steps = np.zeros(B, dtype=np.int32)
        nhyp = np.zeros(B, dtype=np.int32)
        logits = np.empty((B * Kr, (self.dims.vocab + 3) // 4 * 4), dtype=np.float32) if return_logits else None
        with self._lock:
            rc = self.lib.wl_test_search(self.ctx, B, _lib.ptr(flat, C.c_int32), _lib.ptr(off, C.c_int32), C.byref(opts),
                                         C.byref(sc), _lib.ptr(ids, C.c_int32), _lib.ptr(lens, C.c_int32),
                                         _lib.ptr(score, C.c_float), _lib.ptr(nsp, C.c_float), _lib.ptr(steps, C.c_int32),
                                         _lib.ptr(nhyp, C.c_int32), None if logits is None else _lib.ptr(logits, C.c_float))
            _lib.check(self.lib, self.ctx, rc, "wl_test_search")
        results = []
        for b in range(B):
            keep = [h for h in range(NH) if lens[b, h] >= 0]
            results.append(WhisperGenerationResult([ids[b, h, :lens[b, h]].tolist() for h in keep],
                                                   [float(score[b, h]) for h in keep], float(nsp[b]), int(steps[b])))
        return results, nhyp.tolist(), logits

    def test_wgemm(self, w: np.ndarray, x: np.ndarray, bias: Optional[np.ndarray] = None, mode: int = 0,
                   resid: Optional[np.ndarray] = None) -> np.ndarray:
        """Y[R, n_out] = X[R, K] W[n_out, K]^T through the small-batch decode GEMM (wl_test_wgemm) with epilogue ``mode``."""
        w16 = np.ascontiguousarray(w, dtype=np.float16)
        x16 = np.ascontiguousarray(x, dtype=np.float16)
        n_out, K = w16.shape
        R = x16.shape[0]
        out = np.zeros((R, n_out), dtype=np.float32) if resid is None else np.ascontiguousarray(resid, dtype=np.float32).copy()
        bp = None
        if bias is not None:
            bias = np.ascontiguousarray(bias, dtype=np.float32)
            bp = _lib.ptr(bias, C.c_float)
        with self._lock:
            rc = self.lib.wl_test_wgemm(self.ctx, _lib.ptr(w16.view(np.uint16), C.c_uint16), _lib.ptr(x16.view(np.uint16), C.c_uint16),
                                        bp, _lib.ptr(out, C.c_float), R, n_out, K, int(mode))
            _lib.check(self.lib, self.ctx, rc, "wl_test_wgemm")
        return out

    def test_dec_gemm(self, w: np.ndarray, x: np.ndarray, nsplit: int = 0) -> Tuple[np.ndarray, int]:
        """Raw K-range partial sums [nsplit, R, n_out] of X[R, K] W[n_out, K]^T through the split-K decode GEMM
        (wl_test_dec_gemm) and the split used; ``nsplit=0`` takes the engine's plan."""
        w16 = np.ascontiguousarray(w, dtype=np.float16)
        x16 = np.ascontiguousarray(x, dtype=np.float16)
        n_out, K = w16.shape
        R = x16.shape[0]
        used = C.c_int32()
        wp, xp = _lib.ptr(w16.view(np.uint16), C.c_uint16), _lib.ptr(x16.view(np.uint16), C.c_uint16)
        with self._lock:
            rc = self.lib.wl_test_dec_gemm(self.ctx, wp, xp, None, R, n_out, K, int(nsplit), C.byref(used))
            _lib.check(self.lib, self.ctx, rc, "wl_test_dec_gemm")
            out = np.empty((used.value, R, n_out), dtype=np.float32)
            rc = self.lib.wl_test_dec_gemm(self.ctx, wp, xp, _lib.ptr(out, C.c_float), R, n_out, K, used.value, C.byref(used))
            _lib.check(self.lib, self.ctx, rc, "wl_test_dec_gemm")
        return out, used.value

    def test_cross_attn(self, q_part: np.ndarray, q_bias: Optional[np.ndarray], k_pool: np.ndarray, v_pool: np.ndarray,
                        slot: Sequence[int], done: Sequence[int], rows_per_stream: int, nsplit: int = 0,
                        sentinel: float = 0.0, probs: bool = False) -> Tuple[np.ndarray, Optional[np.ndarray], int]:
        """K11 cross attention (wl_test_cross_attn).  q_part [q_nsplit, R, H*64] fp32; k_pool / v_pool fp16
        [n_slots, H, 1500, 64] already in the swizzled pool layout.  Returns (out [R, H*64], probs [R, H, 1500] or None,
        key split used)."""
        qp = np.ascontiguousarray(q_part, dtype=np.float32)
        kp = np.ascontiguousarray(k_pool, dtype=np.float16)
        vp = np.ascontiguousarray(v_pool, dtype=np.float16)
        n_slots, H = kp.shape[:2]
        sl = np.ascontiguousarray(slot, dtype=np.int32)
        dn = np.ascontiguousarray(done, dtype=np.int32)
        B = len(sl)
        R = B * rows_per_stream
        out = np.empty((R, H * 64), dtype=np.float32)
        pr = np.empty((R, H, 1500), dtype=np.float32) if probs else None
        bp = None
        if q_bias is not None:
            q_bias = np.ascontiguousarray(q_bias, dtype=np.float32)
            bp = _lib.ptr(q_bias, C.c_float)
        used = C.c_int32()
        with self._lock:
            rc = self.lib.wl_test_cross_attn(self.ctx, _lib.ptr(qp, C.c_float), bp, qp.shape[0],
                                             _lib.ptr(kp.view(np.uint16), C.c_uint16), _lib.ptr(vp.view(np.uint16), C.c_uint16),
                                             n_slots, _lib.ptr(sl, C.c_int32), _lib.ptr(dn, C.c_int32), B, rows_per_stream, H,
                                             int(nsplit), C.byref(used), float(sentinel), _lib.ptr(out, C.c_float),
                                             None if pr is None else _lib.ptr(pr, C.c_float))
            _lib.check(self.lib, self.ctx, rc, "wl_test_cross_attn")
        return out, pr, used.value

    def test_self_attn(self, qkv_part: np.ndarray, qkv_bias: Optional[np.ndarray], k_cache: np.ndarray, v_cache: np.ndarray,
                       src: np.ndarray, pos: Sequence[int], active: Sequence[int], wrow: Optional[Sequence[int]] = None,
                       sentinel: float = 0.0) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """K10 self attention (wl_test_self_attn).  qkv_part [nsplit, R, 3*H*64] fp32 (nsplit 1 without a bias: the plain
        form); caches fp16 [n_rows, H, 448, 64]; src [R, 448].  Returns (out [R, H*64], k cache, v cache) after the call."""
        qp = np.ascontiguousarray(qkv_part, dtype=np.float32)
        kc = np.ascontiguousarray(k_cache, dtype=np.float16).copy()
        vc = np.ascontiguousarray(v_cache, dtype=np.float16).copy()
        n_rows, H = kc.shape[:2]
        R = qp.shape[1]
        sr = np.ascontiguousarray(src, dtype=np.int16)
        ps = np.ascontiguousarray(pos, dtype=np.int32)
        ac = np.ascontiguousarray(active, dtype=np.int32)
        wr = None if wrow is None else np.ascontiguousarray(wrow, dtype=np.int32)
        out = np.empty((R, H * 64), dtype=np.float32)
        bp = None
        if qkv_bias is not None:
            qkv_bias = np.ascontiguousarray(qkv_bias, dtype=np.float32)
            bp = _lib.ptr(qkv_bias, C.c_float)
        with self._lock:
            rc = self.lib.wl_test_self_attn(self.ctx, _lib.ptr(qp, C.c_float), bp, qp.shape[0],
                                            _lib.ptr(kc.view(np.uint16), C.c_uint16), _lib.ptr(vc.view(np.uint16), C.c_uint16),
                                            n_rows, _lib.ptr(sr, C.c_int16), _lib.ptr(ps, C.c_int32), _lib.ptr(ac, C.c_int32),
                                            None if wr is None else _lib.ptr(wr, C.c_int32), R, H, float(sentinel),
                                            _lib.ptr(out, C.c_float))
            _lib.check(self.lib, self.ctx, rc, "wl_test_self_attn")
        return out, kc, vc

    def test_layernorm_update(self, x: np.ndarray, part: Optional[np.ndarray], bias: Optional[np.ndarray], gamma: np.ndarray,
                              beta: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        """x += bias + the partials [nsplit, rows, d] (none when ``part`` is None), y = LayerNorm(x) as fp16
        (wl_test_fold mode 0).  Returns (updated x, y)."""
        x = np.ascontiguousarray(x, dtype=np.float32).copy()
        rows, d = x.shape
        y = np.empty_like(x)
        self._fold(0, x, part, bias, np.ascontiguousarray(gamma, dtype=np.float32), np.ascontiguousarray(beta, dtype=np.float32),
                   y, rows, d)
        return x, y

    def test_gelu_cast(self, part: np.ndarray, bias: Optional[np.ndarray]) -> np.ndarray:
        """fp16(gelu(bias + the partials [nsplit, rows, cols])) (wl_test_fold mode 1)."""
        _, rows, cols = part.shape
        y = np.empty((rows, cols), dtype=np.float32)
        self._fold(1, None, part, bias, None, None, y, rows, cols)
        return y

    def _fold(self, mode, x, part, bias, gamma, beta, y, rows, cols):
        fp = lambda a: None if a is None else _lib.ptr(a, C.c_float)
        part = None if part is None else np.ascontiguousarray(part, dtype=np.float32)
        bias = None if bias is None else np.ascontiguousarray(bias, dtype=np.float32)
        with self._lock:
            rc = self.lib.wl_test_fold(self.ctx, mode, fp(x), fp(part), 0 if part is None else part.shape[0], fp(bias), fp(gamma),
                                       fp(beta), fp(y), rows, cols)
            _lib.check(self.lib, self.ctx, rc, "wl_test_fold")

    def test_enc_attn(self, qk: np.ndarray, vt: np.ndarray, out: np.ndarray, path: int, ab: int = 0) -> np.ndarray:
        """Encoder self-attention (wl_test_enc_attn).  qk fp16 [nb, 1500, 2*H*64] (Q | K); vt fp16 [nb, H*64, 1536] (V^T
        per head, pad columns as given); out fp16 [nb*1500 + 128, H*64], the buffer as it is before the launch.  path 0:
        the fused kernel; 1: the unfused sequence in sub-passes of ``ab`` streams (0: the engine's rule).  Returns the
        whole output buffer after the launch, guard rows included."""
        qk16 = np.ascontiguousarray(qk, dtype=np.float16)
        vt16 = np.ascontiguousarray(vt, dtype=np.float16)
        o16 = np.ascontiguousarray(out, dtype=np.float16).copy()
        nb, d = qk16.shape[0], qk16.shape[2] // 2
        assert qk16.shape == (nb, 1500, 2 * d) and vt16.shape == (nb, d, 1536) and o16.shape == (nb * 1500 + 128, d)
        with self._lock:
            rc = self.lib.wl_test_enc_attn(self.ctx, _lib.ptr(qk16.view(np.uint16), C.c_uint16), _lib.ptr(vt16.view(np.uint16), C.c_uint16),
                                           _lib.ptr(o16.view(np.uint16), C.c_uint16), nb, d // 64, int(path), int(ab))
            _lib.check(self.lib, self.ctx, rc, "wl_test_enc_attn")
        return o16

    def test_enc_stem(self, feats: np.ndarray) -> np.ndarray:
        """The conv stem with this model's weights (wl_test_enc_stem): features [nb, n_mels, 3000] -> the fp32 residual
        stream [nb, 1500, d] after conv2 + GELU + the positional table."""
        f = np.ascontiguousarray(feats, dtype=np.float32)
        nb = f.shape[0]
        assert f.shape == (nb, self.dims.n_mels, 3000)
        x = np.empty((nb, 1500, self.dims.d_model), dtype=np.float32)
        with self._lock:
            rc = self.lib.wl_test_enc_stem(self.ctx, _lib.ptr(f, C.c_float), _lib.ptr(x, C.c_float), nb)
            _lib.check(self.lib, self.ctx, rc, "wl_test_enc_stem")
        return x

    def test_layernorm(self, x: np.ndarray, gamma: np.ndarray, beta: np.ndarray, y16: Optional[np.ndarray],
                       y32: Optional[np.ndarray]) -> Tuple[Optional[np.ndarray], Optional[np.ndarray]]:
        """layernorm_rows (wl_test_layernorm) over x [rows, d].  y16 / y32: [rows + 8, d] buffers as they are before the
        launch (y16 is rounded to fp16), or None to skip that output.  Returns both buffers after the launch, guard rows
        included."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        rows, d = x.shape
        bufs = [None if y is None else np.ascontiguousarray(y, dtype=np.float32).copy() for y in (y16, y32)]
        for y in bufs:
            assert y is None or y.shape == (rows + 8, d)
        g = np.ascontiguousarray(gamma, dtype=np.float32)
        b = np.ascontiguousarray(beta, dtype=np.float32)
        fp = lambda a: None if a is None else _lib.ptr(a, C.c_float)
        with self._lock:
            rc = self.lib.wl_test_layernorm(self.ctx, fp(x), fp(g), fp(b), fp(bufs[0]), fp(bufs[1]), rows, d)
            _lib.check(self.lib, self.ctx, rc, "wl_test_layernorm")
        return bufs[0], bufs[1]

    GEMM_OUT = {"f32": 0, "resid": 1, "f16": 2, "headsplit": 3}
    GEMM_VARIANT = {"auto": 0, "classic": 1, "pingpong": 2}

    def test_gemm(self, a: np.ndarray, b: np.ndarray, bias: Optional[np.ndarray] = None, transposed_store: bool = False,
                  gelu: bool = False, use_simt: bool = False, out: str = "f32", resid: Optional[np.ndarray] = None,
                  batch: Optional[int] = None, hs_rows: int = 0, variant: str = "auto", bias_on_m: bool = False) -> np.ndarray:
        """C[z] = A[z] @ B[z]^T through the wgmma kernel (or the CUDA-core checker).

        out: "f32"; "resid" (C += the fp32 `resid`, in place); "f16"; "headsplit" (fp16 cross-KV layout of `hs_rows`
        rows per stream, returned raw: [slot][N / 64][hs_rows][64], slots in reverse stream order, see wlb200.h).
        batch: Z when one of a, b is a single 2-D matrix shared by the batch.  variant: "auto", "classic", "pingpong".
        bias_on_m: bias indexed by m (implied by transposed_store)."""
        a16 = np.ascontiguousarray(a, dtype=np.float16)
        b16 = np.ascontiguousarray(b, dtype=np.float16)
        if batch is None:
            if a16.ndim == 2:
                a16, b16 = a16[None], b16[None]
            Z = a16.shape[0]
        else:
            Z = batch
        a_shared, b_shared = a16.ndim == 2, b16.ndim == 2
        M, K = a16.shape[-2:]
        N = b16.shape[-2]
        if resid is not None:
            c = np.ascontiguousarray(resid, dtype=np.float32).reshape((Z, N, M) if transposed_store else (Z, M, N)).copy()
        else:
            c = np.zeros((Z, N, M) if transposed_store else (Z, M, N), dtype=np.float32)
        opts = (self.GEMM_OUT[out] | (4 if a_shared else 0) | (8 if b_shared else 0) | (self.GEMM_VARIANT[variant] << 4)
                | (64 if bias_on_m else 0) | (hs_rows << 8))
        bp = None
        if bias is not None:
            bias = np.ascontiguousarray(bias, dtype=np.float32)
            bp = _lib.ptr(bias, C.c_float)
        with self._lock:
            rc = self.lib.wl_test_gemm(self.ctx, _lib.ptr(a16.view(np.uint16), C.c_uint16), _lib.ptr(b16.view(np.uint16), C.c_uint16),
                                       bp, _lib.ptr(c, C.c_float), M, N, K, Z, int(transposed_store), int(gelu), int(use_simt),
                                       opts)
            _lib.check(self.lib, self.ctx, rc, "wl_test_gemm")
        return c

    def gemm_variant(self, M: int, N: int, K: int, batch: int = 1) -> str:
        """Which GEMM kernel the library picks for this shape on this device: "classic" or "pingpong"."""
        v = C.c_int32()
        with self._lock:
            rc = self.lib.wl_gemm_variant(self.ctx, M, N, K, batch, C.byref(v))
            _lib.check(self.lib, self.ctx, rc, "wl_gemm_variant")
        return {1: "classic", 2: "pingpong"}[v.value]


# the generate keywords a stream may bring to a decode session of its own (DecodeSession.admit(rules=...))
STREAM_RULE_KEYS = ("suppress_tokens", "suppress_blank", "max_initial_timestamp_index", "length_penalty", "patience",
                    "beam_size")


class DecodeSession:
    """Step-level continuous batching on one engine context (``include/wlb200.h``: ``wl_session_*``).

    The reference's batcher runs a batch to completion before it looks at the queue again
    (whisper_live/batch_inference.py:155-187); here a stream is admitted at any token-step boundary into a free index
    of the running decode loop, and a finished stream is collected while the others keep decoding:

        sess = engine.open_decode_session(beam_size=5, suppress_tokens=...)
        idx = sess.admit([enc_a, enc_b], [prompt_a, prompt_b], [448, 448])
        while sess.live:
            for i in sess.run(max_steps=16):        # returns early when a stream finishes
                result = sess.collect(i)            # WhisperGenerationResult, the index is free again
            ... admit whoever arrived meanwhile ...

    One-shot engine calls (``encode``, ``generate``, ``align``, ``detect_language``) may be interleaved between two
    ``run`` calls: the session owns its decode state and self-attention cache.

    The session's own search is beam or greedy.  A stream may instead be admitted for Gumbel-max sampling (a
    temperature-fallback rung): ``admit(..., sampling=[(temperature, num_hypotheses, seed, noise_key), ...])`` decodes it
    over ``num_hypotheses <= rows_per_stream`` independent rows with exactly the draws ``generate(seed=seed)`` gives the
    stream at batch position ``noise_key``, whoever else is in the loop.  A stream admitted with ``rules`` brings its
    own logits rules, length penalty, patience and beam width (``beam_size <= rows_per_stream``; width 1 is greedy)."""

    def __init__(self, engine: B200Whisper, capacity: int, *, beam_size: int = 5, patience: float = 1, num_hypotheses: int = 1,
                 length_penalty: float = 1, repetition_penalty: float = 1, no_repeat_ngram_size: int = 0,
                 max_initial_timestamp_index: int = 50, suppress_blank: bool = True,
                 suppress_tokens: Optional[Sequence[int]] = (-1,), sampling_topk: int = 1, sampling_temperature: float = 1,
                 return_scores: bool = False, return_no_speech_prob: bool = False, max_length: int = T_MAX, **_ignored):
        if repetition_penalty != 1 or no_repeat_ngram_size != 0:
            raise NotImplementedError("repetition_penalty / no_repeat_ngram_size other than the reference's 1 / 0")
        if int(beam_size) == 1 and sampling_topk != 1 and sampling_temperature > 0:
            raise ValueError("a decode session's own search does not sample: pass sampling= per stream to admit()")
        self.engine = engine
        self.capacity = int(capacity)
        self.num_hypotheses = int(num_hypotheses)
        # decoder rows per stream: the most hypotheses a sampled stream, or the widest beam a stream's rules, may ask for
        self.rows_per_stream = int(beam_size) if int(beam_size) > 1 else self.num_hypotheses
        self._nh: Dict[int, int] = {}                 # index -> hypotheses its stream returns
        self._sup = np.asarray(sorted({int(t) for t in (suppress_tokens or ()) if t >= 0}), dtype=np.int32)
        self._opts = _lib.WlGenOpts(
            beam_size=int(beam_size), patience=float(patience), num_hypotheses=self.num_hypotheses,
            length_penalty=float(length_penalty), max_length=int(max_length), suppress_blank=int(bool(suppress_blank)),
            max_initial_timestamp_index=int(max_initial_timestamp_index), sampling_topk=1, sampling_temperature=1.0, seed=0,
            suppress_tokens=_lib.ptr(self._sup, C.c_int32) if len(self._sup) else None, n_suppress=len(self._sup),
            use_cuda_graph=int(engine.use_cuda_graph), max_length_per_stream=None, prefill=1)
        self._held: Dict[int, Any] = {}               # index -> the encoder view its stream decodes against
        self.scripted = False
        self._finished: List[int] = []
        self.steps = 0
        self.runs = 0
        self.closed = False
        with engine._lock:
            rc = engine.lib.wl_session_open(engine.ctx, C.byref(self._opts), self.capacity)
            _lib.check(engine.lib, engine.ctx, rc, "wl_session_open")

    def script(self, script: Optional[Tuple[int, int]]) -> None:
        """Test hook (``wl_test_session_script``): decode the streams admitted from now on over the scripted logits
        ``(seed, pattern)`` of ``B200Whisper.test_search`` instead of the decoder; None goes back.  Only while nothing
        is in flight."""
        eng = self.engine
        sc = None if script is None else _lib.WlSearchScript(seed=int(script[0]) & 0xFFFFFFFF, pattern=int(script[1]))
        with eng._lock:
            rc = eng.lib.wl_test_session_script(eng.ctx, None if sc is None else C.byref(sc))
            _lib.check(eng.lib, eng.ctx, rc, "wl_test_session_script")
        self.scripted = script is not None

    # -- bookkeeping -------------------------------------------------------------------------------
    supports_rules = True            # admit(rules=...): per-stream logits rules

    @property
    def beam_size(self) -> int:
        return int(self._opts.beam_size)

    @property
    def live(self) -> int:
        """streams admitted and not yet collected"""
        return len(self._held)

    def free_indices(self) -> List[int]:
        return [i for i in range(self.capacity) if i not in self._held]

    # -- admission ---------------------------------------------------------------------------------
    def admit(self, features: Sequence[EncoderOutput], prompts: Sequence[Sequence[int]], max_lengths: Sequence[int],
              indices: Optional[Sequence[int]] = None,
              sampling: Optional[Sequence[Optional[Tuple[float, int, int, int]]]] = None,
              rules: Optional[Sequence[Optional[dict]]] = None) -> List[int]:
        """Admit one stream per (single-stream encoder view, prompt, max_length); returns the indices they decode in.
        ``sampling``: per stream None (the session's search) or ``(temperature, num_hypotheses, seed, noise_key)``.
        ``rules``: per stream None (the session's options) or a dict of ``generate`` keywords the stream decodes under
        instead -- ``suppress_tokens``, ``suppress_blank``, ``max_initial_timestamp_index``, ``length_penalty``,
        ``patience`` (missing keys take ``generate``'s defaults) and optionally ``beam_size``, from 1 (greedy) to
        ``rows_per_stream``: the stream decodes as ``generate(beam_size=...)`` would decode it alone, and ``collect`` /
        ``peek`` return its hypotheses.  ``features`` entries may be None when the session runs on scripted logits
        (``script``)."""
        n = len(prompts)
        if n == 0:
            return []
        if len(features) != n or len(max_lengths) != n or (sampling is not None and len(sampling) != n) or (
                rules is not None and len(rules) != n):
            raise ValueError("admit: features / prompts / max_lengths / sampling / rules differ in length")
        free = self.free_indices()
        if indices is None:
            if n > len(free):
                raise RuntimeError(f"admit: {n} streams for {len(free)} free indices")
            indices = free[:n]
        slots = []
        for f in features:
            if f is None and self.scripted:
                slots.append(0)
                continue
            if not isinstance(f, EncoderOutput) or len(f) != 1:
                raise TypeError("admit: every stream needs its own single-stream EncoderOutput view")
            slots.append(int(f.slots[0]))
        ps = [list(map(int, p)) for p in prompts]
        off = np.zeros(n + 1, dtype=np.int32)
        off[1:] = np.cumsum([len(p) for p in ps])
        flat = np.asarray([t for p in ps for t in p], dtype=np.int32)
        idx = np.asarray(list(indices), dtype=np.int32)
        sl = np.asarray(slots, dtype=np.int32)
        ml = np.asarray(list(max_lengths), dtype=np.int32)
        specs = list(sampling) if sampling is not None else [None] * n
        search = (_lib.WlStreamSearch * n)()
        for q, sp in zip(search, specs):
            if sp is not None:
                t, nh, seed, key = sp
                q.sample, q.num_hypotheses, q.temperature = 1, int(nh), float(t)
                q.seed, q.noise_key = int(seed) & 0xFFFFFFFF, int(key)
        rl = (_lib.WlStreamRules * n)()
        keep = []                                      # the suppress arrays the structs point into
        for q, r in zip(rl, rules if rules is not None else [None] * n):
            if r is not None:
                unknown = set(r) - set(STREAM_RULE_KEYS)
                if unknown:
                    raise ValueError(f"admit: {sorted(unknown)} cannot differ from stream to stream in a decode session")
                sup = np.asarray(sorted({int(t) for t in (r.get("suppress_tokens", (-1,)) or ()) if t >= 0}), dtype=np.int32)
                keep.append(sup)
                q.rules, q.beam_size = 1, int(r.get("beam_size", 0))
                q.patience, q.length_penalty = float(r.get("patience", 1)), float(r.get("length_penalty", 1))
                q.suppress_blank = int(bool(r.get("suppress_blank", True)))
                q.max_initial_timestamp_index = int(r.get("max_initial_timestamp_index", 50))
                q.suppress_tokens = _lib.ptr(sup, C.c_int32) if len(sup) else None
                q.n_suppress = len(sup)
        eng = self.engine
        with eng._lock:
            rc = eng.lib.wl_session_admit_ex(eng.ctx, n, _lib.ptr(idx, C.c_int32), _lib.ptr(sl, C.c_int32),
                                             _lib.ptr(flat, C.c_int32), _lib.ptr(off, C.c_int32), _lib.ptr(ml, C.c_int32),
                                             search if sampling is not None else None, rl if rules is not None else None)
            _lib.check(eng.lib, eng.ctx, rc, "wl_session_admit")
        for i, f, sp in zip(idx.tolist(), features, specs):
            self._held[i] = f
            self._nh[i] = self.num_hypotheses if sp is None else int(sp[1])
        return idx.tolist()

    # -- the token loop ----------------------------------------------------------------------------
    def run(self, max_steps: int = 16, break_on_finish: bool = True) -> List[int]:
        """Up to ``max_steps`` token steps over every admitted stream; returns the indices that are finished and waiting
        to be collected."""
        eng = self.engine
        done = np.zeros(self.capacity, dtype=np.int32)
        ran = C.c_int32(0)
        with eng._lock:
            rc = eng.lib.wl_session_run(eng.ctx, int(max_steps), int(bool(break_on_finish)), _lib.ptr(done, C.c_int32), C.byref(ran))
            _lib.check(eng.lib, eng.ctx, rc, "wl_session_run")
        self.steps += int(ran.value)
        self.runs += 1
        self.last_steps = int(ran.value)
        self._finished = [i for i in range(self.capacity) if done[i]]
        return list(self._finished)

    def collect(self, index: int) -> WhisperGenerationResult:
        eng = self.engine
        NH = self._nh.get(int(index), self.num_hypotheses)
        ids = np.zeros((NH, T_MAX), dtype=np.int32)
        lens = np.zeros(NH, dtype=np.int32)
        score = np.zeros(NH, dtype=np.float32)
        nsp = C.c_float(0.0)
        steps = C.c_int32(0)
        with eng._lock:
            rc = eng.lib.wl_session_collect(eng.ctx, int(index), _lib.ptr(ids, C.c_int32), _lib.ptr(lens, C.c_int32),
                                            _lib.ptr(score, C.c_float), C.byref(nsp), C.byref(steps))
            _lib.check(eng.lib, eng.ctx, rc, "wl_session_collect")
        self._held.pop(int(index), None)
        self._nh.pop(int(index), None)
        seqs, scs = [], []
        for h in range(NH):
            if lens[h] >= 0:
                seqs.append(ids[h, :lens[h]].tolist())
                scs.append(float(score[h]))
        return WhisperGenerationResult(seqs, scs, float(nsp.value), int(steps.value))

    def peek(self, indices: Sequence[int]) -> List[Tuple[List[int], float, float, int, bool]]:
        """Interim hypothesis of each index between two ``run`` calls: ``(tokens, score, no_speech_prob, step, final)``.
        A running stream reports its leading row (a beam stream's need not be a prefix of its final hypothesis), a
        finished one the hypothesis ``collect`` returns first, and stays collectable.  One kernel and one copy for all."""
        n = len(indices)
        if n == 0:
            return []
        idx = np.asarray(list(indices), dtype=np.int32)
        ids = np.zeros((n, T_MAX), dtype=np.int32)
        lens = np.zeros(n, dtype=np.int32)
        score = np.zeros(n, dtype=np.float32)
        nsp = np.zeros(n, dtype=np.float32)
        step = np.zeros(n, dtype=np.int32)
        final = np.zeros(n, dtype=np.int32)
        eng = self.engine
        with eng._lock:
            rc = eng.lib.wl_session_peek(eng.ctx, n, _lib.ptr(idx, C.c_int32), _lib.ptr(ids, C.c_int32), _lib.ptr(lens, C.c_int32),
                                         _lib.ptr(score, C.c_float), _lib.ptr(nsp, C.c_float), _lib.ptr(step, C.c_int32),
                                         _lib.ptr(final, C.c_int32))
            _lib.check(eng.lib, eng.ctx, rc, "wl_session_peek")
        return [(ids[i, :max(0, int(lens[i]))].tolist(), float(score[i]), float(nsp[i]), int(step[i]), bool(final[i]))
                for i in range(n)]

    def cancel(self, indices: Sequence[int]) -> None:
        """Take running or finished-but-uncollected streams out of the session; their indices are free at once."""
        idx = np.asarray(list(indices), dtype=np.int32)
        if len(idx) == 0:
            return
        eng = self.engine
        with eng._lock:
            rc = eng.lib.wl_session_cancel(eng.ctx, len(idx), _lib.ptr(idx, C.c_int32))
            _lib.check(eng.lib, eng.ctx, rc, "wl_session_cancel")
        for i in idx.tolist():
            self._held.pop(i, None)
            self._nh.pop(i, None)
        self._finished = [i for i in self._finished if i not in set(idx.tolist())]

    def close(self) -> None:
        if self.closed:
            return
        self.closed = True
        eng = self.engine
        with eng._lock:
            rc = eng.lib.wl_session_close(eng.ctx)
            _lib.check(eng.lib, eng.ctx, rc, "wl_session_close")
        self._held.clear()
