"""Multi-GPU placement of streams (SURVEY.md §8e): the batch dimension is sharded, nothing else.

Streams are independent units (one WebSocket client each, whisper_live/server.py:344); every tensor op of
the hot path fits one H100, so there is no tensor/pipeline parallelism and NO data-path collective:
weights are replicated, a stream's encoder K/V and self-attention cache live on the GPU that owns it
(sticky placement ``stream i -> device i mod G``), and the only exchange is one all-gather of the
emitted token ids (+ segment times) per batch so that every rank -- and the scheduler on rank 0 --
holds the whole batch's result.  The reference has no counterpart (it never passes ``device_index``,
backend/faster_whisper_backend.py:173-178; CT2 would replicate per device, transcriber_faster_whisper.py:598-601).

Two front ends over the same per-device ``B200WhisperModel``:

* ``MultiDeviceWhisperModel``  -- ONE process, G devices: one engine context per GPU, a batch is fanned
  out to all contexts concurrently from worker threads (ctypes releases the GIL inside libwlb200).
  This is what ``ServeClientB200`` builds when several devices are configured.
* ``DistributedTranscriber``   -- one process per GPU under ``torch.distributed`` (what
  ``bench.py --gpus N`` runs under torchrun): every rank calls ``transcribe_batch`` with the whole
  batch, transcribes the streams it owns and all-gathers the results (NCCL on GPUs, gloo in the CPU tests).

Why the north star's *per-step* all-gather is not here: the per-token EOT bookkeeping it would feed
(which streams are done, what to admit next) runs on the device of the owning rank
(csrc/search.cu, the conditional-WHILE decode loop); no other rank consumes a token before the
chunk is finished, so a per-step collective would only add a cross-GPU rendezvous (and couple the
ranks' loop counts) to a latency-bound loop.  One collective per batch carries the same information.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np


def owner_of(stream_index: int, world: int) -> int:
    """Sticky placement: a stream stays on one GPU for the life of its connection."""
    return stream_index % world


# ------------------------------------------------------------------------------------------ one process, G devices
class MultiDeviceWhisperModel:
    """``B200WhisperModel`` surface over several GPUs of one process (weights replicated per device)."""

    def __init__(self, model_size_or_path: str = "small.en", device_index: Sequence[int] = (0,), models=None, **kw):
        if models is None:
            from .transcriber import B200WhisperModel
            models = [B200WhisperModel(model_size_or_path, device_index=int(d), **kw) for d in device_index]
        self.models = list(models)
        if not self.models:
            raise ValueError("MultiDeviceWhisperModel needs at least one device")
        self.device_index = list(device_index)[:len(self.models)] or list(range(len(self.models)))
        self._pool = cf.ThreadPoolExecutor(max_workers=len(self.models), thread_name_prefix="wlb200-dev")
        self._next = 0
        m0 = self.models[0]
        for attr in ("hf_tokenizer", "feature_extractor", "max_length", "frames_per_second", "tokens_per_second",
                     "time_precision", "input_stride", "num_samples_per_token", "supported_languages"):
            if hasattr(m0, attr):
                setattr(self, attr, getattr(m0, attr))
        self.model = m0.model   # engine of device 0: is_multilingual / n_mels for callers that only inspect it

    def transcribe_batch(self, audios: Sequence[np.ndarray], per_stream_kwargs: Optional[Sequence[dict]] = None,
                         placement: Optional[Sequence[int]] = None):
        """``placement[i]`` pins stream i to a device (the scheduler passes the connection's sticky choice);
        default ``i mod G``."""
        n, G = len(audios), len(self.models)
        kws = list(per_stream_kwargs) if per_stream_kwargs is not None else [{} for _ in range(n)]
        place = [int(p) % G for p in placement] if placement is not None else [owner_of(i, G) for i in range(n)]
        shards = [[i for i in range(n) if place[i] == g] for g in range(G)]
        futs = {g: self._pool.submit(self.models[g].transcribe_batch, [audios[i] for i in idx], [kws[i] for i in idx])
                for g, idx in enumerate(shards) if idx}
        out: List[Any] = [None] * n
        for g, f in futs.items():
            for i, r in zip(shards[g], f.result()):
                out[i] = r
        return out

    def transcribe(self, audio: np.ndarray, **kw):
        g = self._next
        self._next = (self._next + 1) % len(self.models)
        return self.models[g].transcribe(audio, **kw)

    def speaker_embeddings(self, audios: Sequence[np.ndarray]) -> np.ndarray:
        """Speaker embeddings on the first device's context (``B200WhisperModel.speaker_embeddings``): the segments of
        a round are few and short next to its decode work, so they stay in one call on one GPU."""
        return self.models[0].speaker_embeddings(audios)

    def open_session(self) -> "MultiDeviceSession":
        """What ``RoundScheduler`` drives: one ``TranscribeSession`` per GPU advanced concurrently, so the step-level
        admission (streams join the running decode loop of THEIR device) works across all of them."""
        return MultiDeviceSession(self)

    def close(self):
        self._pool.shutdown(wait=True)

    @property
    def device_bytes(self) -> Dict[int, int]:
        """Device memory the engine contexts hold right now, summed per CUDA ordinal."""
        out: Dict[int, int] = {}
        for d, m in zip(self.device_index, self.models):
            out[int(d)] = out.get(int(d), 0) + int(m.device_bytes)
        return out

    def destroy(self) -> None:
        """Stop the worker threads and free every device's engine context now."""
        self.close()
        for m in self.models:
            m.destroy()


class _PlacedEntry:
    """A finished stream of one device's session under its scheduler-wide handle."""

    __slots__ = ("handle", "device", "inner")

    def __init__(self, handle, device, inner):
        self.handle, self.device, self.inner = handle, device, inner


class MultiDeviceSession:
    """``TranscribeSession`` surface (add_streams / round / step_round / pending / pop_finished / result_of) over the
    per-device sessions of a ``MultiDeviceWhisperModel``.  A new stream goes to the device with the fewest streams in
    flight (ties: lowest index) and stays there -- its encoder K/V and self-attention cache never move; the rounds of
    all devices that have work run concurrently on the model's worker threads."""

    def __init__(self, md: MultiDeviceWhisperModel):
        self.md = md
        self.sessions = [m.open_session() for m in md.models]
        self._handles = [dict() for _ in self.sessions]     # per device: local handle -> global handle
        self._next_handle = 0
        self.placed: List[int] = []                         # device of every admitted stream, in admission order

    def add_streams(self, audios: Sequence[np.ndarray], per_stream_kwargs: Optional[Sequence[dict]] = None) -> List[int]:
        n, G = len(audios), len(self.sessions)
        kws = list(per_stream_kwargs) if per_stream_kwargs is not None else [{} for _ in range(n)]
        load = [s.pending() for s in self.sessions]
        place = []
        for _ in range(n):
            g = min(range(G), key=lambda k: (load[k], k))
            load[g] += 1
            place.append(g)
        shards = [[i for i in range(n) if place[i] == g] for g in range(G)]
        futs = {g: self.md._pool.submit(self.sessions[g].add_streams, [audios[i] for i in idx], [kws[i] for i in idx])
                for g, idx in enumerate(shards) if idx}
        out = [-1] * n
        for g, f in futs.items():
            for i, local in zip(shards[g], f.result()):
                h = self._next_handle
                self._next_handle += 1
                self._handles[g][local] = h
                out[i] = h
        self.placed += place
        return out

    def _each(self, call) -> None:
        busy = [s for s in self.sessions if s.pending()]
        futs = [self.md._pool.submit(call, s) for s in busy]
        errs = [f.exception() for f in futs]
        for e in errs:
            if e is not None:
                raise e

    def round(self) -> None:
        self._each(lambda s: s.round())

    def step_round(self, max_steps: int = 16) -> None:
        self._each(lambda s: s.step_round(max_steps) if hasattr(s, "step_round") else s.round())

    def pending(self) -> int:
        return sum(s.pending() for s in self.sessions)

    def pop_finished(self) -> List[_PlacedEntry]:
        out = []
        for g, s in enumerate(self.sessions):
            for e in s.pop_finished():
                out.append(_PlacedEntry(self._handles[g].pop(e.handle), g, e))
        return out

    def result_of(self, entry: _PlacedEntry):
        return self.sessions[entry.device].result_of(entry.inner)

    def _locate(self, handles: Sequence[int]) -> List[dict]:
        """per device: local handle -> global handle of those of ``handles`` it holds"""
        want = set(handles)
        return [{lo: h for lo, h in hs.items() if h in want} for hs in self._handles]

    def partials(self, handles: Sequence[int]) -> dict:
        """``TranscribeSession.partials`` on the device that owns each handle (one peek per device)."""
        out = {}
        for g, loc in enumerate(self._locate(handles)):
            if loc:
                for lo, segs in self.sessions[g].partials(list(loc)).items():
                    out[loc[lo]] = segs
        return out

    def settled(self, cursors: dict) -> dict:
        """``TranscribeSession.settled`` on the device that owns each handle."""
        out = {}
        for g, loc in enumerate(self._locate(list(cursors))):
            if loc:
                for lo, segs in self.sessions[g].settled({lo: cursors[h] for lo, h in loc.items()}).items():
                    out[loc[lo]] = segs
        return out

    def info(self, handle: int):
        g, lo = next((g, lo) for g, loc in enumerate(self._locate([handle])) for lo in loc)
        return self.sessions[g].info(lo)

    def cancel(self, handle: int) -> None:
        for g, loc in enumerate(self._locate([handle])):
            for lo in loc:
                self.sessions[g].cancel(lo)
                del self._handles[g][lo]

    def close(self) -> None:
        for s in self.sessions:
            if hasattr(s, "close"):
                s.close()


# ------------------------------------------------------------------------------------------ one process per GPU
class GatheredSegment:
    """A segment transcribed on another rank: what crossed the all-gather (ids and times), text decoded locally."""

    __slots__ = ("id", "start", "end", "tokens", "text", "no_speech_prob", "words", "rank")

    def __init__(self, sid, start, end, tokens, text, rank):
        self.id, self.start, self.end, self.tokens, self.text, self.rank = sid, start, end, tokens, text, rank
        self.no_speech_prob, self.words = 0.0, None


class DistributedTranscriber:
    def __init__(self, model, rank: Optional[int] = None, world_size: Optional[int] = None, group=None, tokenizer_decode=None):
        import torch.distributed as dist
        self.model = model
        self.dist = dist
        self.group = group
        self.distributed = dist.is_available() and dist.is_initialized()
        self.rank = rank if rank is not None else (dist.get_rank(group) if self.distributed else 0)
        self.world = world_size if world_size is not None else (dist.get_world_size(group) if self.distributed else 1)
        self._decode = tokenizer_decode
        self.last_gather_bytes = 0

    def owned(self, n_streams: int) -> List[int]:
        return [i for i in range(n_streams) if owner_of(i, self.world) == self.rank]

    # payload per rank (int32): [n_streams, then per stream: index, n_segments, then per segment: start_ms, end_ms, n_tok, tok...]
    @staticmethod
    def _pack(indices, results) -> np.ndarray:
        buf: List[int] = [len(indices)]
        for i, (segs, _info) in zip(indices, results):
            segs = segs or []
            buf += [i, len(segs)]
            for s in segs:
                buf += [int(round(s.start * 1000)), int(round(s.end * 1000)), len(s.tokens)] + [int(t) for t in s.tokens]
        return np.asarray(buf, dtype=np.int32)

    def _unpack(self, arr: np.ndarray, rank: int, out: List[Any]) -> None:
        p = 1
        for _ in range(int(arr[0])):
            idx, nseg = int(arr[p]), int(arr[p + 1])
            p += 2
            segs = []
            for k in range(nseg):
                st, en, nt = int(arr[p]), int(arr[p + 1]), int(arr[p + 2])
                toks = arr[p + 3:p + 3 + nt].tolist()
                p += 3 + nt
                text = self._decode(toks) if self._decode is not None else ""
                segs.append(GatheredSegment(k + 1, st / 1000.0, en / 1000.0, toks, text, rank))
            out[idx] = (segs, None)

    def transcribe_batch(self, audios: Sequence[np.ndarray], per_stream_kwargs: Optional[Sequence[dict]] = None):
        """Every rank passes the WHOLE batch; returns the whole batch's results on every rank: full
        ``(segments, info)`` for the streams this rank owns, gathered ids/times for the others."""
        import torch
        n = len(audios)
        kws = list(per_stream_kwargs) if per_stream_kwargs is not None else [{} for _ in range(n)]
        mine = self.owned(n)
        local = self.model.transcribe_batch([audios[i] for i in mine], [kws[i] for i in mine]) if mine else []
        out: List[Any] = [None] * n
        for i, r in zip(mine, local):
            out[i] = r
        if not self.distributed or self.world == 1:
            return out
        dist = self.dist
        payload = self._pack(mine, local)
        backend = dist.get_backend(self.group)
        dev = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")
        size = torch.tensor([payload.size], dtype=torch.int64, device=dev)
        dist.all_reduce(size, op=dist.ReduceOp.MAX, group=self.group)
        cap = int(size.item())
        mine_t = torch.zeros(cap + 1, dtype=torch.int32, device=dev)
        mine_t[0] = payload.size
        mine_t[1:1 + payload.size] = torch.from_numpy(payload).to(dev)
        gathered = [torch.empty_like(mine_t) for _ in range(self.world)]
        dist.all_gather(gathered, mine_t, group=self.group)      # the one collective of the path: ids + times per batch
        self.last_gather_bytes = int(mine_t.numel() * 4 * self.world)
        for r, t in enumerate(gathered):
            if r == self.rank:
                continue
            a = t.cpu().numpy()
            self._unpack(a[1:1 + int(a[0])], r, out)
        return out


def devices_from_env() -> List[int]:
    """``WLB200_DEVICES=0,1,2,3`` -> [0, 1, 2, 3]; unset -> [0]."""
    v = os.environ.get("WLB200_DEVICES", "").strip()
    return [int(x) for x in v.split(",") if x.strip() != ""] or [0]
