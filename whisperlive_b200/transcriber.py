"""B200WhisperModel: the transcriber the WhisperLive backend drives (Boundary B, SURVEY.md §8b).

Drop-in for ``whisper_live.transcriber.transcriber_faster_whisper.WhisperModel``
(reference file, class at :574): same ``transcribe`` keyword surface (:692-736), same
result records (``Word`` :33, ``Segment`` :49, ``TranscriptionOptions`` :72,
``TranscriptionInfo`` :102), same attributes ``BatchInferenceWorker`` reads
(``feature_extractor``, ``encode``, ``model``, ``hf_tokenizer``, ``get_prompt``,
``max_length``, ``frames_per_second``, ``_split_segments_by_timestamps``;
whisper_live/batch_inference.py:257-402).

GPU-first differences in *structure* (results are the reference's):
  * the unit of work is a batch of streams: ``transcribe_batch`` advances every
    stream's 30 s-window state machine in lockstep so mel, encoder and the decode loop
    run once per step for all live streams (the reference loops streams serially, or
    batches only the first window: batch_inference.py:259);
  * temperature fallback re-decodes only the failed streams against the SAME
    encoder output handle (reference re-encodes: batch_inference.py:334-339);
  * mel runs on the GPU (K1) -- ``self.feature_extractor`` is the CUDA one.
There is no CPU fallback: without the CUDA engine construction fails.
"""
from __future__ import annotations

import itertools
import json
import threading
import time
import logging
import os
import zlib
from math import ceil
from dataclasses import asdict, dataclass, field, replace
from typing import Any, Dict, Iterable, List, Optional, Sequence, Tuple, Union

import numpy as np

from .engine import STREAM_RULE_KEYS as _RULE_KEYS   # the keywords a stream may bring to a decode session of its own
from .tokenizer import LANGUAGE_CODES, Tokenizer

logger = logging.getLogger("whisperlive_b200")

PUNCT_PREPEND = "\"'“¿([{-"
PUNCT_APPEND = "\"'.。,，!！?？:：”)]}、"
DEFAULT_TEMPERATURES = (0.0, 0.2, 0.4, 0.6, 0.8, 1.0)


# --------------------------------------------------------------------------- records (T1)
@dataclass
class Word:
    start: float
    end: float
    word: str
    probability: float


@dataclass
class Segment:
    id: int
    seek: int
    start: float
    end: float
    text: str
    tokens: List[int]
    avg_logprob: float
    compression_ratio: float
    no_speech_prob: float
    words: Optional[List[Word]]
    temperature: Optional[float]


@dataclass
class TranscriptionOptions:
    beam_size: int
    best_of: int
    patience: float
    length_penalty: float
    repetition_penalty: float
    no_repeat_ngram_size: int
    log_prob_threshold: Optional[float]
    no_speech_threshold: Optional[float]
    compression_ratio_threshold: Optional[float]
    condition_on_previous_text: bool
    prompt_reset_on_temperature: float
    temperatures: List[float]
    initial_prompt: Optional[Union[str, Iterable[int]]]
    prefix: Optional[str]
    suppress_blank: bool
    suppress_tokens: Optional[List[int]]
    without_timestamps: bool
    max_initial_timestamp: float
    word_timestamps: bool
    prepend_punctuations: str
    append_punctuations: str
    multilingual: bool
    max_new_tokens: Optional[int]
    clip_timestamps: Union[str, List[float]]
    hallucination_silence_threshold: Optional[float]
    hotwords: Optional[str]


@dataclass
class TranscriptionInfo:
    language: str
    language_probability: float
    duration: float
    duration_after_vad: float
    all_language_probs: Optional[List[Tuple[str, float]]]
    transcription_options: Optional[TranscriptionOptions]
    vad_options: Any


# --------------------------------------------------------------------------- small host helpers
def get_compression_ratio(text: str) -> float:
    """zlib ratio used as the repetition detector (reference :1826-1828)."""
    raw = text.encode("utf-8")
    return len(raw) / len(zlib.compress(raw))


def get_suppressed_tokens(tokenizer: Tokenizer, suppress_tokens) -> Optional[Tuple[int, ...]]:
    """Reference :1831-1853: -1 expands to the non-speech set; task/sot tokens always added."""
    if suppress_tokens is None:
        ids: List[int] = []
    elif -1 in suppress_tokens:
        ids = [t for t in suppress_tokens if t >= 0] + list(tokenizer.non_speech_tokens)
    else:
        ids = list(suppress_tokens)
    ids += [tokenizer.transcribe, tokenizer.translate, tokenizer.sot, tokenizer.sot_prev, tokenizer.sot_lm]
    return tuple(sorted(set(ids)))


def get_end(segments: List[dict]) -> Optional[float]:
    """End time of the last word, else of the last segment (faster_whisper.utils.get_end)."""
    for seg in reversed(segments):
        for w in reversed(seg.get("words") or []):
            return w["end"]
    return segments[-1]["end"] if segments else None


def merge_punctuations(alignment: List[dict], prepended: str, appended: str) -> None:
    """Glue leading/trailing punctuation onto the neighbouring word (reference :1856-1887)."""
    # right-to-left: prefixes move onto the following word
    nxt = len(alignment) - 1
    for cur in range(len(alignment) - 2, -1, -1):
        a, b = alignment[cur], alignment[nxt]
        if a["word"].startswith(" ") and a["word"].strip() in prepended:
            b["word"] = a["word"] + b["word"]
            b["tokens"] = a["tokens"] + b["tokens"]
            a["word"], a["tokens"] = "", []
        else:
            nxt = cur
    # left-to-right: suffixes move onto the preceding word
    prev = 0
    for cur in range(1, len(alignment)):
        a, b = alignment[prev], alignment[cur]
        if not a["word"].endswith(" ") and b["word"] in appended:
            a["word"] = a["word"] + b["word"]
            a["tokens"] = a["tokens"] + b["tokens"]
            b["word"], b["tokens"] = "", []
        else:
            prev = cur


def _load_vad():
    """VAD gating is unchanged from the reference (CPU Silero via faster_whisper.vad,
    reference :830-838); it is an optional dependency here."""
    try:
        from faster_whisper import vad  # type: ignore
        return vad
    except Exception as e:  # pragma: no cover - absent in the build container
        raise RuntimeError("vad_filter=True needs faster_whisper.vad (Silero VAD, onnxruntime); "
                           "pass use_vad=False or install it") from e


def restore_speech_timestamps(segments: List[Segment], speech_chunks: List[dict], sampling_rate: int, vad=None):
    """Map times on the VAD-concatenated axis back to the original audio (reference :1792-1817)."""
    ts_map = (vad or _load_vad()).SpeechTimestampsMap(speech_chunks, sampling_rate)
    for seg in segments:
        if seg.words:
            for w in seg.words:
                ci = ts_map.get_chunk_index((w.start + w.end) / 2)
                w.start = ts_map.get_original_time(w.start, ci)
                w.end = ts_map.get_original_time(w.end, ci)
            seg.start, seg.end = seg.words[0].start, seg.words[-1].end
        else:
            seg.start = ts_map.get_original_time(seg.start)
            seg.end = ts_map.get_original_time(seg.end)
    return segments


def pad_or_trim(features: np.ndarray, length: int = 3000) -> np.ndarray:
    if hasattr(features, "window"):          # resident features: trimmed here, zero-padded on the device by the encoder's gather
        return features[..., :length]
    n = features.shape[-1]
    if n >= length:
        return features[..., :length]
    pad = [(0, 0)] * (features.ndim - 1) + [(0, length - n)]
    return np.pad(features, pad)


# --------------------------------------------------------------------------- per-stream window state
@dataclass
class _Decoded:
    result: Any
    avg_logprob: float
    temperature: float
    compression_ratio: float


class _StreamJob:
    """Window-by-window state of one stream (the body of the reference's
    ``generate_segments`` loop, :1049-1337, turned inside out so a scheduler can batch
    the device work of many streams per step)."""

    def __init__(self, model: "B200WhisperModel", features: np.ndarray, tokenizer: Tokenizer,
                 options: TranscriptionOptions):
        self.m = model
        self.features = features
        self.tok = tokenizer
        self.opt = options
        fe = model.feature_extractor
        self.content_frames = features.shape[-1] - 1
        self.content_duration = float(self.content_frames * fe.time_per_frame)
        clips = options.clip_timestamps
        if isinstance(clips, str):
            clips = [float(x) for x in clips.split(",")] if clips else []
            options.clip_timestamps = clips
        pts = [round(t * model.frames_per_second) for t in clips] or [0]
        if len(pts) % 2:
            pts.append(self.content_frames)
        self.clips = list(zip(pts[::2], pts[1::2]))
        self.clip_idx = 0
        self.seek = self.clips[0][0]
        self.all_tokens: List[int] = []
        self.prompt_reset_since = 0
        if options.initial_prompt is not None:
            if isinstance(options.initial_prompt, str):
                self.all_tokens.extend(tokenizer.encode(" " + options.initial_prompt.strip()))
            else:
                self.all_tokens.extend(options.initial_prompt)
        self.single_window = False
        self.last_speech_timestamp = 0.0
        self.segments: List[Segment] = []
        self.n_emitted = 0
        # current window
        self.time_offset = 0.0
        self.window_end_time = 0.0
        self.segment_size = 0
        self.segment_duration = 0.0
        self.prompt: List[int] = []
        self.enc = None
        # fallback bookkeeping for the current window
        self.temp_idx = 0
        self.tried: List[_Decoded] = []
        self.below_cr: List[_Decoded] = []

    # -- window selection (reference :1104-1127) -------------------------------------------
    def next_window(self) -> Optional[np.ndarray]:
        """Features of the next 30 s window, zero-padded to 3000 frames (reference :1115-1127), or None at the end."""
        view = self.advance_window()
        return None if view is None else pad_or_trim(view, self.m.feature_extractor.nb_max_frames)

    def advance_window(self) -> Optional[np.ndarray]:
        """Move to the next window and return its un-padded feature view [n_mels, <= 3000]."""
        fe = self.m.feature_extractor
        while self.clip_idx < len(self.clips):
            lo, hi = self.clips[self.clip_idx]
            hi = min(hi, self.content_frames)
            self.seek = max(self.seek, lo)
            if self.seek >= hi:
                self.clip_idx += 1
                if self.clip_idx < len(self.clips):
                    self.seek = self.clips[self.clip_idx][0]
                continue
            self.time_offset = self.seek * fe.time_per_frame
            self.window_end_time = float((self.seek + fe.nb_max_frames) * fe.time_per_frame)
            self.segment_size = min(fe.nb_max_frames, self.content_frames - self.seek, hi - self.seek)
            self.segment_duration = self.segment_size * fe.time_per_frame
            self.temp_idx, self.tried, self.below_cr = 0, [], []
            return self.features[:, self.seek:self.seek + min(self.segment_size, fe.nb_max_frames)]
        return None

    def prepare_decode(self) -> None:
        """The window is encoded (``self.enc``): language id when ``multilingual``, then the prompt."""
        if self.opt.multilingual:
            tok_s, _p = self.m.model.detect_language(self.enc)[0][0]
            self.tok.language = self.tok.tokenizer.token_to_id(tok_s)
            self.tok.language_code = tok_s[2:-2]
        self.build_prompt()

    def build_prompt(self) -> List[int]:
        self.prompt = self.m.get_prompt(
            self.tok, self.all_tokens[self.prompt_reset_since:], without_timestamps=self.opt.without_timestamps,
            prefix=self.opt.prefix if self.seek == 0 else None, hotwords=self.opt.hotwords)
        return self.prompt

    # -- temperature ladder (reference :1380-1478) ------------------------------------------
    @property
    def temperature(self) -> float:
        return self.opt.temperatures[self.temp_idx]

    def generate_kwargs(self) -> dict:
        o = self.opt
        max_length = self.m.max_length if o.max_new_tokens is None else len(self.prompt) + o.max_new_tokens
        if max_length > self.m.max_length:
            raise ValueError(
                f"The length of the prompt is {len(self.prompt)}, and the `max_new_tokens` "
                f"{max_length - len(self.prompt)}. Thus, the combined length of the prompt and `max_new_tokens` is: "
                f"{max_length}. This exceeds the `max_length` of the Whisper model: {self.m.max_length}.")
        kw = dict(self._shared_kwargs(), max_length=max_length)
        t = self.temperature
        if t > 0:
            kw.update(beam_size=1, num_hypotheses=o.best_of, sampling_topk=0, sampling_temperature=t)
        else:
            kw.update(beam_size=o.beam_size, patience=o.patience)
        return kw

    def _shared_kwargs(self) -> dict:
        """The generate options every rung of the ladder shares."""
        o = self.opt
        return dict(length_penalty=o.length_penalty, repetition_penalty=o.repetition_penalty,
                    no_repeat_ngram_size=o.no_repeat_ngram_size, return_scores=True, return_no_speech_prob=True,
                    suppress_blank=o.suppress_blank, suppress_tokens=o.suppress_tokens,
                    max_initial_timestamp_index=int(round(o.max_initial_timestamp / self.m.time_precision)))

    def session_kwargs(self) -> dict:
        """Options of the decode session this stream's windows decode in, whatever rung they are on: rung 0's beam
        search and the shared options (``max_length`` is given per stream at admission, a sampling rung joins with a
        per-stream sampling spec)."""
        o = self.opt
        return dict(self._shared_kwargs(), beam_size=o.beam_size, patience=o.patience, num_hypotheses=1)

    def stream_rules(self) -> dict:
        """The logits rules this stream decodes under when it joins a decode session opened with other options."""
        skw = self.session_kwargs()
        return {k: skw[k] for k in _RULE_KEYS if k in skw}

    def accept(self, result) -> bool:
        """Record one decode; True when the window is settled (else retry at the next temperature)."""
        o = self.opt
        tokens = result.sequences_ids[0]
        n = len(tokens)
        cum = result.scores[0] * (n ** o.length_penalty)
        avg_logprob = cum / (n + 1)
        cr = get_compression_ratio(self.tok.decode(tokens).strip())
        d = _Decoded(result, avg_logprob, self.temperature, cr)
        self.tried.append(d)
        retry = False
        if o.compression_ratio_threshold is not None:
            if cr > o.compression_ratio_threshold:
                retry = True
            else:
                self.below_cr.append(d)
        if o.log_prob_threshold is not None and avg_logprob < o.log_prob_threshold:
            retry = True
        if (o.no_speech_threshold is not None and result.no_speech_prob > o.no_speech_threshold
                and o.log_prob_threshold is not None and avg_logprob < o.log_prob_threshold):
            retry = False  # silence
        if retry and self.temp_idx + 1 < len(o.temperatures):
            self.temp_idx += 1
            return False
        if retry:  # ladder exhausted: best avg_logprob among the non-repetitive ones
            best = max(self.below_cr or self.tried, key=lambda x: x.avg_logprob)
            d = _Decoded(best.result, best.avg_logprob, self.temperature, best.compression_ratio)
        self.decoded = d
        return True

    # -- window post-processing (reference :1162-1330) ---------------------------------------
    def needs_alignment(self) -> bool:
        return self.opt.word_timestamps and not self._skip_as_silence()

    def _skip_as_silence(self) -> bool:
        o, d = self.opt, self.decoded
        if o.no_speech_threshold is None:
            return False
        skip = d.result.no_speech_prob > o.no_speech_threshold
        if o.log_prob_threshold is not None and d.avg_logprob > o.log_prob_threshold:
            skip = False
        return skip

    def split(self) -> None:
        self.previous_seek = self.seek
        self.current, self.seek, self.single_ts_ending = self.m._split_segments_by_timestamps(
            tokenizer=self.tok, tokens=self.decoded.result.sequences_ids[0], time_offset=self.time_offset,
            segment_size=self.segment_size, segment_duration=self.segment_duration, seek=self.seek)

    def alignment_request(self) -> Optional[List[int]]:
        """Text tokens this window wants aligned (after the timestamp split), or None.  Lets the scheduler run ONE
        batched ``align`` for all streams of a window instead of one teacher-forced pass per stream."""
        if not self.needs_alignment():
            return None
        self.split()
        self._presplit = True
        return [t for sub in self.current for t in sub["tokens"] if t < self.tok.eot]

    def finish_window(self) -> None:
        o, d, m = self.opt, self.decoded, self.m
        if self._skip_as_silence():
            self.seek += self.segment_size
            return
        if not getattr(self, "_presplit", False):
            self.split()
        self._presplit = False
        if o.word_timestamps:
            pre = getattr(self, "_align_result", None)
            self._align_result = None
            m.add_word_timestamps([self.current], self.tok, self.enc, self.segment_size, o.prepend_punctuations,
                                  o.append_punctuations, last_speech_timestamp=self.last_speech_timestamp,
                                  precomputed=None if pre is None else [pre])
            if not self.single_ts_ending:
                last_end = get_end(self.current)
                if last_end is not None and last_end > self.time_offset:
                    self.seek = round(last_end * m.frames_per_second)
            if o.hallucination_silence_threshold is not None and self._skip_hallucinations():
                return
            last_end = get_end(self.current)
            if last_end is not None:
                self.last_speech_timestamp = last_end
        for seg in self.current:
            toks = seg["tokens"]
            text = self.tok.decode(toks)
            if seg["start"] == seg["end"] or not text.strip():
                continue
            self.all_tokens.extend(toks)
            self.n_emitted += 1
            self.segments.append(Segment(
                id=self.n_emitted, seek=self.previous_seek, start=seg["start"], end=seg["end"], text=text, tokens=toks,
                temperature=d.temperature, avg_logprob=d.avg_logprob, compression_ratio=d.compression_ratio,
                no_speech_prob=d.result.no_speech_prob,
                words=[Word(**w) for w in seg["words"]] if o.word_timestamps else None))
        if not o.condition_on_previous_text or d.temperature > o.prompt_reset_on_temperature:
            self.prompt_reset_since = len(self.all_tokens)

    def _skip_hallucinations(self) -> bool:
        """Reference :1241-1286. True -> the window is abandoned (``continue`` upstream)."""
        thr = self.opt.hallucination_silence_threshold
        fps = self.m.frames_per_second
        punct = PUNCT_PREPEND + PUNCT_APPEND

        def anomaly(word: dict) -> float:
            dur = word["end"] - word["start"]
            s = 1.0 if word.get("probability", 0.0) < 0.15 else 0.0
            if dur < 0.133:
                s += (0.133 - dur) * 15
            if dur > 2.0:
                s += dur - 2.0
            return s

        def is_anomaly(seg: Optional[dict]) -> bool:
            if seg is None or not seg["words"]:
                return False
            ws = [w for w in seg["words"] if w["word"] not in punct][:8]
            score = sum(anomaly(w) for w in ws)
            return score >= 3 or score + 0.01 >= len(ws)

        def first_with_words(segs):
            return next((s for s in segs if s["words"]), None)

        first = first_with_words(self.current)
        if first is not None and is_anomaly(first):
            gap = first["start"] - self.time_offset
            if gap > thr:
                self.seek = self.previous_seek + round(gap * fps)
                return True
        hal_last_end = self.last_speech_timestamp
        for si, seg in enumerate(self.current):
            if not seg["words"]:
                continue
            if is_anomaly(seg):
                nxt = first_with_words(self.current[si + 1:])
                nxt_start = nxt["words"][0]["start"] if nxt is not None else self.time_offset + self.segment_duration
                before = (seg["start"] - hal_last_end > thr or seg["start"] < thr
                          or seg["start"] - self.time_offset < 2.0)
                after = (nxt_start - seg["end"] > thr or is_anomaly(nxt) or self.window_end_time - seg["end"] < 2.0)
                if before and after:
                    self.seek = round(max(self.time_offset + 1, seg["start"]) * fps)
                    if self.content_duration - seg["end"] < thr:
                        self.seek = self.content_frames
                    self.current[si:] = []
                    break
            hal_last_end = seg["end"]
        return False


# --------------------------------------------------------------------------- rounds
class _Entry:
    __slots__ = ("job", "window", "state", "parent", "index", "handle", "prepared", "error", "file")

    def __init__(self, job, handle, prepared=None):
        self.job, self.handle, self.prepared = job, handle, prepared
        self.window, self.state, self.parent, self.index, self.error = None, "window", None, -1, None
        self.file: Optional["_FileRun"] = None        # the batched file this chunk belongs to (None: a live stream)


class _EncGroup:
    """One ``encode`` call's output and how many of its streams are still decoding (slots go back when the last one is done)."""

    def __init__(self, enc, n):
        self.enc, self.left = enc, n

    def done_one(self):
        self.left -= 1
        if self.left == 0:
            release = getattr(self.enc, "release", None)
            if release is not None:
                release()             # encoder slots back to the pool NOW (explicit, not refcount-driven)
            self.enc = None


class TranscribeSession:
    """The window / fallback state machines of many streams advanced in ROUNDS.  One round =
      1. encode the next 30 s window of every stream that needs one (groups of at most ``engine.max_streams``, never
         more windows than the encoder slot pool has free),
      2. ONE ``generate`` call per distinct option set over every stream that has a window to decode -- first attempts
         and temperature-fallback retries of different streams share the call when their options agree,
      3. batched word alignment + window post-processing of the streams whose decode settled.
    Streams are independent, so a stream's result does not depend on who shares its rounds; but nobody waits for a
    whole batch: a stream added between two rounds joins the next one, a multi-window stream does not hold the others
    in lock-step, and a finished stream's slots are refilled immediately.  (The reference's batcher assembles a batch,
    runs it to completion -- first window only -- and re-encodes on every fallback rung: batch_inference.py:155-187,
    :259, :334-339.)  ``B200WhisperModel.transcribe_batch`` is this with all streams added up front."""

    def __init__(self, model: "B200WhisperModel"):
        self.m = model
        self.entries: List[_Entry] = []
        self._next_handle = 0
        self.rounds = 0
        # step-level rounds (step_round): the engine's decode session, its option key, index -> entry of the streams in it
        self._dsess = None
        self._dsess_key: Optional[str] = None
        self._running: Dict[int, _Entry] = {}
        self._dsess_files = False            # the open decode session was opened for a batched file's chunks
        self.admitted_steps: List[int] = []   # session step count at each admission (tests: > 0 = joined a running loop)
        # batched files (add_file): their chunks enter as entries, at most max_share of the indices each, never while
        # a live stream waits (live_waiting: set by a scheduler whose inbox holds live requests)
        self.files: Dict[int, "_FileRun"] = {}
        self.live_waiting = False
        self.rule_admissions = 0             # streams that joined the decode session with logits rules of their own

    # -- admission -------------------------------------------------------------------------------
    def add_job(self, job: _StreamJob, prepared: Optional[dict] = None) -> int:
        h = self._next_handle
        self._next_handle += 1
        e = _Entry(job, h, prepared)
        e.window = job.advance_window()
        if e.window is None:
            e.state = "done"
        self.entries.append(e)
        return h

    def add_streams(self, audios: Sequence[np.ndarray], per_stream_kwargs: Optional[Sequence[dict]] = None,
                    resident_ok: bool = False) -> List[int]:
        """Admit streams (reference ``WhisperModel.transcribe`` :811-968 up to the window loop, batched): VAD clipping,
        ONE mel call for all of them, language resolution, options.  ``resident_ok``: the features may stay in HBM
        (valid until the next mel call on this engine, i.e. only when nothing else is admitted before these streams
        finish -- ``transcribe_batch``); a scheduler that keeps admitting takes the host-returning extractor."""
        m = self.m
        n = len(audios)
        kws = list(per_stream_kwargs) if per_stream_kwargs is not None else [{} for _ in range(n)]
        tm = getattr(m, "last_timing", None) or {}
        t0 = time.perf_counter()
        def as_pcm(a):    # paths / bytes / file objects go through decode_audio like reference :820-821
            return a if isinstance(a, (str, bytes, bytearray, os.PathLike)) or hasattr(a, "read") else np.asarray(a)
        vad = getattr(m, "_vad", None)
        if hasattr(vad, "speech_timestamps_batch"):
            # every VAD-gated stream of the call through one device VAD call, then the same gating per stream
            inputs = [m._stream_input(as_pcm(a), dict(k)) for a, k in zip(audios, kws)]
            gated = [i for i, (_a, k, _s) in enumerate(inputs) if k["vad_filter"] and k["clip_timestamps"] == "0"]
            found = vad.speech_timestamps_batch([inputs[i][0] for i in gated],
                                                [m._vad_options(vad, inputs[i][1]["vad_parameters"]) for i in gated]
                                                ) if gated else []
            chunks = dict(zip(gated, found))
            prepared = [m._gate_stream(*inp, speech_chunks=chunks.get(i)) for i, inp in enumerate(inputs)]
        else:
            prepared = [m._prepare_stream(as_pcm(a), dict(k)) for a, k in zip(audios, kws)]
        tm["prepare"] = tm.get("prepare", 0.0) + time.perf_counter() - t0
        handles: List[int] = []
        live = [i for i, p in enumerate(prepared) if p is not None]
        feats: List[Any] = []
        if live:
            t0 = time.perf_counter()
            fe = m.feature_extractor
            cap = int(getattr(m.model, "max_streams", 0) or 0)
            chunk_length = prepared[live[0]]["kw"].get("chunk_length")
            if resident_ok and hasattr(fe, "batch_resident") and 0 < len(live) <= cap and not self.entries:
                # mel -> encoder without leaving HBM (the reference's two host-side calls, :862 and :1348, fused on the device)
                feats = fe.batch_resident([prepared[i]["audio"] for i in live], chunk_length=chunk_length)
            else:
                feats = fe.batch([prepared[i]["audio"] for i in live], chunk_length=chunk_length)
            tm["mel"] = tm.get("mel", 0.0) + time.perf_counter() - t0
            for i, f in zip(live, feats):
                prepared[i]["features"] = f
            m._resolve_languages([prepared[i] for i in live])
        for i in range(n):
            p = prepared[i]
            if p is None:      # nothing left after VAD: (None, None) like reference :860-861
                h = self._next_handle
                self._next_handle += 1
                e = _Entry(None, h, None)
                e.state = "done"
                self.entries.append(e)
                handles.append(h)
                continue
            tok = Tokenizer(m.hf_tokenizer, m.model.is_multilingual, task=p["kw"]["task"], language=p["language"])
            p["options"] = m._make_options(tok, p["kw"])
            job = _StreamJob(m, p["features"], tok, p["options"])
            job.single_window = p["single_window"]
            handles.append(self.add_job(job, p))
        return handles

    def result(self, handle: int):
        """``(segments, info)`` of a finished stream (raises what the stream raised)."""
        return self.result_of(next(e for e in self.entries if e.handle == handle))

    def result_of(self, e: "_Entry"):
        if e.state != "done":
            raise RuntimeError("stream is still in flight")
        if e.error is not None:
            raise e.error
        if e.job is None:
            return (None, None)
        m, p, segs = self.m, e.prepared, e.job.segments
        if p is None:
            return (segs, None)
        if p["speech_chunks"]:
            segs = restore_speech_timestamps(segs, p["speech_chunks"], m.feature_extractor.sampling_rate, m._vad)
        return (segs, self._info(p))

    @staticmethod
    def _info(p: dict) -> TranscriptionInfo:
        return TranscriptionInfo(language=p["language"], language_probability=p["language_probability"], duration=p["duration"],
                                 duration_after_vad=p["duration_after_vad"], transcription_options=p["options"],
                                 vad_options=p["vad_parameters"], all_language_probs=p["all_language_probs"])

    def info(self, handle: int) -> Optional[TranscriptionInfo]:
        """The ``TranscriptionInfo`` of an admitted stream (its language is resolved at admission); None for a stream
        that VAD left empty."""
        e = next(x for x in self.entries if x.handle == handle)
        return None if e.job is None or e.prepared is None else self._info(e.prepared)

    def settled(self, cursors: Dict[int, int]) -> Dict[int, List[Segment]]:
        """``handle -> cursor``: the segments each live stream settled past its cursor (streams with none are left
        out).  Copies, with the timestamps of the final result; host state only, no device call.  A settled segment
        does not change afterwards, so a caller that advances its cursor reads each one once."""
        out = {}
        for e in self.entries:
            n = cursors.get(e.handle)
            if n is not None and e.job is not None and len(e.job.segments) > n:
                out[e.handle] = self._settled_copy(e, e.job.segments[n:])
        return out

    def _settled_copy(self, e: _Entry, segments: List[Segment]) -> List[Segment]:
        # copies down to the words: restore_speech_timestamps maps them in place, and result_of maps the stream's own
        # segments and words once, when it finishes
        segs = [replace(s, words=None if s.words is None else [replace(w) for w in s.words]) for s in segments]
        p = e.prepared
        if p is not None and p.get("speech_chunks"):
            segs = restore_speech_timestamps(segs, p["speech_chunks"], self.m.feature_extractor.sampling_rate, self.m._vad)
        return segs

    def pending(self) -> int:
        return sum(1 for e in self.entries if e.state != "done")

    def pop_finished(self) -> List[_Entry]:
        done = [e for e in self.entries if e.state == "done"]
        self.entries = [e for e in self.entries if e.state != "done"]
        return done

    # -- one round ---------------------------------------------------------------------------------
    def round(self) -> None:
        """Window-level round: encode, ONE generate call per option set run to completion, settle."""
        self.rounds += 1
        self._feed_files()
        self._encode_pending()
        settled = self._generate_groups([e for e in self.entries if e.state == "decode"])
        self._settle(settled)
        self._finalise_files()

    def step_round(self, max_steps: int = 16) -> None:
        """Token-step-level round (N2): the streams whose windows are ready JOIN the decode loop that is already running
        (``engine.open_decode_session``), the loop advances by at most ``max_steps`` token steps -- or until some stream
        finishes -- and whatever finished is settled while the others stay in the loop.  A stream that arrives while 31
        others are in the middle of a 100-token decode starts decoding a few token steps later, and is answered when ITS
        last window settles.  Falls back to ``round()`` on engines without decode sessions.

        A session is keyed by its streams' rung-0 options (``_StreamJob.session_kwargs``), so every rung of a stream
        decodes in it: a sampling rung of the temperature ladder joins the running loop with a per-stream sampling spec
        when ``best_of`` fits the session's rows per stream, its noise seeded by ``session_noise_seed`` (noise key 0).
        What stays on the one-shot path: sampling rungs whose ``best_of`` does not fit, or whose rung-0 options differ
        from the open session's while it is busy (beam rungs in that case wait for the session to drain)."""
        m = self.m
        if not hasattr(m.model, "open_decode_session"):
            return self.round()
        tm = getattr(m, "last_timing", None) or {}
        self.rounds += 1
        self._feed_files()
        self._encode_pending()
        one_shot: List[_Entry] = []
        joining: List[Tuple[_Entry, int, Optional[tuple], Optional[dict]]] = []
        waiting = [e for e in self.entries if e.state == "decode"]
        for e in waiting:
            try:
                kw = e.job.generate_kwargs()
                skw = e.job.session_kwargs()
            except Exception as ex:
                self._fail(e, ex)
                continue
            key = json.dumps(skw, sort_keys=True, default=list)
            ds = self._dsess
            if ds is None or (key != self._dsess_key and ds.live == 0 and not joining):
                if ds is not None:
                    ds.close()
                ds = self._dsess = m.model.open_decode_session(**skw)
                self._dsess_key = key
                self._dsess_files = e.file is not None
            rules = None
            if key != self._dsess_key and (e.file is not None or self._dsess_files) and _rules_fit(ds, skw):
                # a file's chunk in a live session, or a live stream in a session a file opened: the stream joins the
                # running loop with its own logits rules (DecodeSession.admit(rules=...)) instead of waiting for it to drain
                rules = e.job.stream_rules()
            spec = None
            if kw.get("beam_size", 1) == 1 and kw.get("sampling_topk", 1) != 1 and kw.get("sampling_temperature", 0) > 0:
                # a session model without per-stream sampling has no rows_per_stream: its rungs stay one-shot
                if (key != self._dsess_key and rules is None) or kw["num_hypotheses"] > getattr(ds, "rows_per_stream", 0):
                    one_shot.append(e)
                    continue
                spec = (kw["sampling_temperature"], kw["num_hypotheses"],
                        session_noise_seed(e.handle, e.job.seek, e.job.temp_idx), 0)
            if (key != self._dsess_key and rules is None) or len(joining) >= len(ds.free_indices()):
                continue                                   # next step_round: the loop has to drain / free an index first
            joining.append((e, kw["max_length"], spec, rules))
        if joining:                                        # ONE admission = one batched prefill pass for all of them
            ds = self._dsess
            specs = [sp for _, _, sp, _ in joining]
            rls = [r for _, _, _, r in joining]
            extra = {}
            if any(sp is not None for sp in specs):
                extra["sampling"] = specs
            if any(r is not None for r in rls):
                extra["rules"] = rls
            try:
                idxs = ds.admit([e.job.enc for e, _, _, _ in joining], [e.job.prompt for e, _, _, _ in joining],
                                [ml for _, ml, _, _ in joining], **extra)
            except Exception as ex:
                for e, _, _, _ in joining:
                    self._fail(e, ex)
                idxs = []
            for idx, (e, _, _, r) in zip(idxs, joining):
                e.state = "running"
                self._running[idx] = e
                self.admitted_steps.append(getattr(ds, "steps", 0))
                self.rule_admissions += r is not None
        settled = self._generate_groups(one_shot)
        ds = self._dsess
        if ds is not None and ds.live:
            t0 = time.perf_counter()
            try:
                finished = ds.run(max_steps=max_steps, break_on_finish=True)
            except Exception as ex:
                for e in list(self._running.values()):
                    self._fail(e, ex)
                self._running.clear()
                try:
                    ds.close()                             # the engine-side session must not keep their indices
                except Exception:
                    pass
                self._dsess = None
                finished = []
            tm["generate"] = tm.get("generate", 0.0) + time.perf_counter() - t0
            for idx in finished:
                e = self._running.pop(idx)
                try:
                    r = ds.collect(idx)
                    if e.job.accept(r):
                        settled.append(e)
                    else:
                        e.state = "decode"                 # next rung of the temperature ladder
                except Exception as ex:
                    self._fail(e, ex)
        self._settle(settled)
        self._finalise_files()

    def close(self) -> None:
        if self._dsess is not None:
            self._dsess.close()
            self._dsess = None

    # -- between two rounds: interim text, cancellation --------------------------------------------
    def partials(self, handles: Sequence[int]) -> Dict[int, List[Segment]]:
        """Interim segments of the streams ``handles`` (live entries only): the segments of the windows that already
        settled, then the running window's tokens so far cut by ``_split_segments_by_timestamps`` -- ONE ``peek`` of the
        decode session for all of them.  Only a rung-0 decode gives interim text: a window on a fallback rung shows
        nothing more until it settles.  Interim segments carry no words (alignment runs once, at settle); VAD-clipped
        streams get the mapping of their final result."""
        m = self.m
        want = set(handles)
        live = [e for e in self.entries if e.handle in want and e.job is not None]
        running = {id(e): idx for idx, e in self._running.items()}
        ds = self._dsess
        peek_on = [e for e in live if id(e) in running and e.job.temp_idx == 0] if ds is not None and hasattr(ds, "peek") else []
        peeked = dict(zip((id(e) for e in peek_on), ds.peek([running[id(e)] for e in peek_on]))) if peek_on else {}
        out: Dict[int, List[Segment]] = {}
        for e in live:
            j = e.job
            # copies down to the words: restore_speech_timestamps below maps them in place, and result_of maps the
            # stream's own segments and words once, when it finishes
            segs = [replace(s, words=None if s.words is None else [replace(w) for w in s.words]) for s in j.segments]
            if id(e) in peeked:
                tokens, score, no_speech, _step, _final = peeked[id(e)]
                n = len(tokens)
                avg_logprob = score * (n ** j.opt.length_penalty) / (n + 1)
                pieces, _seek, _single = m._split_segments_by_timestamps(
                    tokenizer=j.tok, tokens=tokens, time_offset=j.time_offset, segment_size=j.segment_size,
                    segment_duration=j.segment_duration, seek=j.seek)
                cr = get_compression_ratio(j.tok.decode(tokens).strip()) if n else 0.0
                for piece in pieces:
                    text = j.tok.decode(piece["tokens"])
                    if piece["start"] == piece["end"] or not text.strip():
                        continue
                    segs.append(Segment(id=len(segs) + 1, seek=j.seek, start=piece["start"], end=piece["end"], text=text,
                                        tokens=piece["tokens"], avg_logprob=avg_logprob, compression_ratio=cr,
                                        no_speech_prob=no_speech, words=None, temperature=j.temperature))
            p = e.prepared
            if p is not None and p.get("speech_chunks"):
                segs = restore_speech_timestamps(segs, p["speech_chunks"], m.feature_extractor.sampling_rate, m._vad)
            out[e.handle] = segs
        return out

    def cancel(self, handle: int) -> None:
        """Drop a stream in any state: its decode-session index (if it is running) and its encoder slots are free when
        this returns, and the session forgets it.  A handle it does not hold is ignored."""
        e = next((x for x in self.entries if x.handle == handle), None)
        if e is None:
            return
        idx = next((i for i, x in self._running.items() if x is e), None)
        if idx is not None:
            self._dsess.cancel([idx])
            del self._running[idx]
        if e.job is not None:
            e.job.enc = None
        if e.parent is not None:
            e.parent.done_one()
            e.parent = None
        self.entries.remove(e)

    # -- batched files: a file's speech chunks as streams of this session ------------------------------------
    def add_file(self, run: "_ChunkRun", max_share: float = 0.5, capacity: Optional[int] = None) -> int:
        """Take the chunks of one ``BatchedInferencePipeline`` file (``run``); they enter as indices free up, at most
        ``max_share`` of ``capacity`` streams at once (a scheduler's capacity; never more than the engine's
        ``max_streams``), and never while a live stream waits.  Returns the file's handle: ``file_segments`` /
        ``file_done`` / ``file_error`` / ``drop_file``."""
        cap = int(getattr(self.m.model, "max_streams", 0) or 0) or 8
        if capacity is not None:
            cap = min(cap, int(capacity))
        h = self._next_handle
        self._next_handle += 1
        self.files[h] = _FileRun(run, h, max(1, int(max_share * cap)))
        return h

    def file_streams(self) -> int:
        """Streams the files' chunks count for: those in the session, and decoded ones that still hold an encoder slot
        (word timestamps on an engine whose outputs cannot be joined keep it until the chunk is finalised)."""
        return sum(f.held() for f in self.files.values())

    def file_segments(self, handle: int, n: int) -> List[Segment]:
        """The file's finalised segments after the first ``n``, in chunk order, ids counted on, original time axis."""
        return self.files[handle].segments[n:]

    def file_done(self, handle: int) -> bool:
        return self.files[handle].done

    def file_error(self, handle: int) -> Optional[Exception]:
        return self.files[handle].error

    def drop_file(self, handle: int) -> None:
        """Forget a finished file, or cancel one in flight: its chunks leave the decode session and their slots go back."""
        f = self.files.pop(handle, None)
        if f is None:
            return
        for e in list(f.active):
            self.cancel(e.handle)
        for e in f.decoded.values():
            if e.parent is not None:
                e.parent.done_one()
                e.parent = None
        f.active, f.decoded = [], {}

    def _feed_files(self) -> None:
        if not self.files:
            return
        if self.live_waiting or any(e.file is None and e.state in ("window", "decode") for e in self.entries):
            return                                       # live streams first
        for f in self.files.values():
            n = len(f.run.features)
            while f.error is None and f.next_chunk < n and f.held() < f.limit:
                job = _ChunkJob(f.run, f.next_chunk)
                f.next_chunk += 1
                f.run.jobs.append(job)
                self.add_job(job)
                e = self.entries[-1]
                e.file = f
                f.active.append(e)

    def _finalise_files(self) -> None:
        """Segments and words of every file's decoded chunks, in chunk order: the word-timestamp carry-over
        (``last_speech_timestamp``) runs through them as through the one-shot pipeline's groups."""
        from . import vad as vad_mod
        sr = self.m.feature_extractor.sampling_rate
        for f in self.files.values():
            for e in list(f.active):
                if e.state == "done" and e.error is not None and f.error is None:
                    f.error = e.error
            while f.error is None and f.next_final in f.decoded:
                e = f.decoded.pop(f.next_final)
                j = e.job
                try:
                    j.finish_window()
                except Exception as ex:
                    f.error = ex
                j.enc = None
                if e.parent is not None:
                    e.parent.done_one()
                    e.parent = None
                f.next_final += 1
                f.steps.append(j.steps)
                if f.error is not None:
                    break
                for s in j.segments:
                    f.n_ids += 1
                    s.id = f.n_ids
                f.segments.extend(restore_speech_timestamps(j.segments, f.run.clips, sr, vad_mod))
            if f.error is not None:
                for e in list(f.active):
                    self.cancel(e.handle)
                f.active = []

    # -- the three parts of a round -----------------------------------------------------------------
    def _encode_pending(self) -> None:
        """Encode the next 30 s window of every stream that needs one (groups of at most ``engine.max_streams``, never
        more windows than the encoder slot pool has free); language id + prompt for each."""
        m = self.m
        tm = getattr(m, "last_timing", None) or {}
        cap = int(getattr(m.model, "max_streams", 0) or 0) or max(1, len(self.entries))
        need = [e for e in self.entries if e.state == "window"]
        free = getattr(m.model, "free_slots", None)
        if callable(free):
            need = need[:max(0, free())]
        for g0 in range(0, len(need), cap):
            grp = need[g0:g0 + cap]
            t0 = time.perf_counter()
            try:
                enc = m.encode(m._stack_windows([e.window for e in grp]))
            except Exception as ex:
                for e in grp:
                    e.error, e.state = ex, "done"
                continue
            tm["encode"] = tm.get("encode", 0.0) + time.perf_counter() - t0
            parent = _EncGroup(enc, len(grp))
            for k, e in enumerate(grp):
                e.parent, e.index, e.window = parent, k, None
                e.job.enc = enc.select([k]) if hasattr(enc, "select") else _EncoderSlice(enc, k)
            for e in grp:
                try:
                    e.job.prepare_decode()
                    e.state = "decode"
                except Exception as ex:
                    self._fail(e, ex)

    def _generate_groups(self, entries: List[_Entry]) -> List[_Entry]:
        """ONE run-to-completion ``generate`` call per distinct option set over ``entries``; returns those whose window
        settled (the others stay in "decode" for the next rung of the temperature ladder)."""
        m = self.m
        tm = getattr(m, "last_timing", None) or {}
        groups: Dict[str, List[_Entry]] = {}
        kwargs = {}
        for e in entries:
            try:
                kw = e.job.generate_kwargs()
            except Exception as ex:
                self._fail(e, ex)
                continue
            kwargs[e.handle] = kw
            key = {a: v for a, v in kw.items() if a != "max_length"}
            groups.setdefault(json.dumps(key, sort_keys=True, default=list), []).append(e)
        settled: List[_Entry] = []
        for _key, es in groups.items():
            kw = dict(kwargs[es[0].handle])
            lengths = [kwargs[e.handle]["max_length"] for e in es]
            if len(set(lengths)) > 1:
                kw["max_length_per_stream"] = lengths
                kw["max_length"] = max(lengths)
            t0 = time.perf_counter()
            try:
                outs = m.model.generate(_join_encoded([e.job.enc for e in es]), [e.job.prompt for e in es], **kw)
            except Exception as ex:
                for e in es:
                    self._fail(e, ex)
                continue
            t1 = time.perf_counter()
            for e, r in zip(es, outs):
                if e.job.accept(r):
                    settled.append(e)
            tm["generate"] = tm.get("generate", 0.0) + t1 - t0
            tm["host_decode"] = tm.get("host_decode", 0.0) + time.perf_counter() - t1
        return settled

    def _settle(self, settled: List[_Entry]) -> None:
        """Batched word alignment + window post-processing of the streams whose decode settled; each moves on to its
        next window or is done."""
        m = self.m
        tm = getattr(m, "last_timing", None) or {}
        t0 = time.perf_counter()
        try:
            m._align_entries(settled)
        except Exception as ex:
            for e in settled:
                self._fail(e, ex)
            settled = []
        for e in settled:
            j = e.job
            if e.file is not None:
                # a file's chunk: its segments and words are finalised in chunk order (_finalise_files); the encoder
                # slot goes back now unless word timestamps still need it (an engine whose outputs cannot be joined)
                if not (j.opt.word_timestamps and j._align_result is None):
                    j.enc = None
                    e.parent.done_one()
                    e.parent = None
                e.file.decoded[j.index] = e
                e.file.active.remove(e)
                e.state = "done"
                continue
            try:
                j.finish_window()
                if j.single_window:
                    j.seek = j.content_frames     # bench switch: one 30 s window per chunk (pinned work)
                nxt = j.advance_window()
            except Exception as ex:
                self._fail(e, ex)
                continue
            j.enc = None
            e.parent.done_one()
            e.parent = None
            e.window, e.state = nxt, ("window" if nxt is not None else "done")
        tm["finish"] = tm.get("finish", 0.0) + time.perf_counter() - t0

    def _fail(self, e: _Entry, ex: Exception) -> None:
        e.error, e.state = ex, "done"
        e.job.enc = None
        if e.parent is not None:
            e.parent.done_one()
            e.parent = None


def _lowbias32(x: int) -> int:
    x &= 0xFFFFFFFF
    x ^= x >> 16
    x = (x * 0x7FEB352D) & 0xFFFFFFFF
    x ^= x >> 15
    x = (x * 0x846CA68B) & 0xFFFFFFFF
    return x ^ (x >> 16)


def session_noise_seed(handle: int, seek: int, rung: int) -> int:
    """32-bit noise seed of a sampling rung decoded in a step-round decode session (noise key 0):
    ``lowbias32(lowbias32(lowbias32(handle) ^ seek) ^ rung)`` over the stream's handle in its ``TranscribeSession``, the
    window's ``seek`` (frames) and the rung's index in the temperature ladder.  A stream's draws therefore depend only
    on the stream itself -- not on which streams share its rounds or when it arrived."""
    return _lowbias32(_lowbias32(_lowbias32(handle) ^ (seek & 0xFFFFFFFF)) ^ (rung & 0xFFFFFFFF))


ENGINE_MAX_INITIAL_TIMESTAMP_INDEX = 50     # generate's default, which BatchedInferencePipeline's chunks decode under


def _rules_fit(ds, skw: dict) -> bool:
    """Whether a stream with session options ``skw`` can join the open session ``ds`` with rules of its own: the session
    takes per-stream rules, and the stream's beam width fits the session's rows per stream (a session that does not
    report ``rows_per_stream`` takes only its own width)."""
    if not getattr(ds, "supports_rules", False):
        return False
    if any(skw.get(k, d) != d for k, d in (("repetition_penalty", 1), ("no_repeat_ngram_size", 0))):
        return False
    width = int(skw.get("beam_size", 5))
    rows = getattr(ds, "rows_per_stream", None)
    fits = width <= int(rows) if rows is not None else width == int(ds.beam_size)
    return fits and int(skw.get("num_hypotheses", 1)) == 1


class _FileRun:
    """A batched file in a ``TranscribeSession``: which chunks have started, are decoding, wait for an earlier chunk,
    or are finalised."""

    def __init__(self, run: "_ChunkRun", handle: int, limit: int):
        self.run, self.handle, self.limit = run, handle, int(limit)   # limit: streams the file may hold at once
        self.next_chunk = 0                      # next chunk to enter the session
        self.active: List[_Entry] = []           # chunks in the session, not yet decoded
        self.decoded: Dict[int, _Entry] = {}     # chunk index -> decoded chunk waiting for the earlier ones
        self.next_final = 0                      # next chunk to finalise
        self.segments: List[Segment] = []
        self.n_ids = 0
        self.steps: List[int] = []
        self.error: Optional[Exception] = None

    @property
    def done(self) -> bool:
        return self.error is not None or self.next_final >= len(self.run.features)

    def held(self) -> int:
        """Chunks in the session, plus decoded chunks waiting for an earlier one that still hold an encoder slot."""
        return len(self.active) + sum(1 for e in self.decoded.values() if e.parent is not None)


def _join_encoded(views: List[Any]):
    """Encoder outputs of several streams (views into possibly different ``encode`` calls) as ONE batch for generate /
    align.  Engine handles are slot lists and join without copying; a mocked engine must hand out handles with ``join``."""
    if len(views) == 1:
        return views[0]
    first = views[0]
    if hasattr(first, "join"):
        return first.join(views)
    raise TypeError("this engine cannot batch encoder outputs of different encode() calls")


# --------------------------------------------------------------------------- the model
class B200WhisperModel:
    def __init__(self, model_size_or_path: str = "small.en", device: str = "cuda", device_index: Union[int, List[int]] = 0,
                 compute_type: str = "float16", cpu_threads: int = 0, num_workers: int = 1,
                 download_root: Optional[str] = None, local_files_only: bool = True, files: dict = None,
                 engine=None, hf_tokenizer=None, feature_extractor=None, weights=None, seed: int = 0,
                 max_streams: int = 8, max_beam: int = 5, vad=None, **model_kwargs):
        """``engine`` / ``hf_tokenizer`` / ``feature_extractor`` injection is for tests; the
        product path builds the CUDA engine (whisperlive_b200.engine.B200Whisper) and fails
        loudly when libwlb200.so, a GPU, the checkpoint or tokenizer.json is missing.
        ``weights="random"`` / ``hf_tokenizer="synthetic"`` are the explicit opt-ins bench.py and
        the tests use (no checkpoints offline).
        ``vad``: None gates ``vad_filter`` streams with ``faster_whisper.vad`` (CPU Silero, as the reference does); a
        module with that interface replaces it; ``"device"`` computes the Silero probabilities on this model's own GPU
        context (``vad.DeviceVad``, the Silero weights from ``WLB200_VAD_MODEL`` or faster-whisper's bundled model; with
        ``weights="random"`` seeded random ones)."""
        self.logger = logger
        if engine is None:
            from .engine import B200Whisper  # raises if the CUDA library cannot be loaded
            engine = B200Whisper.from_model(model_size_or_path, device_index=device_index, compute_type=compute_type,
                                            weights=weights, seed=seed, max_streams=max_streams, max_beam=max_beam,
                                            download_root=download_root, local_files_only=local_files_only)
        if isinstance(vad, str):
            if vad != "device":
                raise ValueError(f"vad={vad!r}: pass None, a faster_whisper.vad-like module, or 'device'")
            from .vad import DeviceVad
            vad = DeviceVad(engine, weights="random" if weights == "random" else None, seed=seed)
        self._vad = vad
        self.model = engine
        self._spk_weights = "random" if weights == "random" else None   # loaded by the first speaker_embeddings call
        self._spk_seed = seed
        self._spk_loaded = False
        model_dir = getattr(engine, "model_dir", None) or model_size_or_path
        if isinstance(hf_tokenizer, str):
            if hf_tokenizer != "synthetic":
                raise ValueError("hf_tokenizer must be a tokenizers.Tokenizer, None, or the explicit opt-in 'synthetic'")
            from .tokenizer import build_synthetic_tokenizer
            hf_tokenizer = build_synthetic_tokenizer(engine.vocab_size)
        if hf_tokenizer is None:
            hf_tokenizer = self._load_tokenizer(model_dir, files)
        self.hf_tokenizer = hf_tokenizer
        if feature_extractor is None:
            from .feature_extractor import FeatureExtractor
            feature_extractor = FeatureExtractor(engine=engine, **self._get_feature_kwargs(model_dir, files))
        self.feature_extractor = feature_extractor
        self.input_stride = 2
        self.num_samples_per_token = self.feature_extractor.hop_length * self.input_stride
        self.frames_per_second = self.feature_extractor.sampling_rate // self.feature_extractor.hop_length
        self.tokens_per_second = self.feature_extractor.sampling_rate // self.num_samples_per_token
        self.time_precision = 0.02
        self.max_length = 448

    # -- construction helpers ----------------------------------------------------------------
    def _load_tokenizer(self, path: str, files: Optional[dict]):
        import tokenizers
        if files and "tokenizer.json" in files:
            return tokenizers.Tokenizer.from_buffer(files["tokenizer.json"])
        cand = os.path.join(path, "tokenizer.json") if isinstance(path, str) else None
        if cand and os.path.isfile(cand):
            return tokenizers.Tokenizer.from_file(cand)
        # reference :620-656 resolves tokenizer.json from the model directory or the hub; there is no fallback
        # vocabulary (a transcriber that emits made-up text must never start silently)
        raise FileNotFoundError(
            f"tokenizer.json not found for {path!r}: pass a model directory that holds it, files={{'tokenizer.json': ...}}, "
            "or hf_tokenizer='synthetic' (fabricated vocabulary, bench/tests only)")

    def _get_feature_kwargs(self, path: str, files: Optional[dict]) -> dict:
        cfg: dict = {}
        raw = (files or {}).get("preprocessor_config.json")
        try:
            if raw:
                cfg = json.loads(raw)
            elif isinstance(path, str) and os.path.isfile(os.path.join(path, "preprocessor_config.json")):
                with open(os.path.join(path, "preprocessor_config.json"), "r", encoding="utf-8") as f:
                    cfg = json.load(f)
        except json.JSONDecodeError as e:
            self.logger.warning("Could not load preprocessor config: %s", e)
        keep = ("feature_size", "sampling_rate", "hop_length", "chunk_length", "n_fft")
        out = {k: v for k, v in cfg.items() if k in keep}
        out.setdefault("feature_size", self.model.n_mels)
        return out

    @property
    def supported_languages(self) -> List[str]:
        return list(LANGUAGE_CODES) if self.model.is_multilingual else ["en"]

    @property
    def device_bytes(self) -> int:
        """Device memory the engine context holds right now (``B200Whisper.device_bytes``)."""
        return int(self.model.device_bytes)

    def destroy(self) -> None:
        """Free the engine context and its device memory now (a model registry evicting this model)."""
        self.model.destroy()

    def speaker_embeddings(self, audios: Sequence[np.ndarray]) -> np.ndarray:
        """Speaker embeddings [B, 256] of 16 kHz segments (at least 400 samples each) on this model's engine context, one
        ``wl_spk_embed`` call for all of them.  The first call loads the wespeaker weights (``speaker.resolve_weights``:
        ``WLB200_SPK_MODEL`` or a local snapshot of the reference's default embedding model; seeded random ones when the
        model itself was built with ``weights="random"``)."""
        if not self._spk_loaded:
            from .speaker import resolve_weights
            self.model.spk_load(resolve_weights(self._spk_weights, self._spk_seed))
            self._spk_loaded = True
        return self.model.spk_embeddings(audios)

    # -- Boundary B ---------------------------------------------------------------------------
    def transcribe(self, audio: np.ndarray, language: Optional[str] = None, task: str = "transcribe",
                   log_progress: bool = False, beam_size: int = 5, best_of: int = 5, patience: float = 1,
                   length_penalty: float = 1, repetition_penalty: float = 1, no_repeat_ngram_size: int = 0,
                   temperature: Union[float, Sequence[float]] = DEFAULT_TEMPERATURES,
                   compression_ratio_threshold: Optional[float] = 2.4, log_prob_threshold: Optional[float] = -1.0,
                   no_speech_threshold: Optional[float] = 0.6, condition_on_previous_text: bool = True,
                   prompt_reset_on_temperature: float = 0.5, initial_prompt=None, prefix: Optional[str] = None,
                   suppress_blank: bool = True, suppress_tokens: Optional[List[int]] = [-1],
                   without_timestamps: bool = False, max_initial_timestamp: float = 1.0, word_timestamps: bool = False,
                   prepend_punctuations: str = PUNCT_PREPEND, append_punctuations: str = PUNCT_APPEND,
                   multilingual: bool = False, vad_filter: bool = False, vad_parameters=None,
                   max_new_tokens: Optional[int] = None, chunk_length: Optional[int] = None,
                   clip_timestamps: Union[str, List[float]] = "0", hallucination_silence_threshold: Optional[float] = None,
                   hotwords: Optional[str] = None, language_detection_threshold: Optional[float] = 0.5,
                   language_detection_segments: int = 1):
        """Single-stream entry with the reference's keyword surface; a batch of one."""
        kw = dict(locals())
        kw.pop("self")
        audio = kw.pop("audio")
        return self.transcribe_batch([audio], [kw])[0]

    def transcribe_batch(self, audios: Sequence[np.ndarray], per_stream_kwargs: Optional[Sequence[dict]] = None):
        """Transcribe several independent streams together.  Returns ``[(segments, info)]`` in
        order; an empty (after VAD) stream yields ``(None, None)`` like reference :860-861."""
        self.last_timing = {"prepare": 0.0, "mel": 0.0, "encode": 0.0, "generate": 0.0, "host_decode": 0.0, "finish": 0.0}
        sess = TranscribeSession(self)
        handles = sess.add_streams(audios, per_stream_kwargs, resident_ok=True)
        while sess.pending():
            sess.round()
        return [sess.result(h) for h in handles]

    # -- stream preparation (reference :811-861) --------------------------------------------------
    _DEFAULTS = dict(language=None, task="transcribe", log_progress=False, beam_size=5, best_of=5, patience=1,
                     length_penalty=1, repetition_penalty=1, no_repeat_ngram_size=0, temperature=DEFAULT_TEMPERATURES,
                     compression_ratio_threshold=2.4, log_prob_threshold=-1.0, no_speech_threshold=0.6,
                     condition_on_previous_text=True, prompt_reset_on_temperature=0.5, initial_prompt=None, prefix=None,
                     suppress_blank=True, suppress_tokens=[-1], without_timestamps=False, max_initial_timestamp=1.0,
                     word_timestamps=False, prepend_punctuations=PUNCT_PREPEND, append_punctuations=PUNCT_APPEND,
                     multilingual=False, vad_filter=False, vad_parameters=None, max_new_tokens=None, chunk_length=None,
                     clip_timestamps="0", hallucination_silence_threshold=None, hotwords=None,
                     language_detection_threshold=0.5, language_detection_segments=1)

    def _prepare_stream(self, audio: np.ndarray, kw: dict) -> Optional[dict]:
        return self._gate_stream(*self._stream_input(audio, kw))

    def _stream_input(self, audio, kw: dict) -> Tuple[np.ndarray, dict, bool]:
        """The stream's PCM (decoded when given as a path / bytes / file), its full keyword set, and the bench-only
        single-window flag."""
        single_window = bool(kw.pop("_single_window", False))   # not part of the reference surface (bench.py only)
        full = dict(self._DEFAULTS)
        unknown = set(kw) - set(full)
        if unknown:
            raise TypeError(f"transcribe() got unexpected keyword arguments {sorted(unknown)}")
        full.update(kw)
        kw = full
        sr = self.feature_extractor.sampling_rate
        if not isinstance(audio, np.ndarray):
            from .audio import decode_audio
            audio = decode_audio(audio, sampling_rate=sr)
        if kw["multilingual"] and not self.model.is_multilingual:
            self.logger.warning("The current model is English-only but the multilingual parameter is set to True; "
                                "setting to False instead.")
            kw["multilingual"] = False
        return audio, kw, single_window

    @staticmethod
    def _vad_options(vad, vad_parameters):
        if vad_parameters is None:
            return vad.VadOptions()
        if isinstance(vad_parameters, dict):
            return vad.VadOptions(**vad_parameters)
        return vad_parameters

    def _gate_stream(self, audio: np.ndarray, kw: dict, single_window: bool, speech_chunks=None) -> Optional[dict]:
        """VAD clipping (``speech_chunks``: already found for this stream by a batched VAD call) and the stream record."""
        sr = self.feature_extractor.sampling_rate
        duration = audio.shape[0] / sr
        duration_after_vad = duration
        vad_parameters = kw["vad_parameters"]
        if kw["vad_filter"] and kw["clip_timestamps"] == "0":
            vad = self._vad or _load_vad()
            vad_parameters = self._vad_options(vad, vad_parameters)
            if speech_chunks is None:
                speech_chunks = vad.get_speech_timestamps(audio, vad_parameters)
            chunks, _meta = vad.collect_chunks(audio, speech_chunks)
            audio = np.concatenate(chunks, axis=0) if len(chunks) else audio[:0]
            duration_after_vad = audio.shape[0] / sr
        if audio.shape[0] == 0:
            return None
        return dict(audio=np.ascontiguousarray(audio, dtype=np.float32), kw=kw, duration=duration,
                    duration_after_vad=duration_after_vad, speech_chunks=speech_chunks, vad_parameters=vad_parameters,
                    language=None, language_probability=1, all_language_probs=None, single_window=single_window)

    def _resolve_languages(self, prepared: List[dict]) -> None:
        """Reference :868-907, batched: one detect_language pass over all streams that need it."""
        need = []
        for p in prepared:
            lang = p["kw"]["language"]
            if lang is None:
                if not self.model.is_multilingual:
                    p["language"], p["language_probability"] = "en", 1
                else:
                    need.append(p)
            else:
                if not self.model.is_multilingual and lang != "en":
                    self.logger.warning("The current model is English-only but the language parameter is set to "
                                        "'%s'; using 'en' instead." % lang)
                    lang = "en"
                p["language"], p["language_probability"] = lang, 1
        for p in need:
            kw = p["kw"]
            clips = kw["clip_timestamps"]
            start_ts = float(clips.split(",")[0]) if isinstance(clips, str) else clips[0]
            content_frames = p["features"].shape[-1] - 1
            seek = int(start_ts * self.frames_per_second) if start_ts * self.frames_per_second < content_frames else 0
            p["language"], p["language_probability"], p["all_language_probs"] = self.detect_language(
                features=p["features"][..., seek:], language_detection_segments=kw["language_detection_segments"],
                language_detection_threshold=kw["language_detection_threshold"])

    def _make_options(self, tok: Tokenizer, kw: dict) -> TranscriptionOptions:
        t = kw["temperature"]
        sup = kw["suppress_tokens"]
        return TranscriptionOptions(
            beam_size=kw["beam_size"], best_of=kw["best_of"], patience=kw["patience"],
            length_penalty=kw["length_penalty"], repetition_penalty=kw["repetition_penalty"],
            no_repeat_ngram_size=kw["no_repeat_ngram_size"], log_prob_threshold=kw["log_prob_threshold"],
            no_speech_threshold=kw["no_speech_threshold"],
            compression_ratio_threshold=kw["compression_ratio_threshold"],
            condition_on_previous_text=kw["condition_on_previous_text"],
            prompt_reset_on_temperature=kw["prompt_reset_on_temperature"],
            temperatures=list(t) if isinstance(t, (list, tuple)) else [t], initial_prompt=kw["initial_prompt"],
            prefix=kw["prefix"], suppress_blank=kw["suppress_blank"],
            suppress_tokens=get_suppressed_tokens(tok, list(sup)) if sup else sup,
            without_timestamps=kw["without_timestamps"], max_initial_timestamp=kw["max_initial_timestamp"],
            word_timestamps=kw["word_timestamps"], prepend_punctuations=kw["prepend_punctuations"],
            append_punctuations=kw["append_punctuations"], multilingual=kw["multilingual"],
            max_new_tokens=kw["max_new_tokens"], clip_timestamps=kw["clip_timestamps"],
            hallucination_silence_threshold=kw["hallucination_silence_threshold"], hotwords=kw["hotwords"])

    # -- the round scheduler ---------------------------------------------------------------------
    def _run_jobs(self, jobs: List[_StreamJob]) -> None:
        """Run the window state machines of ``jobs`` to completion (``transcribe_batch``, ``generate_segments``)."""
        sess = TranscribeSession(self)
        for j in jobs:
            sess.add_job(j)
        while sess.pending():
            sess.round()
        for e in sess.entries:
            if e.error is not None:
                raise e.error

    def open_session(self) -> "TranscribeSession":
        """Incremental front end for a scheduler: ``add()`` streams at any time, ``round()`` advances everything that
        is in flight by one device round."""
        return TranscribeSession(self)

    def _align_entries(self, entries: List["_Entry"]) -> None:
        """K14 batched: ONE ``align`` call (one teacher-forced pass over all positions of all streams, DTW on the device)
        for every stream of the round that wants word timestamps -- the reference aligns stream by stream
        (:1230, :1657-1663).  Streams are grouped by sot sequence (language / task), which ``align`` takes once per call.
        The per-stream call inside ``finish_window`` remains the fallback for engines whose handles cannot be joined."""
        groups: Dict[Tuple[int, ...], List[Tuple[_StreamJob, List[int]]]] = {}
        for e in entries:
            j = e.job
            if not j.opt.word_timestamps or not hasattr(j.enc, "join"):
                continue
            toks = j.alignment_request()
            if toks is not None:
                groups.setdefault(tuple(j.tok.sot_sequence), []).append((j, toks))
        for sot_seq, items in groups.items():
            res = self.model.align(_join_encoded([j.enc for j, _ in items]), list(sot_seq), [t for _, t in items],
                                   [j.segment_size for j, _ in items], median_filter_width=7)
            for (j, _), r in zip(items, res):
                j._align_result = r

    def _stack_windows(self, views: List[np.ndarray]) -> np.ndarray:
        """[B, n_mels, 3000] batch of zero-padded windows, written straight into a buffer that is reused from call to
        call (the 49 MB batch of 32 large-v3 windows is otherwise allocated, page-faulted and copied twice per step:
        np.pad per stream, then np.stack).  The engine consumes the batch before encode() returns, and the buffer is
        per thread, so nothing else can touch it in between."""
        fe = self.feature_extractor
        if hasattr(views[0], "window"):
            return [v.window(fe.nb_max_frames) for v in views]      # resident: the device gathers + pads
        n_frames, n_mels = fe.nb_max_frames, views[0].shape[0]
        tls = self.__dict__.setdefault("_win_tls", threading.local())   # one buffer per calling thread: no sharing
        buf = getattr(tls, "buf", None)
        if buf is None or buf.shape[0] < len(views) or buf.shape[1] != n_mels or buf.shape[2] != n_frames:
            buf = tls.buf = np.zeros((len(views), n_mels, n_frames), dtype=np.float32)
        out = buf[:len(views)]
        for k, v in enumerate(views):
            t = v.shape[1]
            out[k, :, :t] = v
            out[k, :, t:] = 0.0
        return out

    def generate_segments(self, features: np.ndarray, tokenizer: Tokenizer, options: TranscriptionOptions,
                          log_progress=False, encoder_output=None) -> List[Segment]:
        """Reference :1049-1337 for one stream (returns a list, like the vendored fork)."""
        job = _StreamJob(self, features, tokenizer, options)
        self._run_jobs([job])
        return job.segments

    def encode(self, features: np.ndarray):
        """Reference :1339-1348.  Also takes features resident on the device (one ``ResidentFeatures`` view or the
        window list ``_stack_windows`` builds from them)."""
        if hasattr(features, "window"):
            return self.model.encode_windows([features.window(self.feature_extractor.nb_max_frames)])
        if isinstance(features, list):
            return self.model.encode_windows(features)
        if features.ndim == 2:
            features = features[None]
        return self.model.encode(np.ascontiguousarray(features, dtype=np.float32), to_cpu=False)

    def generate_with_fallback(self, encoder_output, prompt: List[int], tokenizer: Tokenizer,
                               options: TranscriptionOptions):
        """Reference :1350-1478 for one stream: (result, avg_logprob, temperature, compression_ratio)."""
        job = _StreamJob.__new__(_StreamJob)
        job.m, job.tok, job.opt, job.prompt = self, tokenizer, options, list(prompt)
        job.temp_idx, job.tried, job.below_cr = 0, [], []
        while True:
            r = self.model.generate(encoder_output, [job.prompt], **job.generate_kwargs())[0]
            if job.accept(r):
                d = job.decoded
                return d.result, d.avg_logprob, d.temperature, d.compression_ratio

    def get_prompt(self, tokenizer: Tokenizer, previous_tokens: List[int], without_timestamps: bool = False,
                   prefix: Optional[str] = None, hotwords: Optional[str] = None) -> List[int]:
        """Reference :1480-1513: [sot_prev, hotwords, previous[-223:]] + sot sequence (+ notimestamps) (+ prefix)."""
        half = self.max_length // 2
        use_hotwords = bool(hotwords) and not prefix
        prompt: List[int] = []
        if previous_tokens or use_hotwords:
            prompt.append(tokenizer.sot_prev)
            if use_hotwords:
                hw = tokenizer.encode(" " + hotwords.strip())
                prompt.extend(hw[:half - 1] if len(hw) >= half else hw)
            if previous_tokens:
                prompt.extend(previous_tokens[-(half - 1):])
        prompt.extend(tokenizer.sot_sequence)
        if without_timestamps:
            prompt.append(tokenizer.no_timestamps)
        if prefix:
            pt = tokenizer.encode(" " + prefix.strip())
            if len(pt) >= half:
                pt = pt[:half - 1]
            if not without_timestamps:
                prompt.append(tokenizer.timestamp_begin)
            prompt.extend(pt)
        return prompt

    def _split_segments_by_timestamps(self, tokenizer: Tokenizer, tokens: List[int], time_offset: float,
                                      segment_size: int, segment_duration: float, seek: int):
        """Reference :970-1047: cut the token list at consecutive timestamp pairs; returns
        (segments, new_seek, single_timestamp_ending)."""
        tb = tokenizer.timestamp_begin
        is_ts = [t >= tb for t in tokens]
        single_ending = len(tokens) >= 2 and (not is_ts[-2]) and is_ts[-1]
        cuts = [i for i in range(1, len(tokens)) if is_ts[i] and is_ts[i - 1]]
        out = []
        if cuts:
            if single_ending:
                cuts.append(len(tokens))
            lo = 0
            for hi in cuts:
                piece = tokens[lo:hi]
                out.append(dict(seek=seek, start=time_offset + (piece[0] - tb) * self.time_precision,
                                end=time_offset + (piece[-1] - tb) * self.time_precision, tokens=piece))
                lo = hi
            if single_ending:
                seek += segment_size  # no speech after the final timestamp
            else:
                seek += (tokens[lo - 1] - tb) * self.input_stride  # resume at the last closed timestamp
        else:
            duration = segment_duration
            stamps = [t for t in tokens if t >= tb]
            if stamps and stamps[-1] != tb:
                duration = (stamps[-1] - tb) * self.time_precision
            out.append(dict(seek=seek, start=time_offset, end=time_offset + duration, tokens=tokens))
            seek += segment_size
        return out, seek, single_ending

    # -- word timestamps (K14 host part; reference :1515-1714) ------------------------------------
    def add_word_timestamps(self, segments: List[List[dict]], tokenizer: Tokenizer, encoder_output,
                            num_frames: Union[int, Sequence[int]], prepend_punctuations: str, append_punctuations: str,
                            last_speech_timestamp: float, precomputed=None):
        """``num_frames``: one count for every window, or one per window (``BatchedInferencePipeline``, reference
        :163-172, whose chunks differ in length)."""
        if len(segments) == 0:
            return
        per_seg_tokens = [[[t for t in sub["tokens"] if t < tokenizer.eot] for sub in seg] for seg in segments]
        text_tokens = [list(itertools.chain.from_iterable(x)) for x in per_seg_tokens]
        alignments = self.find_alignment(tokenizer, text_tokens, encoder_output, num_frames, results=precomputed)
        limits = []
        for al in alignments:
            durs = np.array([w["end"] - w["start"] for w in al])
            durs = durs[durs.nonzero()]
            med = min(0.7, float(np.median(durs))) if len(durs) > 0 else 0.0
            mx = med * 2
            if len(durs) > 0:
                marks = ".。!！?？"
                for i in range(1, len(al)):
                    if al[i]["end"] - al[i]["start"] > mx:
                        if al[i]["word"] in marks:
                            al[i]["end"] = al[i]["start"] + mx
                        elif al[i - 1]["word"] in marks:
                            al[i]["start"] = al[i]["end"] - mx
            merge_punctuations(al, prepend_punctuations, append_punctuations)
            limits.append((med, mx))
        for si, seg in enumerate(segments):
            wi = 0
            t0 = seg[0]["seek"] / self.frames_per_second
            med, mx = limits[si]
            al = alignments[si]
            for bi, sub in enumerate(seg):
                used = 0
                words = []
                n_sub = len(per_seg_tokens[si][bi])
                while wi < len(al) and used < n_sub:
                    tm = al[wi]
                    if tm["word"]:
                        words.append(dict(word=tm["word"], start=round(t0 + tm["start"], 2),
                                          end=round(t0 + tm["end"], 2), probability=tm["probability"]))
                    used += len(tm["tokens"])
                    wi += 1
                if words:
                    # a pause before: the first words cannot be longer than twice the median
                    if words[0]["end"] - last_speech_timestamp > med * 4 and (
                            words[0]["end"] - words[0]["start"] > mx
                            or (len(words) > 1 and words[1]["end"] - words[0]["start"] > mx * 2)):
                        if len(words) > 1 and words[1]["end"] - words[1]["start"] > mx:
                            b = max(words[1]["end"] / 2, words[1]["end"] - mx)
                            words[0]["end"] = words[1]["start"] = b
                        words[0]["start"] = max(0, words[0]["end"] - mx)
                    if sub["start"] < words[0]["end"] and sub["start"] - 0.5 > words[0]["start"]:
                        words[0]["start"] = max(0, min(words[0]["end"] - med, sub["start"]))
                    else:
                        sub["start"] = words[0]["start"]
                    if sub["end"] > words[-1]["start"] and sub["end"] + 0.5 < words[-1]["end"]:
                        words[-1]["end"] = max(words[-1]["start"] + med, sub["end"])
                    else:
                        sub["end"] = words[-1]["end"]
                    last_speech_timestamp = sub["end"]
                sub["words"] = words
        return last_speech_timestamp

    def find_alignment(self, tokenizer: Tokenizer, text_tokens: List[List[int]], encoder_output,
                       num_frames: Union[int, Sequence[int]], median_filter_width: int = 7,
                       results=None) -> List[List[dict]]:
        if len(text_tokens) == 0:
            return []
        if results is None:   # (the batched scheduler path hands in the engine results of its one align call)
            results = self.model.align(encoder_output, tokenizer.sot_sequence, text_tokens, num_frames,
                                       median_filter_width=median_filter_width)
        out = []
        for res, toks in zip(results, text_tokens):
            words, word_tokens = tokenizer.split_to_word_tokens(toks + [tokenizer.eot])
            if len(word_tokens) <= 1:
                out.append([])
                continue
            bounds = np.pad(np.cumsum([len(t) for t in word_tokens[:-1]]), (1, 0))
            if len(bounds) <= 1:
                out.append([])
                continue
            ti = np.array([p[0] for p in res.alignments])
            fi = np.array([p[1] for p in res.alignments])
            jumps = np.pad(np.diff(ti), (1, 0), constant_values=1).astype(bool)
            jump_times = fi[jumps] / self.tokens_per_second
            starts, ends = jump_times[bounds[:-1]], jump_times[bounds[1:]]
            probs = [np.mean(res.text_token_probs[i:j]) for i, j in zip(bounds[:-1], bounds[1:])]
            out.append([dict(word=w, tokens=t, start=s, end=e, probability=p)
                        for w, t, s, e, p in zip(words, word_tokens, starts, ends, probs)])
        return out

    # -- language id (K13 host part; reference :1716-1789) ----------------------------------------
    def detect_language(self, audio: Optional[np.ndarray] = None, features: Optional[np.ndarray] = None,
                        vad_filter: bool = False, vad_parameters=None, language_detection_segments: int = 1,
                        language_detection_threshold: float = 0.5):
        assert audio is not None or features is not None, "Either `audio` or `features` must be provided."
        fe = self.feature_extractor
        if audio is not None:
            if vad_filter:
                vad = self._vad or _load_vad()
                chunks, _ = vad.collect_chunks(audio, vad.get_speech_timestamps(audio, vad_parameters))
                audio = np.concatenate(chunks, axis=0)
            features = fe(audio[: language_detection_segments * fe.n_samples])
        features = features[..., : language_detection_segments * fe.nb_max_frames]
        votes: Dict[str, List[float]] = {}
        all_probs = None
        language, prob = None, 0.0
        for i in range(0, features.shape[-1], fe.nb_max_frames):
            enc = self.encode(pad_or_trim(features[..., i:i + fe.nb_max_frames], fe.nb_max_frames))
            all_probs = [(tok[2:-2], p) for tok, p in self.model.detect_language(enc)[0]]
            language, prob = all_probs[0]
            if prob > language_detection_threshold:
                return language, prob, all_probs
            votes.setdefault(language, []).append(prob)
        language = max(votes, key=lambda k: len(votes[k]))
        return language, max(votes[language]), all_probs


class _EncoderSlice:
    """Fallback sub-batch view for engines without ``select`` (e.g. a mocked engine)."""

    def __init__(self, enc, index):
        self.enc, self.index = enc, index


# --------------------------------------------------------------------------- batched long-file transcription
class _ChunkRun:
    """What the chunks of one ``BatchedInferencePipeline.transcribe`` call share: options, tokenizer, prompt, the
    features, the word-timestamp carry-over from chunk to chunk, and the group being decoded."""

    def __init__(self, model: "B200WhisperModel", tok: Tokenizer, options: TranscriptionOptions, audio_chunks,
                 metadata: List[dict], features: List[Any], clips: List[dict]):
        self.m, self.tok, self.opt = model, tok, options
        self.audio_chunks, self.metadata, self.features, self.clips = audio_chunks, metadata, features, clips
        self.last_speech_timestamp = 0.0
        self.jobs: List["_ChunkJob"] = []
        ip = options.initial_prompt
        previous = [] if ip is None else (tok.encode(ip) if isinstance(ip, str) else list(ip))   # reference :184-193
        self.prompt = model.get_prompt(tok, previous_tokens=previous, without_timestamps=options.without_timestamps,
                                       hotwords=options.hotwords)
        self.language_index = self.prompt.index(tok.language) if options.multilingual else -1

    def max_length(self) -> int:
        """Reference :195-209."""
        o, m, n = self.opt, self.m, len(self.prompt)
        max_length = m.max_length if o.max_new_tokens is None else n + o.max_new_tokens
        if max_length > m.max_length:
            raise ValueError(
                f"The length of the prompt is {n}, and the `max_new_tokens` {max_length - n}. Thus, the combined length "
                f"of the prompt and `max_new_tokens` is: {max_length}. This exceeds the `max_length` of the Whisper "
                f"model: {m.max_length}. You should either reduce the length of your prompt, or reduce the value of "
                f"`max_new_tokens`, so that their combined length is less that {m.max_length}.")
        return max_length

    def refresh_resident(self) -> None:
        """Features kept in HBM are valid until the next mel call on the engine; if one ran while the caller held the
        generator, compute them again (the same mel call, so the same values)."""
        if self.features and not getattr(self.features[0], "resident", True):
            fe = self.m.feature_extractor
            self.features = [pad_or_trim(f[..., :-1]) for f in fe.batch_resident(self.audio_chunks)]

    def chunk_language(self, job: "_ChunkJob") -> int:
        """Language token of ``job``'s chunk: the top language of ONE ``detect_language`` call over every chunk of the
        group whose encoder output is ready (reference :214-222)."""
        if job.language is None:
            todo = [j for j in self.jobs if j.enc is not None and j.language is None]
            for j, langs in zip(todo, self.m.model.detect_language(_join_encoded([j.enc for j in todo]))):
                j.language = self.tok.tokenizer.token_to_id(langs[0][0])
        return job.language


class _ChunkJob:
    """One speech chunk of ``BatchedInferencePipeline``, driven by ``TranscribeSession`` rounds like a ``_StreamJob``
    but with the reference's chunk rules (:121-254): one window, no previous text, no temperature ladder, no skipping
    for silence, every sub-segment emitted."""

    single_window = False

    def __init__(self, run: _ChunkRun, index: int):
        self.run, self.index = run, index
        self.m, self.tok, self.opt = run.m, run.tok, run.opt
        meta = run.metadata[index]
        # the reference reads start_time / end_time; faster-whisper 1.2.0's collect_chunks gives offset / duration
        # (start_time = offset, end_time = offset + duration), and the duration is taken back from the two the same way
        start_time, end_time = meta["offset"], meta["offset"] + meta["duration"]
        self.time_offset = start_time
        self.segment_duration = end_time - start_time
        self.segment_size = int(ceil(self.segment_duration) * self.m.frames_per_second)
        self.seek = int(start_time * self.m.frames_per_second)
        self.enc = None
        self.prompt: List[int] = []
        self.language: Optional[int] = None
        self.segments: List[Segment] = []
        self.current: Optional[List[dict]] = None
        self.steps = 0
        self._align_result = None
        self._started = False

    def advance_window(self):
        if self._started:
            return None
        self._started = True
        return self.run.features[self.index]

    def prepare_decode(self) -> None:
        self.prompt = list(self.run.prompt)
        if self.opt.multilingual:
            self.prompt[self.run.language_index] = self.run.chunk_language(self)

    def generate_kwargs(self) -> dict:
        """The reference's generate arguments (:224-238); what it leaves out stays at the engine's default
        (``max_initial_timestamp_index`` 50, ``sampling_topk`` 1, so ``sampling_temperature`` does not sample)."""
        o = self.opt
        return dict(beam_size=o.beam_size, patience=o.patience, length_penalty=o.length_penalty,
                    max_length=self.run.max_length(), suppress_blank=o.suppress_blank, suppress_tokens=o.suppress_tokens,
                    return_scores=True, return_no_speech_prob=True, sampling_temperature=o.temperatures[0],
                    repetition_penalty=o.repetition_penalty, no_repeat_ngram_size=o.no_repeat_ngram_size)

    temp_idx = 0      # one rung

    def session_kwargs(self) -> dict:
        """Options of a decode session opened for this chunk (``TranscribeSession.step_round``)."""
        kw = self.generate_kwargs()
        for k in ("max_length", "sampling_temperature"):
            kw.pop(k)
        return dict(kw, num_hypotheses=1)

    def stream_rules(self) -> dict:
        """What the chunk decodes under when it joins a session opened with other options."""
        o = self.opt
        return dict(beam_size=o.beam_size, patience=o.patience, length_penalty=o.length_penalty,
                    suppress_blank=o.suppress_blank, suppress_tokens=o.suppress_tokens,
                    max_initial_timestamp_index=ENGINE_MAX_INITIAL_TIMESTAMP_INDEX)

    def accept(self, result) -> bool:
        n = len(result.sequences_ids[0])
        self.result = result
        self.avg_logprob = result.scores[0] * (n ** self.opt.length_penalty) / (n + 1)
        self.steps = int(getattr(result, "steps", n))
        return True

    def split(self) -> None:
        pieces, _seek, _single = self.m._split_segments_by_timestamps(
            tokenizer=self.tok, tokens=self.result.sequences_ids[0], time_offset=self.time_offset,
            segment_size=self.segment_size, segment_duration=self.segment_duration, seek=0)
        self.current = [dict(seek=self.seek, start=p["start"], end=p["end"], tokens=p["tokens"]) for p in pieces]

    def alignment_request(self) -> List[int]:
        self.split()
        return [t for sub in self.current for t in sub["tokens"] if t < self.tok.eot]

    def finish_window(self) -> None:
        """Sub-segments (reference :128-162), words (:163-172; chunks settle in order, so the carry-over
        ``last_speech_timestamp`` runs through them as through the reference's one call per batch), records (:547-566)."""
        o, tok, run = self.opt, self.tok, self.run
        if self.current is None:
            self.split()
        if o.word_timestamps:
            pre = self._align_result
            run.last_speech_timestamp = self.m.add_word_timestamps(
                [self.current], tok, self.enc, [self.segment_size], o.prepend_punctuations, o.append_punctuations,
                run.last_speech_timestamp, precomputed=None if pre is None else [pre])
        for p in self.current:
            text = tok.decode(p["tokens"])
            self.segments.append(Segment(
                id=0, seek=p["seek"], start=round(p["start"], 3), end=round(p["end"], 3), text=text, tokens=p["tokens"],
                avg_logprob=self.avg_logprob, compression_ratio=get_compression_ratio(text),
                no_speech_prob=self.result.no_speech_prob, temperature=o.temperatures[0],
                words=[Word(**w) for w in p["words"]] if o.word_timestamps else None))


class BatchedInferencePipeline:
    """faster-whisper's batched long-file transcription (the reference vendors it: transcriber_faster_whisper.py
    :113-571): VAD cuts the file into speech chunks of at most ``chunk_length`` seconds, and every chunk is decoded on
    its own -- no previous-text prompt, no temperature ladder -- ``batch_size`` chunks per encode and ``generate``.

    Two things differ from the vendored code, both as faster-whisper 1.2.0 has them: the chunks come from
    ``collect_chunks(..., max_duration=chunk_length)`` (its ``offset`` / ``duration`` on the speech-only axis), and
    ``restore_speech_timestamps`` maps the segments and words back to the original time axis.

    On this engine one group is ``min(batch_size, max_streams)`` chunks: one mel call for the whole file, then per
    group one encode, one ``detect_language`` (``multilingual``), one ``generate`` and one ``align``
    (``word_timestamps``), driven by ``TranscribeSession`` rounds.  The calls are one-shot, so a ``TranscribeSession``
    with an open step-level decode session on the same model keeps its streams."""

    def __init__(self, model: "B200WhisperModel", scheduler=None, max_share: float = 0.5):
        """``scheduler``: a running ``RoundScheduler`` on the same model.  Its owner thread then decodes the file's
        chunks as streams of its running decode loop, beside the live connections, instead of one-shot calls on the
        caller's thread: a chunk enters as soon as an index is free (at most ``max_share`` of the indices, and live
        requests first), and the segments come out in chunk order as chunks settle.  The result is the same."""
        self.model = model
        self.scheduler = scheduler
        self.max_share = float(max_share)
        self.resident_features = True        # False: features always go through the host (tests compare the paths)
        self.group_steps: List[List[int]] = []   # token steps of every chunk, per group of the last transcribe call
        self.last_request = None             # the FileRequest of the last file sent to the scheduler

    def transcribe(self, audio, language: Optional[str] = None, task: str = "transcribe", log_progress: bool = False,
                   beam_size: int = 5, best_of: int = 5, patience: float = 1, length_penalty: float = 1,
                   repetition_penalty: float = 1, no_repeat_ngram_size: int = 0,
                   temperature: Union[float, List[float], Tuple[float, ...]] = [0.0, 0.2, 0.4, 0.6, 0.8, 1.0],
                   compression_ratio_threshold: Optional[float] = 2.4, log_prob_threshold: Optional[float] = -1.0,
                   no_speech_threshold: Optional[float] = 0.6, condition_on_previous_text: bool = True,
                   prompt_reset_on_temperature: float = 0.5, initial_prompt=None, prefix: Optional[str] = None,
                   suppress_blank: bool = True, suppress_tokens: Optional[List[int]] = [-1],
                   without_timestamps: bool = True, max_initial_timestamp: float = 1.0, word_timestamps: bool = False,
                   prepend_punctuations: str = PUNCT_PREPEND, append_punctuations: str = PUNCT_APPEND,
                   multilingual: bool = False, vad_filter: bool = True, vad_parameters=None,
                   max_new_tokens: Optional[int] = None, chunk_length: Optional[int] = None,
                   clip_timestamps: Optional[List[dict]] = None, hallucination_silence_threshold: Optional[float] = None,
                   batch_size: int = 8, hotwords: Optional[str] = None,
                   language_detection_threshold: Optional[float] = 0.5, language_detection_segments: int = 1):
        """Reference :256-532: ``(generator of Segment, TranscriptionInfo)``.  The generator decodes group by group as
        it is consumed.  ``compression_ratio_threshold``, ``log_prob_threshold``, ``no_speech_threshold``,
        ``condition_on_previous_text``, ``prompt_reset_on_temperature``, ``prefix``, ``max_initial_timestamp`` and
        ``hallucination_silence_threshold`` are accepted and unused, as in the reference; of ``temperature`` only the
        first value is kept."""
        if repetition_penalty != 1:
            raise NotImplementedError(f"repetition_penalty={repetition_penalty}: the engine implements only 1")
        if no_repeat_ngram_size != 0:
            raise NotImplementedError(f"no_repeat_ngram_size={no_repeat_ngram_size}: the engine implements only 0")
        m = self.model
        fe = m.feature_extractor
        sr = fe.sampling_rate
        if multilingual and not m.model.is_multilingual:
            m.logger.warning("The current model is English-only but the multilingual parameter is set to True; "
                             "setting to False instead.")
            multilingual = False
        if not isinstance(audio, np.ndarray):
            from .audio import decode_audio
            audio = decode_audio(audio, sampling_rate=sr)
        duration = audio.shape[0] / sr
        chunk_length = chunk_length or fe.chunk_length
        if not clip_timestamps:                                    # reference :393-417
            if vad_filter:
                vad = m._vad or _load_vad()
                if vad_parameters is None:
                    vad_parameters = vad.VadOptions(max_speech_duration_s=chunk_length, min_silence_duration_ms=160)
                elif isinstance(vad_parameters, dict):
                    params = {k: v for k, v in vad_parameters.items() if k != "max_speech_duration_s"}
                    vad_parameters = vad.VadOptions(**params, max_speech_duration_s=chunk_length)
                clip_timestamps = vad.get_speech_timestamps(audio, vad_parameters)
            elif duration < chunk_length:
                clip_timestamps = [{"start": 0, "end": audio.shape[0]}]
            else:
                raise RuntimeError("No clip timestamps found. Set 'vad_filter' to True or provide 'clip_timestamps'.")
        duration_after_vad = sum(c["end"] - c["start"] for c in clip_timestamps) / sr

        from . import vad as vad_mod
        audio_chunks, metadata = vad_mod.collect_chunks(audio, clip_timestamps, sr, max_duration=chunk_length)
        detect = language is None and m.model.is_multilingual
        features: List[Any] = []
        if duration_after_vad:
            # ONE mel call for every chunk; resident in HBM when the chunks fit one call and nothing needs host values
            cap = int(getattr(m.model, "max_streams", 0) or 0)
            resident = (self.resident_features and hasattr(fe, "batch_resident") and len(audio_chunks) <= cap
                        and not detect and self.scheduler is None)
            feats = fe.batch_resident(audio_chunks) if resident else fe.batch(audio_chunks)
            features = [f[..., :-1] for f in feats]

        all_language_probs = None
        if language is None:                                       # reference :431-467
            if not m.model.is_multilingual:
                language, language_probability = "en", 1
            else:
                language, language_probability, all_language_probs = m.detect_language(
                    features=np.concatenate(features + [np.full((m.model.n_mels, 1), -1.5, dtype="float32")], axis=1),
                    language_detection_segments=language_detection_segments,
                    language_detection_threshold=language_detection_threshold)
                m.logger.info("Detected language '%s' with probability %.2f", language, language_probability)
        else:
            if not m.model.is_multilingual and language != "en":
                m.logger.warning("The current model is English-only but the language parameter is set to '%s'; "
                                 "using 'en' instead." % language)
                language = "en"
            language_probability = 1
        tokenizer = Tokenizer(m.hf_tokenizer, m.model.is_multilingual, task=task, language=language)
        features = [pad_or_trim(f) for f in features]

        options = TranscriptionOptions(
            beam_size=beam_size, best_of=best_of, patience=patience, length_penalty=length_penalty,
            repetition_penalty=repetition_penalty, no_repeat_ngram_size=no_repeat_ngram_size,
            log_prob_threshold=log_prob_threshold, no_speech_threshold=no_speech_threshold,
            compression_ratio_threshold=compression_ratio_threshold,
            temperatures=temperature[:1] if isinstance(temperature, (list, tuple)) else [temperature],
            initial_prompt=initial_prompt, prefix=prefix, suppress_blank=suppress_blank,
            suppress_tokens=get_suppressed_tokens(tokenizer, suppress_tokens),
            prepend_punctuations=prepend_punctuations, append_punctuations=append_punctuations,
            max_new_tokens=max_new_tokens, hotwords=hotwords, word_timestamps=word_timestamps,
            hallucination_silence_threshold=None, condition_on_previous_text=False, clip_timestamps=clip_timestamps,
            prompt_reset_on_temperature=0.5, multilingual=multilingual, without_timestamps=without_timestamps,
            max_initial_timestamp=0.0)
        info = TranscriptionInfo(language=language, language_probability=language_probability, duration=duration,
                                 duration_after_vad=duration_after_vad, transcription_options=options,
                                 vad_options=vad_parameters, all_language_probs=all_language_probs)
        run = _ChunkRun(m, tokenizer, options, audio_chunks, metadata, features, clip_timestamps)
        self.group_steps = []
        if self.scheduler is not None:
            return self._scheduled_segments(run), info
        return self._segments(run, batch_size), info

    def _scheduled_segments(self, run: _ChunkRun):
        """The file as one request of the scheduler: segments as its chunks settle, in chunk order.  Closing the
        generator early cancels the chunks still in flight."""
        if not run.features:
            return
        from .scheduler import FileRequest
        req = self.last_request = FileRequest(run=run, max_share=self.max_share)
        self.scheduler.submit(req)
        n = 0
        try:
            while True:
                req.settled.event.clear()
                segs = req.settled.since(n)
                if segs:
                    n += len(segs)
                    yield from segs
                    continue
                if req.future.is_set():
                    if len(req.settled) > n:
                        continue
                    if req.error is not None:
                        raise req.error
                    break
                req.settled.event.wait(1.0)
        finally:
            if not req.future.is_set():
                req.cancel()
            self.group_steps = [list(req.steps)]

    def _segments(self, run: _ChunkRun, batch_size: int):
        """Reference :534-571, one ``TranscribeSession`` run per group; ids count on across groups."""
        m = self.model
        from . import vad as vad_mod
        cap = int(getattr(m.model, "max_streams", 0) or 0)
        group = max(1, min(batch_size, cap) if cap else batch_size)
        free = getattr(m.model, "free_slots", None)
        seg_idx = 0
        for g0 in range(0, len(run.features), group):
            run.refresh_resident()
            run.jobs = [_ChunkJob(run, k) for k in range(g0, min(g0 + group, len(run.features)))]
            sess = TranscribeSession(m)
            for j in run.jobs:
                sess.add_job(j)
            while sess.pending():
                if callable(free) and free() == 0:
                    raise RuntimeError("no free encoder slot: release encoder outputs held elsewhere on this model")
                sess.round()
            for e in sess.entries:
                if e.error is not None:
                    raise e.error
            self.group_steps.append([j.steps for j in run.jobs])
            segs = [s for j in run.jobs for s in j.segments]
            for s in segs:
                seg_idx += 1
                s.id = seg_idx
            yield from restore_speech_timestamps(segs, run.clips, m.feature_extractor.sampling_rate, vad_mod)
