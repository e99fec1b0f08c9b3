"""Oracle K12: logits processors + beam / greedy / sampling search (TEST INFRASTRUCTURE ONLY).

PARITY UNPINNED.  The reference delegates this row to ``ctranslate2.models.Whisper.generate``
(call sites whisper_live/transcriber/transcriber_faster_whisper.py:1394-1407,
whisper_live/batch_inference.py:342-357); CTranslate2 (4.x, pulled by
faster-whisper==1.2.0) is neither vendored in /root/reference nor installed, so
the algorithm below is restated from its published sources (src/models/whisper.cc
``ApplyTimestampRules`` / ``SuppressTokens*``; src/decoding.cc ``BeamSearch`` /
``GreedySearch``) and from OpenAI whisper/decoding.py ``ApplyTimestampRules`` which
CT2 re-implements.  What IS anchored in-tree: the score convention
``score = cum_logprob / len(tokens)**length_penalty`` that
transcriber_faster_whisper.py:1411-1414 inverts, ``max_initial_timestamp_index``
(:1361-1363), the suppress list (:1831-1853), and the result shape mocked at
tests/test_batch_inference.py:58-68.

Semantics restated:
  processors, in order, on the raw logits of each row (masking = -inf):
    1. suppress_tokens every step
    2. suppress_blank at the first generated step: blank (" ") and eot
    3. timestamp rules unless the prompt ends with <|notimestamps|>
       a. <|notimestamps|> never
       b. first step: only timestamps <= ts_begin + max_initial_timestamp_index
       c. after a timestamp: if the one before is a timestamp too -> no timestamp,
          else -> no text token (< eot)
       d. timestamps never decrease; a segment has non-zero length
       e. (steps > 0) if logsumexp(logp[ts]) > max(logp[text]) -> no text token
  then log-softmax.
  beam search: candidates = top 2K of (cum + logp) over the K live rows (first step:
  one row); walking the top K, an EOT candidate closes a hypothesis and its slot is
  refilled from candidates K..2K; a stream ends with max(1, round(K*patience))
  hypotheses or at the last step (everything in the top K closes).  The rounding is
  half away from zero, CT2's ``std::round`` as recalled from its sources, not pinned
  against a CT2 run: K=5 with patience 0.5 gives 3, K=3 with patience 1.5 gives 5.
  Ties break toward the lower flat index (row-major beam*vocab).
  greedy/sampling (K=1): argmax, or Gumbel-max with a counter hash
  (``gumbel_noise``) when sampling_topk != 1 and temperature > 0, ``num_hypotheses``
  independent rows.  A row whose every token is masked finishes without a token
  (the device's behaviour; CT2 leaves that case undefined).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

NEG_INF = float("-inf")


@dataclass
class VocabSpec:
    """Token ids the engine needs (CT2 reads them from the vocabulary / config.json)."""
    vocab: int
    eot: int
    sot: int
    no_speech: int
    no_timestamps: int
    timestamp_begin: int
    blank: int = 220  # " " in the GPT-2 byte-level BPE

    @classmethod
    def from_vocab_size(cls, vocab: int) -> "VocabSpec":
        multilingual = vocab >= 51865
        if not multilingual:
            eot, ts_begin = 50256, 50363
        else:
            n_lang = vocab - 51765 - 1
            eot, ts_begin = 50257, 50258 + 1 + n_lang + 6
        return cls(vocab=vocab, eot=eot, sot=eot + 1, no_speech=ts_begin - 2,
                   no_timestamps=ts_begin - 1, timestamp_begin=ts_begin)

    def language_ids(self) -> List[int]:
        n_lang = (self.vocab - 51765 - 1) if self.vocab >= 51865 else 0
        return list(range(self.sot + 1, self.sot + 1 + n_lang))


@dataclass
class GenOptions:
    beam_size: int = 5
    patience: float = 1.0
    num_hypotheses: int = 1
    length_penalty: float = 1.0
    max_length: int = 448
    suppress_blank: bool = True
    suppress_tokens: Sequence[int] = ()
    max_initial_timestamp_index: int = 50
    sampling_topk: int = 1
    sampling_temperature: float = 1.0
    seed: int = 0
    trace: bool = False


def max_new_tokens(prompt_len: int, max_length: int) -> int:
    """CT2 Whisper: decode at most min(max_length/2, max_length - prompt_len) tokens."""
    return max(0, min(max_length // 2, max_length - prompt_len))


def _hash_u32(x: np.ndarray) -> np.ndarray:
    """lowbias32 integer hash on uint32 arrays."""
    x = x.astype(np.uint64)
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x7FEB352D)) & np.uint64(0xFFFFFFFF)
    x ^= x >> np.uint64(15)
    x = (x * np.uint64(0x846CA68B)) & np.uint64(0xFFFFFFFF)
    x ^= x >> np.uint64(16)
    return x.astype(np.uint32)


def gumbel_noise(seed: int, row: int, step: int, vocab: int) -> np.ndarray:
    """Deterministic Gumbel(0,1) per (seed,row,step,token); the CUDA sampler uses the same hash."""
    idx = np.arange(vocab, dtype=np.uint32)
    key = _hash_u32(np.uint32((seed * 0x9E3779B1) & 0xFFFFFFFF) ^ _hash_u32(np.full(1, (row * 65537 + step) & 0xFFFFFFFF, dtype=np.uint32)))
    h = _hash_u32(idx ^ key)
    u = (h.astype(np.float64) + 0.5) / 4294967296.0
    return (-np.log(-np.log(u))).astype(np.float32)


def sample_begin(prompt: Sequence[int], spec: VocabSpec) -> int:
    """CT2's prompt length [upstream-recalled, models/whisper.cc]: index after <|startoftranscript|> and every
    following id in [sot, no_timestamps] (language, task, notimestamps).  Prompt tokens from there on -- the
    ``prefix`` built at transcriber_faster_whisper.py:1505-1511, including its leading <|0.00|> -- are treated as
    already-sampled text by the timestamp rules."""
    if spec.sot not in prompt:
        return len(prompt)
    i = list(prompt).index(spec.sot) + 1
    while i < len(prompt) and spec.sot <= prompt[i] <= spec.no_timestamps:
        i += 1
    return i


def apply_processors(logits: torch.Tensor, gen: List[int], spec: VocabSpec, opts: GenOptions,
                     use_timestamps: bool, prefix: Sequence[int] = (), rule_margin: Optional[List[float]] = None) -> torch.Tensor:
    """One row: raw logits [V] f32 -> log-probabilities [V] f32 after all masks.  ``gen`` are the generated tokens,
    ``prefix`` the prompt tokens after the sot sequence (history of the timestamp rules = prefix + gen; blank
    suppression is keyed to the first generated step).  ``rule_margin``, when given, receives |log P(any timestamp) -
    max log P(text token)| if the timestamp-probability rule was evaluated: that rule is a decision of its own, and a
    near-tie in it changes the next token however large the sampling / arg-max margin is."""
    x = logits.clone()
    if len(opts.suppress_tokens):
        x[torch.as_tensor(list(opts.suppress_tokens), dtype=torch.long)] = NEG_INF
    if opts.suppress_blank and len(gen) == 0:
        x[spec.blank] = NEG_INF
        x[spec.eot] = NEG_INF
    gen = list(prefix) + list(gen)
    first = len(gen) == 0
    tb = spec.timestamp_begin
    if use_timestamps:
        x[spec.no_timestamps] = NEG_INF
        if first:
            x[:tb] = NEG_INF
            x[tb + opts.max_initial_timestamp_index + 1:] = NEG_INF
        else:
            last_ts = gen[-1] >= tb
            penult_ts = len(gen) < 2 or gen[-2] >= tb
            if last_ts:
                if penult_ts:
                    x[tb:] = NEG_INF
                else:
                    x[:spec.eot] = NEG_INF
            stamps = [t for t in gen if t >= tb]
            if stamps:
                cutoff = stamps[-1] if (last_ts and not penult_ts) else stamps[-1] + 1
                x[tb:cutoff] = NEG_INF
            if not bool(torch.isfinite(x).any()):
                return x          # every token masked: no candidate (not the NaN row of a log-softmax over nothing)
            logp = torch.log_softmax(x, dim=-1)
            ts_lp = torch.logsumexp(logp[tb:], dim=-1)
            if rule_margin is not None:
                rule_margin.append(abs(float(ts_lp - logp[:tb].max())))
            if ts_lp > logp[:tb].max():
                x[:tb] = NEG_INF
    if not bool(torch.isfinite(x).any()):
        return x
    return torch.log_softmax(x, dim=-1)


def topk_stable(values: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """top-k, descending, ties toward the lower index."""
    v = values.numpy()
    k = min(k, v.shape[0])
    part = np.argpartition(-v, k - 1)[:k] if k < v.shape[0] else np.arange(v.shape[0])
    # include anything tied with the k-th value so the tie rule is exact
    kth = v[part].min()
    cand = np.nonzero(v >= kth)[0]
    order = np.lexsort((cand, -v[cand]))[:k]
    idx = cand[order]
    return torch.from_numpy(v[idx].copy()), torch.from_numpy(idx.astype(np.int64))


@dataclass
class Hypothesis:
    tokens: List[int]
    cum_logprob: float
    score: float


@dataclass
class StreamResult:
    sequences_ids: List[List[int]] = field(default_factory=list)
    scores: List[float] = field(default_factory=list)
    no_speech_prob: float = 0.0
    steps: int = 0
    # per-step decision margins (top1 - top2 of the ranked candidates, or the timestamp-rule margin when that is smaller)
    # for divergence-aware comparison
    margins: List[float] = field(default_factory=list)
    # beam search only, when GenOptions.trace: per step {"alive": [token tuples], "cand": [(beam, token, total)]}
    # with 2K+2 ranked candidates -- lets a test name the near-tie behind a pruning difference
    trace: List[dict] = field(default_factory=list)
    # sampling only: per hypothesis row, the margin of the Gumbel-perturbed arg-max at every step
    row_margins: dict = field(default_factory=dict)
    row_tokens: List[List[int]] = field(default_factory=list)
    # beam search: hypotheses finished before the best num_hypotheses were kept, and why the search ended
    # ("max_cand", "last_step" or "no_alive")
    n_hypotheses: int = 0
    stop: str = ""


def _normalise(cum: float, n_tokens: int, length_penalty: float) -> float:
    if length_penalty == 0:
        return cum
    return cum / (max(n_tokens, 1) ** length_penalty)


def max_candidates(beam_size: int, patience: float) -> int:
    """Hypotheses that end a beam search: round(K * patience) half away from zero, at least 1."""
    return max(1, int(math.floor(abs(beam_size * patience) + 0.5)))


def search_stream(step_fn, prompt: List[int], spec: VocabSpec, opts: GenOptions, stream_index: int = 0) -> StreamResult:
    """Run the search for one stream.

    ``step_fn(tokens [R,T] int64, parents or None) -> logits [R,T,V]`` advances the
    decoder: ``parents`` (LongTensor [R]) re-gathers cache rows first (None keeps them)."""
    res = StreamResult()
    sb = sample_begin(prompt, spec)
    prefix = list(prompt[sb:])
    use_ts = not (sb > 0 and prompt[sb - 1] == spec.no_timestamps)
    sot_index = prompt.index(spec.sot) if spec.sot in prompt else None
    n_new = max_new_tokens(len(prompt), opts.max_length)

    sampling = opts.beam_size == 1 and opts.sampling_topk != 1 and opts.sampling_temperature > 0
    n_rows0 = opts.num_hypotheses if opts.beam_size == 1 else 1

    # prefill: everything before the last prompt token, on one row
    p = torch.tensor([prompt], dtype=torch.long)
    logits_last = None
    if len(prompt) > 1:
        pre = step_fn(p[:, :-1], None)
        if sot_index is not None and sot_index < len(prompt) - 1:
            res.no_speech_prob = float(torch.softmax(pre[0, sot_index], -1)[spec.no_speech])
    if n_new == 0:
        res.sequences_ids, res.scores = [[]], [0.0]
        return res

    if opts.beam_size == 1:
        rows = n_rows0
        gens: List[List[int]] = [[] for _ in range(rows)]
        cums = [0.0] * rows
        done = [False] * rows
        cur = torch.full((rows, 1), prompt[-1], dtype=torch.long)
        parents = torch.zeros(rows, dtype=torch.long) if rows > 1 else None
        for step in range(n_new):
            logits = step_fn(cur, parents)[:, -1]
            parents = None
            if step == 0 and sot_index == len(prompt) - 1:
                res.no_speech_prob = float(torch.softmax(logits[0], -1)[spec.no_speech])
            nxt = []
            for r in range(rows):
                if done[r]:
                    nxt.append(spec.eot)
                    continue
                rule = []
                logp = apply_processors(logits[r], gens[r], spec, opts, use_ts, prefix, rule)
                rule_m = min(rule) if rule else float("inf")
                if not bool(torch.isfinite(logp).any()):   # every token masked: the row ends with no token
                    done[r] = True
                    nxt.append(spec.eot)
                    continue
                if sampling:
                    z = logp / opts.sampling_temperature
                    if opts.sampling_topk > 0:
                        kth = torch.topk(z, opts.sampling_topk).values[-1]
                        z = torch.where(z >= kth, z, torch.full_like(z, NEG_INF))
                    z = z + torch.from_numpy(gumbel_noise(opts.seed, stream_index * 64 + r, step, spec.vocab))
                    zv, zi = topk_stable(z, 2)
                    tok = int(zi[0])
                    res.row_margins.setdefault(r, []).append(min(float(zv[0] - zv[1]), rule_m))
                    if r == 0:
                        res.margins.append(min(float(zv[0] - zv[1]), rule_m))
                else:
                    vals, idx = topk_stable(logp, 2)
                    tok = int(idx[0])
                    if r == 0:
                        res.margins.append(min(float(vals[0] - vals[1]), rule_m))
                cums[r] += float(logp[tok])
                if tok == spec.eot:
                    done[r] = True
                else:
                    gens[r].append(tok)
                    if step + 1 == n_new:
                        done[r] = True
                nxt.append(tok)
            res.steps = step + 1
            if all(done):
                break
            cur = torch.tensor(nxt, dtype=torch.long)[:, None]
        hyps = [Hypothesis(g, c, _normalise(c, len(g), opts.length_penalty)) for g, c in zip(gens, cums)]
        res.row_tokens = [list(g) for g in gens]
    else:
        K = opts.beam_size
        max_cand = max_candidates(K, opts.patience)
        alive_tokens: List[List[int]] = [[]]
        alive_cum = [0.0]
        hyps: List[Hypothesis] = []
        cur = torch.tensor([[prompt[-1]]], dtype=torch.long)
        parents = None
        for step in range(n_new):
            logits = step_fn(cur, parents)[:, -1]
            if step == 0 and sot_index == len(prompt) - 1:
                res.no_speech_prob = float(torch.softmax(logits[0], -1)[spec.no_speech])
            n_alive = len(alive_tokens)
            total = torch.stack([apply_processors(logits[r], alive_tokens[r], spec, opts, use_ts, prefix) + alive_cum[r]
                                 for r in range(n_alive)]).reshape(-1)
            if opts.trace:
                tv, ti = topk_stable(total, 2 * K + 2)
                res.trace.append({"alive": [tuple(t) for t in alive_tokens], "alive_cum": [float(c) for c in alive_cum],
                                  "cand": [(int(i) // spec.vocab, int(i) % spec.vocab, float(v)) for v, i in zip(tv, ti)]})
            vals, idx = topk_stable(total, 2 * K)
            n_c = idx.shape[0]
            if n_c >= 2:
                res.margins.append(float(vals[0] - vals[1]))
            cand = [(int(i) // spec.vocab, int(i) % spec.vocab, float(v)) for v, i in zip(vals, idx)]
            last_step = step + 1 == n_new
            new_tokens, new_cum, new_parent = [], [], []
            secondary = K
            ev = {"closed_eot": 0, "closed_last": 0, "refilled": 0, "ran_out": 0}
            for k in range(min(K, n_c)):
                beam, tok, sc = cand[k]
                if not math.isfinite(sc):
                    continue
                if tok == spec.eot or last_step:
                    toks = alive_tokens[beam] + ([] if tok == spec.eot else [tok])
                    hyps.append(Hypothesis(toks, sc, _normalise(sc, len(toks), opts.length_penalty)))
                    ev["closed_last" if last_step else "closed_eot"] += 1
                    if last_step:
                        continue
                    repl = None
                    while secondary < n_c:
                        b2, t2, s2 = cand[secondary]
                        secondary += 1
                        if t2 != spec.eot and math.isfinite(s2):
                            repl = (b2, t2, s2)
                            break
                    if repl is None:
                        ev["ran_out"] += 1
                        continue
                    ev["refilled"] += 1
                    beam, tok, sc = repl
                new_tokens.append(alive_tokens[beam] + [tok])
                new_cum.append(sc)
                new_parent.append(beam)
            res.steps = step + 1
            if opts.trace:
                res.trace[-1].update(ev, n_alive=len(new_tokens))
            res.n_hypotheses = len(hyps)
            if len(hyps) >= max_cand or last_step or not new_tokens:
                res.stop = "max_cand" if len(hyps) >= max_cand else ("last_step" if last_step else "no_alive")
                break
            alive_tokens, alive_cum = new_tokens, new_cum
            parents = torch.tensor(new_parent, dtype=torch.long)
            cur = torch.tensor([t[-1] for t in alive_tokens], dtype=torch.long)[:, None]

    order = sorted(range(len(hyps)), key=lambda i: (-hyps[i].score, i))
    keep = order[:max(1, opts.num_hypotheses)]
    res.sequences_ids = [hyps[i].tokens for i in keep]
    res.scores = [hyps[i].score for i in keep]
    return res
