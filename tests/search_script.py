"""numpy restatement of the scripted logits of ``wl_test_search`` (csrc/search.cu, ``scripted_logits_kernel``) and an
``oracle.search`` step function that serves them.

A row's logits are a pure function of the tokens it has consumed -- ``prompt[:fed + 1]`` while the prompt is fed, then
the whole prompt followed by the row's generated tokens -- and of the search options (which tokens a rule masks at this
step).  Every value is an exact float32 number, so the device and this module give bit-identical logits:

* ``h = lowbias32(FNV-1a(seed, tokens))`` over 32-bit token words;
* ``base(t) = ((lowbias32(h ^ t * 0x9E3779B1) >> 20) - 2048) / 256``, a 1/256 grid over [-8, 8);
* a timestamp bias ``TS_BIAS[h & 3]``, an EOT bias ``EOT_BIAS[(h >> 2) & 3]`` and, right after ``<|startoftranscript|>``,
  +10 on ``<|nospeech|>`` when bit 4 of h is set;
* a pattern (the script's, or ``(h >> 5) % 6`` when it is -1), with ``g = lowbias32(h ^ 0x5BD1E995)``:
  1 all of one ``search_rows`` thread's strided set (``((t % 4096) >> 2) == g % 1024``) at ``8 + floor(4 base) / 4``;
  2 one float4 group (``t >> 2 == g % (V >> 2)``) the same way; 3 the last 8 tokens of the vocabulary the same way;
  4 the whole row on a grid of 1/4 (exact ties everywhere); 5 one or two text tokens at 48 (the log-softmax is then
  exact, so ties between rows are exact too);
* on a row that searches, ``60 + base / 8`` on every token a rule must mask at this step (suppress list,
  ``<|notimestamps|>``, blank / EOT at the first generated step, the first step's ``max_initial_timestamp_index`` bound,
  timestamps below the last one): a missed mask changes the arg-max.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np
import torch

from oracle.search import GenOptions, VocabSpec, sample_begin

TS_BIAS = (-8.0, -5.0, -2.0, 2.0)
EOT_BIAS = (-8.0, -2.0, 2.0, 8.0)
M32 = 0xFFFFFFFF


def hash_u32(x):
    """lowbias32 on a uint32 array (or a Python int)."""
    scalar = not isinstance(x, np.ndarray)
    x = np.asarray(x, dtype=np.uint64) & np.uint64(M32)
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x7FEB352D)) & np.uint64(M32)
    x ^= x >> np.uint64(15)
    x = (x * np.uint64(0x846CA68B)) & np.uint64(M32)
    x ^= x >> np.uint64(16)
    return int(x) if scalar else x.astype(np.uint32)


def seq_hash(seed: int, tokens: Sequence[int]) -> int:
    h = ((2166136261 ^ (seed & M32)) * 16777619) & M32
    for t in tokens:
        h = ((h ^ (int(t) & M32)) * 16777619) & M32
    return hash_u32(h)


@dataclass
class RowRules:
    """The masking rules of one searching row at one step (what search_rows_kernel derives from the state)."""
    first: bool
    suppress_blank: bool
    last_is_ts: bool
    penult_is_ts: bool
    last_ts: int          # -1: no timestamp in the history
    cutoff: int


class Script:
    """The scripted logits of one stream: ``prompt``, the generate options and the script ``(seed, pattern)``."""

    def __init__(self, spec: VocabSpec, prompt: Sequence[int], opts: GenOptions, seed: int, pattern: int):
        self.spec, self.prompt, self.opts = spec, list(prompt), opts
        self.seed, self.pattern = int(seed), int(pattern)
        self.P = len(self.prompt)
        sb = sample_begin(self.prompt, spec)
        self.prefix = self.prompt[sb:]
        self.use_ts = not (sb > 0 and self.prompt[sb - 1] == spec.no_timestamps)
        V = spec.vocab
        self.t = np.arange(V, dtype=np.uint64)
        self.tmul = ((self.t * np.uint64(0x9E3779B1)) & np.uint64(M32))
        self.suppress = np.zeros(V, dtype=bool)
        sup = [t for t in opts.suppress_tokens if 0 <= t < V]
        self.suppress[sup] = True

    def rules(self, gen: Sequence[int]) -> RowRules:
        tb = self.spec.timestamp_begin
        hist = self.prefix + list(gen)
        n = len(hist)
        stamps = [t for t in hist if t >= tb]
        last_is_ts = n > 0 and hist[-1] >= tb
        penult_is_ts = n < 2 or hist[-2] >= tb
        lts = stamps[-1] if stamps else -1
        cutoff = lts if (last_is_ts and not penult_is_ts) else lts + 1
        return RowRules(n == 0, bool(self.opts.suppress_blank) and len(gen) == 0, last_is_ts, penult_is_ts, lts, cutoff)

    def masked(self, r: RowRules) -> np.ndarray:
        """Tokens the adversarial boost covers (the rules a, b, d, the suppress list and blank suppression)."""
        sp, V = self.spec, self.spec.vocab
        tb = sp.timestamp_begin
        m = self.suppress.copy()
        if r.suppress_blank:
            m[sp.blank] = m[sp.eot] = True
        if self.use_ts:
            m[sp.no_timestamps] = True
            if r.first:
                m[tb + self.opts.max_initial_timestamp_index + 1:] = True
            elif r.last_ts >= 0:
                m[tb:max(tb, r.cutoff)] = True
        return m[:V]

    def logits(self, seq: Sequence[int]) -> np.ndarray:
        """float32 [V] logits after the row consumed ``seq``."""
        sp, V = self.spec, self.spec.vocab
        h = seq_hash(self.seed, seq)
        g = hash_u32(h ^ 0x5BD1E995)
        raw = hash_u32((self.tmul ^ np.uint64(h)).astype(np.uint64))
        base = ((raw >> np.uint32(20)).astype(np.int64) - 2048).astype(np.float64) / 256.0
        x = base.copy()
        tb = sp.timestamp_begin
        x[tb:] += TS_BIAS[h & 3]
        x[sp.eot] += EOT_BIAS[(h >> 2) & 3]
        if seq[-1] == sp.sot and (h >> 4) & 1:
            x[sp.no_speech] += 10.0
        pattern = self.pattern if self.pattern >= 0 else (h >> 5) % 6
        t = np.arange(V)
        quarter = 8.0 + np.floor(base * 4.0) * 0.25
        if pattern == 1:
            sel = ((t % 4096) >> 2) == g % 1024
            x[sel] = quarter[sel]
        elif pattern == 2:
            sel = (t >> 2) == g % (V >> 2)
            x[sel] = quarter[sel]
        elif pattern == 3:
            x[V - 8:] = quarter[V - 8:]
        elif pattern == 4:
            x = np.floor(x * 4.0) * 0.25
        elif pattern == 5:
            d = g % sp.eot
            x[d] = 48.0
            if (h >> 7) & 1:
                x[(d + 1 + ((g >> 24) & 63)) % sp.eot] = 48.0
        if len(seq) >= self.P:      # the row searches: boost what a rule must mask
            m = self.masked(self.rules(seq[self.P:]))
            x[m] = 60.0 + base[m] / 8.0
        return x.astype(np.float32)

    def pattern_of(self, seq: Sequence[int]) -> int:
        h = seq_hash(self.seed, seq)
        return self.pattern if self.pattern >= 0 else (h >> 5) % 6


class ScriptStep:
    """``oracle.search.search_stream`` step function serving a Script: keeps every row's consumed tokens (parents
    regather them, like the decoder's cache rows) and records, per searching row and step, what the rules did."""

    def __init__(self, script: Script):
        self.script = script
        self.rows: List[List[int]] = [[]]
        self.events: List[dict] = []

    def __call__(self, tokens: torch.Tensor, parents: Optional[torch.Tensor]) -> torch.Tensor:
        if parents is not None:
            self.rows = [list(self.rows[int(p)]) for p in parents]
        if tokens.shape[0] != len(self.rows):
            self.rows = [list(self.rows[0]) for _ in range(tokens.shape[0])]
        out = []
        for r, row in enumerate(self.rows):
            steps = []
            for tok in tokens[r].tolist():
                row.append(int(tok))
                steps.append(self.script.logits(row))
                if len(row) >= self.script.P:
                    self.events.append(self.row_events(row, steps[-1]))
            out.append(np.stack(steps))
        return torch.from_numpy(np.stack(out))

    def row_events(self, seq: Sequence[int], logits: np.ndarray) -> dict:
        """What the rules do to this row's logits: which branches apply, the rule-e decision and its margin."""
        s = self.script
        sp, tb = s.spec, s.spec.timestamp_begin
        r = s.rules(seq[s.P:])
        masked = s.masked(r)
        x = np.where(masked, -np.inf, logits.astype(np.float64))
        ev = {"pattern": s.pattern_of(seq), "first": r.first and s.use_ts, "rule_c": None, "rule_d": False,
              "rule_e": None, "rule_e_margin": np.inf}
        if s.use_ts and not r.first:
            if r.last_is_ts:
                ev["rule_c"] = "no_ts" if r.penult_is_ts else "no_text"
                if r.penult_is_ts:
                    x[tb:] = -np.inf
                else:
                    x[:sp.eot] = -np.inf
            ev["rule_d"] = r.last_ts >= 0 and r.cutoff > tb
            if np.isfinite(x).any():
                mx = x.max()
                lse = mx + np.log(np.exp(x - mx).sum())
                ts = x[tb:]
                ts_lse = -np.inf if not np.isfinite(ts).any() else ts.max() + np.log(np.exp(ts - ts.max()).sum())
                text_max = x[:tb].max()
                ev["rule_e"] = bool(ts_lse > text_max)
                if np.isfinite(ts_lse) and np.isfinite(text_max):
                    ev["rule_e_margin"] = abs((ts_lse - lse) - (text_max - lse))
                if ev["rule_e"]:
                    x[:tb] = -np.inf
        # exact ties at the top of the masked row: between tokens of one selection thread's strided set or not
        fin = np.isfinite(x)
        if fin.sum() >= 2:
            top = np.nonzero(x == x.max())[0]
            if len(top) >= 2:
                ev["tie"] = True
                owners = (top % 4096) >> 2
                ev["tie_same_thread"] = bool(len(set(owners.tolist())) < len(top))
        return ev
