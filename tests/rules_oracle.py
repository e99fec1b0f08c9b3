"""The CPU oracle engine with a decode session that takes per-stream logits rules (``DecodeSession.admit(rules=...)``):
a stream's hypotheses are what ``generate`` returns for it alone under the session's options updated by its rules.
Host-side tests of the batched pipeline through the scheduler run on it."""
from __future__ import annotations

from oracle.engine import OracleDecodeSession, OracleWhisper


class RulesOracleSession(OracleDecodeSession):
    supports_rules = True

    def __init__(self, engine, capacity, **kw):
        super().__init__(engine, capacity, **kw)
        self.rule_admissions = 0          # streams admitted with rules of their own

    @property
    def beam_size(self) -> int:
        return int(self.kw.get("beam_size", 5))

    def admit(self, features, prompts, max_lengths, indices=None, rules=None) -> list:
        if rules is None:
            return super().admit(features, prompts, max_lengths, indices)
        free = self.free_indices()
        if indices is None:
            if len(prompts) > len(free):
                raise RuntimeError(f"admit: {len(prompts)} streams for {len(free)} free indices")
            indices = free[:len(prompts)]
        for i, f, p, ml, r in zip(indices, features, prompts, max_lengths, rules):
            if r is not None and int(r.get("beam_size", self.beam_size)) != self.beam_size:
                raise RuntimeError("beam_size differs from the session's")
            kw = dict(self.kw, **(r or {}))
            self.rule_admissions += r is not None
            res = self.engine.generate(f, [list(p)], max_length=int(ml), **kw)[0]
            self._res[i] = res
            self._left[i] = max(1, int(res.steps) - (len(p) - 1))
        return list(indices)


class RulesOracleWhisper(OracleWhisper):
    max_streams = 8

    def open_decode_session(self, capacity=None, **generate_kwargs) -> RulesOracleSession:
        return RulesOracleSession(self, capacity or self.max_streams, **generate_kwargs)
