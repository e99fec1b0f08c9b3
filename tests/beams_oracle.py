"""The CPU oracle engine with a decode session that also takes a per-stream beam width
(``DecodeSession.admit(rules=[{"beam_size": k, ...}])``, ``k <= rows_per_stream``): a stream's hypotheses are what
``generate`` returns for it alone under the session's options updated by its rules, width included.  Host-side tests
of a file decoded at another beam than the live streams run on it."""
from __future__ import annotations

from tests.rules_oracle import RulesOracleSession, RulesOracleWhisper


class BeamsOracleSession(RulesOracleSession):
    def __init__(self, engine, capacity, **kw):
        super().__init__(engine, capacity, **kw)
        # as DecodeSession: the session's beam, or its num_hypotheses greedy rows
        self.rows_per_stream = self.beam_size if self.beam_size > 1 else int(self.kw.get("num_hypotheses", 1))

    def admit(self, features, prompts, max_lengths, indices=None, rules=None, sampling=None) -> list:
        if sampling is not None and any(s is not None for s in sampling):
            raise NotImplementedError("the oracle session does not sample per stream")
        if rules is None:
            return super().admit(features, prompts, max_lengths, indices)
        for r in rules:
            k = int((r or {}).get("beam_size", 0))
            if not 0 <= k <= self.rows_per_stream:
                raise RuntimeError(f"beam_size {k} outside 1 .. {self.rows_per_stream} rows per stream")
        free = self.free_indices()
        if indices is None:
            if len(prompts) > len(free):
                raise RuntimeError(f"admit: {len(prompts)} streams for {len(free)} free indices")
            indices = free[:len(prompts)]
        for i, f, p, ml, r in zip(indices, features, prompts, max_lengths, rules):
            kw = dict(self.kw, **(r or {}))
            if not kw.get("beam_size"):
                kw["beam_size"] = self.beam_size              # 0: the session's width
            self.rule_admissions += r is not None
            res = self.engine.generate(f, [list(p)], max_length=int(ml), **kw)[0]
            self._res[i] = res
            self._left[i] = max(1, int(res.steps) - (len(p) - 1))
        return list(indices)


class BeamsOracleWhisper(RulesOracleWhisper):
    def open_decode_session(self, capacity=None, **generate_kwargs) -> BeamsOracleSession:
        return BeamsOracleSession(self, capacity or self.max_streams, **generate_kwargs)
