"""Float64 restatement of M2M100 (SMaLL-100) and of Hugging Face's beam search, the yardstick of the device translator.

The network follows transformers 5.5.0 ``models/m2m_100`` (pre-LN layers, biased projections, scores scaled by
head_dim^-0.5, ReLU FFN, final LayerNorms, tied head).  ``beam_search`` restates ``GenerationMixin._beam_search`` step by
step with the bookkeeping in float32 as Hugging Face keeps it (-1e9 penalties, ``_check_early_stop_heuristic``), on the
log-probabilities a ``logits_fn`` gives; ties go to the lower flattened (beam, token) index.  ``num_beams == 1`` is
greedy search."""
from __future__ import annotations

import math

import numpy as np

from whisperlive_b200.translation import MtConfig, position_table


def _ln(x, w, b):
    m = x.mean(-1, keepdims=True)
    v = ((x - m) ** 2).mean(-1, keepdims=True)
    return (x - m) / np.sqrt(v + 1e-5) * w + b


def _attn(q, k, v, H):
    n, d = q.shape
    hd = d // H
    q = q.reshape(n, H, hd).transpose(1, 0, 2)
    k = k.reshape(-1, H, hd).transpose(1, 0, 2)
    v = v.reshape(-1, H, hd).transpose(1, 0, 2)
    s = q @ k.transpose(0, 2, 1) * hd ** -0.5
    s = s - s.max(-1, keepdims=True)
    p = np.exp(s)
    p /= p.sum(-1, keepdims=True)
    return (p @ v).transpose(1, 0, 2).reshape(n, d)


class OracleM2M100:
    def __init__(self, ck: dict, cfg: MtConfig):
        self.cfg = cfg
        self.w = {k: np.asarray(v, dtype=np.float64) for k, v in ck.items()}
        self.pos = position_table(cfg).astype(np.float64)

    def _lin(self, x, name):
        return x @ self.w[name + ".weight"].T + self.w[name + ".bias"]

    def _embed(self, ids, positions):
        return self.w["model.shared.weight"][ids] * self.cfg.embed_scale + self.pos[positions]

    def encode(self, src: list) -> np.ndarray:
        c, pad = self.cfg, self.cfg.pad_id
        ids = np.asarray(src)
        positions = np.where(ids == pad, pad, pad + np.cumsum(ids != pad))   # create_position_ids_from_input_ids
        x = self._embed(ids, positions)
        for l in range(c.enc_layers):
            p = f"model.encoder.layers.{l}."
            h = _ln(x, self.w[p + "self_attn_layer_norm.weight"], self.w[p + "self_attn_layer_norm.bias"])
            a = _attn(self._lin(h, p + "self_attn.q_proj"), self._lin(h, p + "self_attn.k_proj"), self._lin(h, p + "self_attn.v_proj"), c.n_heads)
            x = x + self._lin(a, p + "self_attn.out_proj")
            h = _ln(x, self.w[p + "final_layer_norm.weight"], self.w[p + "final_layer_norm.bias"])
            x = x + self._lin(np.maximum(self._lin(h, p + "fc1"), 0.0), p + "fc2")
        return _ln(x, self.w["model.encoder.layer_norm.weight"], self.w["model.encoder.layer_norm.bias"])

    def decoder_logits(self, enc: np.ndarray, tokens: list, last_only: bool = False) -> np.ndarray:
        """Teacher-forced logits [len(tokens)][vocab] of the decoder over ``tokens`` (decoder start first); the last
        position's only with ``last_only``."""
        c, pad = self.cfg, self.cfg.pad_id
        ids = np.asarray(tokens)
        positions = np.where(ids == pad, pad, pad + 1 + np.arange(len(ids)))   # past length + padding_idx + 1
        x = self._embed(ids, positions)
        n = len(ids)
        causal = np.triu(np.full((n, n), -np.inf), 1)
        for l in range(c.dec_layers):
            p = f"model.decoder.layers.{l}."
            h = _ln(x, self.w[p + "self_attn_layer_norm.weight"], self.w[p + "self_attn_layer_norm.bias"])
            q, k, v = (self._lin(h, p + f"self_attn.{t}_proj") for t in "qkv")
            H, hd = c.n_heads, c.d_model // c.n_heads
            qh, kh, vh = (t.reshape(n, H, hd).transpose(1, 0, 2) for t in (q, k, v))
            s = qh @ kh.transpose(0, 2, 1) * hd ** -0.5 + causal
            s = s - s.max(-1, keepdims=True)
            pr = np.exp(s)
            pr /= pr.sum(-1, keepdims=True)
            a = (pr @ vh).transpose(1, 0, 2).reshape(n, c.d_model)
            x = x + self._lin(a, p + "self_attn.out_proj")
            h = _ln(x, self.w[p + "encoder_attn_layer_norm.weight"], self.w[p + "encoder_attn_layer_norm.bias"])
            a = _attn(self._lin(h, p + "encoder_attn.q_proj"), self._lin(enc, p + "encoder_attn.k_proj"),
                      self._lin(enc, p + "encoder_attn.v_proj"), c.n_heads)
            x = x + self._lin(a, p + "encoder_attn.out_proj")
            h = _ln(x, self.w[p + "final_layer_norm.weight"], self.w[p + "final_layer_norm.bias"])
            x = x + self._lin(np.maximum(self._lin(h, p + "fc1"), 0.0), p + "fc2")
        x = _ln(x, self.w["model.decoder.layer_norm.weight"], self.w["model.decoder.layer_norm.bias"])
        if last_only:
            x = x[-1:]
        return x @ self.w["model.shared.weight"].T

    def generate(self, src: list, gen):
        enc = self.encode(src)
        return beam_search(lambda seqs: np.stack([self.decoder_logits(enc, s, last_only=True)[0] for s in seqs]), gen)


def log_softmax(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, dtype=np.float64)
    m = x.max(-1, keepdims=True)
    return x - m - np.log(np.exp(x - m).sum(-1, keepdims=True))


def _forced(lp: np.ndarray, cur_len: int, gen) -> np.ndarray:
    f = None
    if cur_len == 1 and gen.forced_bos_token_id is not None:
        f = gen.forced_bos_token_id
    if cur_len == gen.max_length - 1 and gen.forced_eos_token_id is not None:
        f = gen.forced_eos_token_id
    if f is None:
        return lp
    out = np.full_like(lp, -np.inf)
    out[..., f] = 0.0
    return out


def _topk(v: np.ndarray, k: int) -> np.ndarray:
    """Indices of the k largest values, ties to the lower index."""
    return np.argsort(-v, kind="stable")[:k]


class SearchResult:
    def __init__(self, tokens, score, steps, margins):
        self.tokens, self.score, self.steps, self.margins = tokens, score, steps, margins


def beam_search(logits_fn, gen) -> SearchResult:
    """One segment.  logits_fn(list of running sequences) -> logits [n][V] (numpy) of the next token of each.
    Returns the best hypothesis without the decoder start token, its score, the running length it stopped at, and the
    selection margins of every step (the gap between the last kept and the first dropped candidate)."""
    f32 = np.float32
    K, eos, L, lp = gen.num_beams, gen.eos_token_id, gen.max_length, gen.length_penalty
    es = gen.early_stopping
    start = gen.decoder_start_token_id
    margins = []
    if K == 1:
        seq, cum = [start], 0.0
        while True:
            cur_len = len(seq)
            logits = np.asarray(logits_fn([seq])[0], dtype=np.float64)
            lpv = _forced(log_softmax(logits), cur_len, gen)
            order = np.argsort(-lpv, kind="stable")
            t = int(order[0])
            margins.append(float(lpv[order[0]] - lpv[order[1]]))
            seq.append(t)
            cum += float(lpv[t])
            if t == eos or cur_len + 1 >= L:
                return SearchResult(seq[1:], f32(cum), cur_len, margins)
    run = [[start] for _ in range(K)]
    run_scores = np.full(K, -1e9, dtype=f32)
    run_scores[0] = 0.0
    fin = [[start] for _ in range(K)]
    fin_scores = np.full(K, -1e9, dtype=f32)
    fin_flag = np.zeros(K, dtype=bool)
    unsat = True
    cur_len = 1
    while True:
        logits = np.asarray(logits_fn(run), dtype=np.float64)
        V = logits.shape[1]
        lpv = _forced(log_softmax(logits), cur_len, gen).astype(f32)
        acc = (lpv + run_scores[:, None]).reshape(-1)
        idx = _topk(acc, 2 * K)
        srt = np.sort(acc)[::-1]
        margins.append(float(srt[2 * K - 1] - srt[2 * K]) if np.isfinite(srt[2 * K]) else math.inf)
        top_v = acc[idx]
        top_seq = [run[i // V] + [int(i % V)] for i in idx]
        hits = np.array([s[-1] == eos or cur_len + 1 >= L for s in top_seq])
        rv = (top_v + hits.astype(f32) * f32(-1.0e9)).astype(f32)
        nxt = _topk(rv, K)
        new_run = [top_seq[i] for i in nxt]
        new_run_scores = rv[nxt]
        did = hits & (np.arange(2 * K) < K)
        v = (top_v / f32((cur_len + 1 - 1) ** lp)).astype(f32)
        full = bool(fin_flag.all()) and es is True
        v = (v + f32(full) * f32(-1.0e9)).astype(f32)
        v = (v + f32(not unsat) * f32(-1.0e9)).astype(f32)
        v = (v + (~did).astype(f32) * f32(-1.0e9)).astype(f32)
        m_scores = np.concatenate([fin_scores, v])
        m_seqs = fin + top_seq
        m_flag = np.concatenate([fin_flag, did])
        keep = _topk(m_scores, K)
        fin = [m_seqs[i] for i in keep]
        fin_scores = m_scores[keep]
        fin_flag = m_flag[keep]
        run, run_scores = new_run, new_run_scores
        cur_len += 1
        bhl = (L - 1) if (es == "never" and lp > 0.0) else (cur_len - 1)
        best = f32(run_scores[0] / f32(bhl ** lp))
        worst = np.where(fin_flag, fin_scores.min(), f32(-1.0e9))
        unsat = unsat and bool(np.any(best > worst))
        at_max = cur_len >= L
        if (not unsat) or (es is True and fin_flag.all()) or at_max:
            return SearchResult(fin[0][1:], fin_scores[0], cur_len - 1, margins)
