"""Device translator (csrc/mt.cu, csrc/mt_engine.cu) against the float64 oracle (tests/mt_oracle.py), on an H100."""
from __future__ import annotations

import ctypes as C
import dataclasses

import numpy as np
import pytest

from tests import mt_oracle as O
from whisperlive_b200 import translation as T

pytestmark = pytest.mark.gpu

MICRO = T.MtConfig(d_model=128, n_heads=2, enc_layers=2, dec_layers=1, ffn=512, vocab=1000, max_positions=1024)
LENGTHS = [1, 2, 63, 64, 65, 127, 128, 129, 1022]
NAN16 = np.uint16(0x7E00)


@pytest.fixture(scope="module")
def lib():
    from whisperlive_b200 import _lib
    return _lib.load()


def _ctx(lib, cfg=MICRO, capacity=4, beams=5, tokens=256):
    from whisperlive_b200 import _lib
    mc = _lib.WlMtConfig(abi_version=_lib.ABI_VERSION, d_model=cfg.d_model, n_heads=cfg.n_heads, enc_layers=cfg.enc_layers,
                         dec_layers=cfg.dec_layers, ffn=cfg.ffn, vocab=cfg.vocab, max_positions=cfg.max_positions,
                         pad_id=cfg.pad_id, embed_scale=cfg.embed_scale, max_src_tokens=tokens)
    ctx = C.c_void_p()
    assert lib.wl_mt_init(C.byref(mc), 0, capacity, beams, C.byref(ctx)) == 0, lib.wl_mt_last_error(None)
    return ctx


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def _segments(lengths):
    """The measured segments packed with a 3-token fence segment after each."""
    out = []
    for n in lengths:
        out.append(("seg", n))
        out.append(("fence", 3))
    return out


def _qkv(rng, lengths, H, fence_k=60.0, fence_v=1e4):
    d = 64 * H
    parts, offs, kinds = [], [0], []
    for kind, n in _segments(lengths):
        if kind == "seg":
            x = rng.standard_normal((n, 3 * d)).astype(np.float16)
            # the maximum of every query planted at the first and the last key of the segment
            x[0, d:2 * d] *= 3
            x[-1, d:2 * d] *= 3
        else:
            x = np.empty((n, 3 * d), np.float16)
            x[:, :d] = 1.0
            x[:, d:2 * d] = fence_k
            x[:, 2 * d:] = fence_v
        parts.append(x)
        offs.append(offs[-1] + n)
        kinds.append(kind)
    return np.concatenate(parts), np.asarray(offs, np.int32), kinds


def _attn64(q, k, v, H):
    return O._attn(q.astype(np.float64), k.astype(np.float64), v.astype(np.float64), H)


def test_encoder_attention_ragged_against_float64(lib):
    H = 16
    d = 64 * H
    ctx = _ctx(lib)
    try:
        rng = np.random.default_rng(0)
        qkv, off, kinds = _qkv(rng, LENGTHS, H)
        out = np.full((off[-1], d), NAN16, np.uint16)
        assert lib.wl_test_mt_attn(ctx, _p(qkv.view(np.uint16), C.c_uint16), _p(off, C.c_int32), len(kinds), H,
                                   _p(out, C.c_uint16)) == 0, lib.wl_mt_last_error(ctx)
        got = out.view(np.float16).astype(np.float64)
        for b, kind in enumerate(kinds):
            if kind != "seg":
                continue
            x = qkv[off[b]:off[b + 1]]
            ref = _attn64(x[:, :d], x[:, d:2 * d], x[:, 2 * d:], H)
            g = got[off[b]:off[b + 1]]
            assert np.isfinite(g).all(), b
            err = np.abs(g - ref).max()
            assert err < 4e-3 * max(1.0, np.abs(ref).max()), (off[b + 1] - off[b], err)
            # alone: bit-identical
            one = np.full((off[b + 1] - off[b], d), NAN16, np.uint16)
            o1 = np.asarray([0, off[b + 1] - off[b]], np.int32)
            xa = np.ascontiguousarray(x)
            assert lib.wl_test_mt_attn(ctx, _p(xa.view(np.uint16), C.c_uint16), _p(o1, C.c_int32), 1, H, _p(one, C.c_uint16)) == 0
            assert np.array_equal(one, out[off[b]:off[b + 1]]), off[b + 1] - off[b]
    finally:
        lib.wl_mt_destroy(ctx)


def test_cross_attention_ragged_against_float64(lib):
    H, K = 16, 5
    d = 64 * H
    L = 3
    ldkv = 2 * d * L
    ctx = _ctx(lib)
    try:
        rng = np.random.default_rng(1)
        kinds, offs, parts = [], [0], []
        for kind, n in _segments(LENGTHS):
            x = rng.standard_normal((n, ldkv)).astype(np.float16)
            if kind == "fence":
                x[:] = 1e4
            else:
                x[0] *= 3
                x[-1] *= 3
            parts.append(x)
            offs.append(offs[-1] + n)
            kinds.append(kind)
        kv = np.ascontiguousarray(np.concatenate(parts))
        off = np.asarray(offs, np.int32)
        B = len(kinds)
        q = rng.standard_normal((B * K, d)).astype(np.float32)
        for layer in range(L):
            koff, voff = 2 * d * layer, 2 * d * layer + d
            out = np.full((B * K, d), NAN16, np.uint16)
            assert lib.wl_test_mt_cross_attn(ctx, _p(q, C.c_float), _p(kv.view(np.uint16), C.c_uint16), ldkv, koff, voff,
                                             _p(off, C.c_int32), B, K, H, _p(out, C.c_uint16)) == 0, lib.wl_mt_last_error(ctx)
            got = out.view(np.float16).astype(np.float64)
            for b, kind in enumerate(kinds):
                if kind != "seg":
                    continue
                x = kv[off[b]:off[b + 1]]
                ref = _attn64(q[b * K:(b + 1) * K], x[:, koff:koff + d], x[:, voff:voff + d], H)
                err = np.abs(got[b * K:(b + 1) * K] - ref).max()
                assert err < 4e-3 * max(1.0, np.abs(ref).max()), (off[b + 1] - off[b], layer, err)
    finally:
        lib.wl_mt_destroy(ctx)


SEARCH_CASES = [
    dict(num_beams=5, early_stopping=False, length_penalty=1.0, max_length=24),
    dict(num_beams=5, early_stopping=True, length_penalty=1.0, max_length=24),
    dict(num_beams=5, early_stopping="never", length_penalty=1.0, max_length=24),
    dict(num_beams=4, early_stopping=False, length_penalty=0.0, max_length=24),
    dict(num_beams=4, early_stopping="never", length_penalty=2.0, max_length=24),
    dict(num_beams=8, early_stopping=False, length_penalty=1.0, max_length=12),
    dict(num_beams=5, early_stopping=False, length_penalty=1.0, max_length=6),
    dict(num_beams=5, early_stopping=False, length_penalty=1.0, max_length=10, forced_bos_token_id=7, forced_eos_token_id=2),
    dict(num_beams=1, max_length=24),
    dict(num_beams=1, max_length=9, forced_bos_token_id=7, forced_eos_token_id=2),
]


def _script(rng, steps, R, V, eos, eos_rate):
    lg = (2.0 * rng.standard_normal((steps, R, V))).astype(np.float32)
    # EOS near the top in a share of the rows (often at ranks >= K inside the top 2K)
    boost = rng.random((steps, R)) < eos_rate
    lg[..., eos] = np.where(boost, lg.max(-1) + rng.uniform(-2.0, 3.0, (steps, R)), lg[..., eos])
    return lg


@pytest.mark.parametrize("case", range(len(SEARCH_CASES)))
def test_beam_step_against_oracle_on_scripted_logits(lib, case):
    spec = SEARCH_CASES[case]
    gen = dataclasses.replace(T.GenSettings(), **spec)
    from whisperlive_b200 import _lib
    V, B, K = 1000, 6, gen.num_beams
    ctx = _ctx(lib, capacity=B, beams=8)
    try:
        rng = np.random.default_rng(100 + case)
        steps = gen.max_length - 1
        lg = _script(rng, steps, B * K, V, gen.eos_token_id, eos_rate=0.3 + 0.1 * (case % 3))
        opts = _lib.WlMtOpts(num_beams=K, max_length=gen.max_length, length_penalty=gen.length_penalty,
                             early_stopping=gen.early_stopping_code, decoder_start=gen.decoder_start_token_id, eos=gen.eos_token_id,
                             forced_bos=-1 if gen.forced_bos_token_id is None else gen.forced_bos_token_id,
                             forced_eos=-1 if gen.forced_eos_token_id is None else gen.forced_eos_token_id, use_cuda_graph=0)
        ids = np.full((B, gen.max_length), -1, np.int32)
        n = np.zeros(B, np.int32)
        sc = np.zeros(B, np.float32)
        st = np.zeros(B, np.int32)
        lgc = np.ascontiguousarray(lg)
        assert lib.wl_test_mt_search(ctx, _p(lgc, C.c_float), V, B, C.byref(opts), _p(ids, C.c_int32), _p(n, C.c_int32),
                                     _p(sc, C.c_float), _p(st, C.c_int32)) == 0, lib.wl_mt_last_error(ctx)
        seen_steps = set()
        for b in range(B):
            def fn(seqs, b=b):
                t = len(seqs[0]) - 1
                return lg[t, b * K:b * K + len(seqs)]
            ref = O.beam_search(fn, gen)
            assert n[b] == len(ref.tokens) and ids[b, :n[b]].tolist() == ref.tokens, (b, ids[b, :n[b]].tolist(), ref.tokens)
            assert st[b] == ref.steps, (b, st[b], ref.steps)
            assert abs(float(sc[b]) - float(ref.score)) <= 1e-4 * max(1.0, abs(float(ref.score))), (b, sc[b], ref.score)
            seen_steps.add(int(st[b]))
        if K > 1 and gen.max_length > 10 and gen.early_stopping != "never":
            assert len(seen_steps) > 1, "segments should finish at different steps"
    finally:
        lib.wl_mt_destroy(ctx)


def _micro_translator(capacity=4, beams=5, **kw):
    ck = T.random_checkpoint(MICRO, seed=3)
    gen = T.GenSettings(num_beams=beams, max_length=kw.pop("max_length", 24))
    return T.DeviceTranslator(MICRO, gen, ck, capacity=capacity, max_src_tokens=kw.pop("max_src_tokens", 512), **kw), ck, gen


def _logits_against_oracle(tr, orc, srcs, prefixes):
    """Teacher-forced device logits against the float64 oracle's for every segment; returns the largest log-probability
    error seen (what a sequence comparison may attribute to fp16)."""
    got = tr.decoder_logits(srcs, prefixes)
    assert np.isfinite(got).all()
    worst = 0.0
    for b, (s, p) in enumerate(zip(srcs, prefixes)):
        ref = orc.decoder_logits(orc.encode(s), p)
        g = got[b].astype(np.float64)
        scale = ref.std()
        err = np.abs(g - ref).max()
        rms = np.sqrt(np.mean((g - ref) ** 2)) / scale
        print(f"segment {b}: max |logit err| {err:.3e} ({err / scale:.3%} of the logit std), rms {rms:.3%}")
        assert err < 0.02 * scale and rms < 0.005, (b, err, scale, rms)   # measured on H100: <= 0.35 % and 0.07 %
        worst = max(worst, float(np.abs(O.log_softmax(g) - O.log_softmax(ref)).max()))
    return worst


def _near_tie(ref, got, tol):
    """got departs from the oracle's best hypothesis only after a step whose selection margin is within tol (twice the
    measured log-probability error): a choice fp16 rounding may flip."""
    i = next((k for k, (a, b) in enumerate(zip(got, ref.tokens)) if a != b), min(len(got), len(ref.tokens)))
    return min(ref.margins[:i + 1] or [0.0]) < tol


def _prefixes(rng, B, P, vocab):
    return [[2] + rng.integers(3, vocab - 200, P - 1).tolist() for _ in range(B)]


@pytest.mark.parametrize("B", [1, 8, 32])
def test_micro_teacher_forced_logits(B):
    tr, ck, _ = _micro_translator(capacity=32, max_src_tokens=32 * 48)
    try:
        orc = O.OracleM2M100(ck, MICRO)
        rng = np.random.default_rng(20 + B)
        srcs = [[900 + int(rng.integers(0, 100))] + rng.integers(3, 900, int(rng.integers(1, 40))).tolist() + [2] for _ in range(B)]
        print("worst log-prob error", _logits_against_oracle(tr, orc, srcs, _prefixes(rng, B, 8, MICRO.vocab)))
    finally:
        tr.close()


@pytest.mark.parametrize("beams", [1, 5])
def test_micro_translate_against_oracle(beams):
    tr, ck, gen = _micro_translator(beams=beams)
    try:
        orc = O.OracleM2M100(ck, MICRO)
        rng = np.random.default_rng(7)
        srcs = [[900 + int(rng.integers(0, 100))] + rng.integers(3, 900, n).tolist() + [2] for n in (1, 5, 14, 40)]
        tol = 2 * _logits_against_oracle(tr, orc, srcs, _prefixes(rng, 4, 8, MICRO.vocab))
        ids, scores = tr.translate_ids(srcs)
        for s, g, score in zip(srcs, ids, scores):
            ref = orc.generate(s, gen)
            if g != ref.tokens:
                assert _near_tie(ref, g, tol), (g, ref.tokens, tol)
            else:
                assert abs(score - float(ref.score)) < 2 * tol + 1e-3, (score, ref.score)
        # a segment's result does not depend on the segments beside it
        for s, g in zip(srcs, ids):
            alone, _ = tr.translate_ids([s])
            assert alone[0] == g
    finally:
        tr.close()


def test_micro_graph_and_host_loop_agree():
    tr, _, _ = _micro_translator()
    tr2, _, _ = _micro_translator(use_cuda_graph=False)
    try:
        srcs = [[905, 10, 11, 12, 2], [950, 400, 2], [901] + list(range(100, 160)) + [2]]
        assert tr.translate_ids(srcs) == tr2.translate_ids(srcs)
    finally:
        tr.close()
        tr2.close()


def test_device_bytes_match_footprint():
    tr, _, _ = _micro_translator()
    try:
        got, est = tr.device_bytes(), T.mt_footprint(MICRO, 4, 5, 512)
        assert est <= got <= 1.10 * est, (got, est)
    finally:
        tr.close()


@pytest.mark.parametrize("B", [1, 8, 32])
def test_small100_shape_against_oracle(B):
    """Teacher-forced logits of every segment at 1 / 8 / 32 segments, then beam-5 sequences of the first segments."""
    cfg = T.MtConfig(**T.SMALL100_SHAPE)
    ck = T.random_checkpoint(cfg, seed=11)
    gen = T.GenSettings(num_beams=5, max_length=10)
    tr = T.DeviceTranslator(cfg, gen, ck, capacity=32, max_src_tokens=32 * 16)
    try:
        orc = O.OracleM2M100(ck, cfg)
        rng = np.random.default_rng(12 + B)
        srcs = [[128020] + rng.integers(3, 128000, int(rng.integers(4, 14))).tolist() + [2] for _ in range(B)]
        tol = 2 * _logits_against_oracle(tr, orc, srcs, _prefixes(rng, B, 4, cfg.vocab))
        print("near-tie tolerance", tol)
        ids, _ = tr.translate_ids(srcs)
        for s, g in list(zip(srcs, ids))[:2]:
            ref = orc.generate(s, gen)
            if g != ref.tokens:
                assert _near_tie(ref, g, tol), (g, ref.tokens, tol)
    finally:
        tr.close()


def test_micro_snapshot_on_the_reference_source_ids():
    """The micro snapshot of tests/golden/ through wl_mt_translate on the source ids the reference's tokenizer produced:
    the generated ids equal Hugging Face's (recorded by the reference's model), or depart after a measured near tie."""
    import json
    import os
    golden = os.path.join(os.path.dirname(__file__), "golden")
    with open(os.path.join(golden, "translate_reference.json")) as f:
        ref = json.load(f)
    with open(os.path.join(golden, "small100_micro", "config.json")) as f:
        cfg = T.config_from_json(json.load(f))
    ck = T.random_checkpoint(cfg, ref["seed"])
    orc = O.OracleM2M100(ck, cfg)
    checked = 0
    for name, case in ref["translate"].items():
        gen = T.GenSettings(**{**dict(early_stopping=False, length_penalty=1.0), **case["settings"]})
        rows = [r for r in case["rows"] if r["src"]]
        tr = T.DeviceTranslator(cfg, gen, ck, capacity=len(rows), max_src_tokens=64 * len(rows))
        try:
            srcs = [r["src"] for r in rows]
            tol = 2 * _logits_against_oracle(tr, orc, srcs[:2], [[2, 5, 6, 7]] * 2)
            ids, _ = tr.translate_ids(srcs)
            for r, g in zip(rows, ids):
                if g != r["generated"]:
                    assert _near_tie(orc.generate(r["src"], gen), g, tol), (name, r["text"], g, r["generated"])
                checked += 1
        finally:
            tr.close()
    assert checked >= 40
