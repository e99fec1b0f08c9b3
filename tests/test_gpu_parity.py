"""GPU parity tests (run on an H100: ``pytest -m gpu``).  Everything goes through the C ABI
(ctypes -> libwlb200.so); the oracle is only the checker.

Tolerances: the engine stores weights/activations entering a GEMM in fp16 and accumulates in fp32
(the reference's CUDA default is float16: backend/faster_whisper_backend.py:88-91); the oracle is fp32
with the same fp16-representable weights.  Integer results (token ids, alignment pairs) are
compared with a divergence-aware rule: a mismatch is tolerated only where the oracle's own decision
margin at that step is below the fp16 logit tolerance.
"""
import os

import numpy as np
import pytest
import torch

from oracle import mel as omel
from oracle.engine import OracleWhisper
from oracle.mel import OracleFeatureExtractor
from whisperlive_b200 import synth
from whisperlive_b200.config import dims_for
from whisperlive_b200.tokenizer import build_synthetic_tokenizer
from whisperlive_b200.weights import random_init

pytestmark = pytest.mark.gpu

LOGIT_TOL = 0.12       # fp16 logit tolerance (logit std is ~3)
MARGIN_TOL = 0.20      # a greedy token decision closer than this may legitimately flip
SCORE_TOL = 0.05       # length-normalised hypothesis score: beam-search near-ties within this are interchangeable
ALIGN_MAX_SHIFT = 6    # frames (0.12 s) a DTW jump may move under an fp16-sized perturbation of the attention weights
BEAM_TIE_TOL = 0.25    # cumulative log-prob gap between two beam candidates that an fp16-sized logit perturbation,
                       # accumulated over the decoded prefix (2 x LOGIT_TOL), can flip

_ENGINES = {}


def engine(name, seed=0, **kw):
    key = (name, seed, tuple(sorted(kw.items())))
    if key not in _ENGINES:
        from whisperlive_b200.engine import B200Whisper
        dims = dims_for(name)
        w = random_init(dims, seed=seed)
        _ENGINES[key] = (B200Whisper(dims, w, max_streams=kw.get("max_streams", 4), max_beam=kw.get("max_beam", 5)),
                         OracleWhisper(w, dims))
    return _ENGINES[key]


def feats_for(dims, seconds, seed):
    return omel.pad_or_trim(omel.log_mel(synth.speech_like(seconds, seed=seed), dims.n_mels)[:, :-1])


# --------------------------------------------------------------------------------------- GEMM (wgmma)
GEMM_CASES = [
    # (Z, M, N, K, transposed, gelu, bias)
    (1, 128, 128, 64, False, False, False),
    (1, 128, 128, 256, False, False, True),
    (1, 256, 384, 128, False, True, True),
    (1, 1500, 384, 384, False, False, True),
    (2, 300, 64, 1536, False, False, False),
    (3, 1500, 1500, 64, False, False, False),
    (1, 384, 5, 384, True, False, True),       # swap-AB decode shape, N tile 16
    (1, 1152, 20, 384, True, True, True),      # N tile 32
    (1, 51864, 10, 128, True, False, False),   # vocabulary projection, M tail
    (1, 200, 40, 72, False, False, False),     # K tail (zero fill) + N tile 64
    (1, 640, 160, 1280, True, False, True),    # N tile 128 (x2)
]


@pytest.mark.parametrize("case", GEMM_CASES)
def test_gemm_tcgen05(case):
    eng, _ = engine("micro.en")
    Z, M, N, K, tr, gelu, has_bias = case
    rng = np.random.default_rng(hash(case) % (2 ** 31))
    a = rng.standard_normal((Z, M, K)).astype(np.float16)
    b = rng.standard_normal((Z, N, K)).astype(np.float16)
    bias = rng.standard_normal(M if tr else N).astype(np.float32) if has_bias else None
    ref = np.einsum("zmk,znk->zmn", a.astype(np.float32), b.astype(np.float32))
    if has_bias:
        ref = ref + (bias[None, :, None] if tr else bias[None, None, :])
    if gelu:
        ref = torch.nn.functional.gelu(torch.from_numpy(ref)).numpy()
    if tr:
        ref = ref.transpose(0, 2, 1)
    simt = eng.test_gemm(a, b, bias, transposed_store=tr, gelu=gelu, use_simt=True)
    np.testing.assert_allclose(simt, ref, atol=2e-3 * np.sqrt(K), rtol=1e-3)
    tc = eng.test_gemm(a, b, bias, transposed_store=tr, gelu=gelu, use_simt=False)
    err = np.abs(tc - ref).max()
    print(f"gemm {case}: max err tc {err:.3e}  simt {np.abs(simt - ref).max():.3e}")
    np.testing.assert_allclose(tc, ref, atol=2e-3 * np.sqrt(K), rtol=1e-3)


WGEMM_CASES = [
    # (R, n_out, K, mode)   mode 0 bias, 1 residual in place, 2 gelu -> fp16, 3 split-K partials (K > 1280)
    (16, 1280, 1280, 0), (5, 384, 384, 0), (1, 768, 768, 0), (16, 3840, 1280, 0), (20, 1280, 1280, 1), (32, 128, 128, 1),
    (16, 5120, 1280, 2), (16, 1280, 5120, 3), (12, 768, 3072, 3), (3, 128, 512, 1), (16, 51200, 1280, 0), (9, 1536, 384, 2),
]


@pytest.mark.parametrize("case", WGEMM_CASES)
def test_wgemm_small_batch(case):
    """The small-batch decode GEMM (csrc/wgemm.cu: mma.sync, bulk-copied weight slices, fused epilogues) against fp32
    numpy on the same fp16 inputs, all four epilogues, ragged row counts, every K the Whisper sizes produce."""
    eng, _ = engine("micro.en")
    R, n_out, K, mode = case
    rng = np.random.default_rng(abs(hash(case)) % (2 ** 31))
    w = (rng.standard_normal((n_out, K)) / np.sqrt(K)).astype(np.float16)
    x = rng.standard_normal((R, K)).astype(np.float16)
    bias = rng.standard_normal(n_out).astype(np.float32) if mode != 3 else None
    resid = rng.standard_normal((R, n_out)).astype(np.float32) if mode == 1 else None
    ref = x.astype(np.float32) @ w.astype(np.float32).T
    if bias is not None:
        ref = ref + bias[None, :]
    if mode == 1:
        ref = ref + resid
    if mode == 2:
        ref = torch.nn.functional.gelu(torch.from_numpy(ref)).numpy()
    got = eng.test_wgemm(w, x, bias, mode=mode, resid=resid)
    err = np.abs(got - ref).max()
    print(f"wgemm {case}: max err {err:.3e}")
    np.testing.assert_allclose(got, ref, atol=2e-3 if mode != 2 else 4e-3, rtol=2e-3)


# --------------------------------------------------------------------------------------- K1 mel
@pytest.mark.parametrize("n_mels_model", ["micro.en", "large-v3-mel"])
def test_mel_matches_oracle(n_mels_model):
    if n_mels_model == "large-v3-mel":
        from whisperlive_b200.config import WhisperDims
        from whisperlive_b200.engine import B200Whisper
        dims = WhisperDims("mel128", 128, 2, 1, 1, 128, 51866)
        eng = B200Whisper(dims, random_init(dims, seed=5), max_streams=4, max_beam=1)
    else:
        eng, _ = engine("micro.en")
        dims = eng.dims
    waves = [synth.speech_like(1.0, seed=11), synth.speech_like(7.31, seed=12), synth.white_noise(30.0, seed=13),
             synth.silence(2.0), synth.speech_like(17001 / 16000, seed=14), synth.speech_like(0.05, seed=15)]
    outs = eng.mel(waves)
    for w, o in zip(waves, outs):
        ref = omel.log_mel(w, dims.n_mels)
        assert o.shape == ref.shape and o.dtype == np.float32
        err = np.abs(o - ref).max()
        print(f"mel n={len(w)} n_mels={dims.n_mels}: max err {err:.2e}")
        assert err < 2e-4
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "mel_reference.npz"))
    for k in g.files:
        if k.startswith("wav__") or not k.endswith(f"__{dims.n_mels}"):
            continue
        o = eng.mel([g["wav__" + k.split("__")[0]]])[0]
        assert np.abs(o - g[k]).max() < 2e-4, k


# --------------------------------------------------------------------------------------- K2-K7 encoder
@pytest.mark.parametrize("name", ["micro.en", "tiny"])
def test_encoder_matches_oracle(name):
    eng, orc = engine(name, seed=1)
    dims = eng.dims
    feats = np.stack([feats_for(dims, 6.0, 1), feats_for(dims, 29.0, 2), feats_for(dims, 1.2, 3)])
    enc = eng.encode(feats)
    got = np.asarray(enc)
    ref = orc.encode(feats).enc.numpy()
    err = np.abs(got - ref)
    print(f"encoder {name}: max err {err.max():.4f} mean err {err.mean():.5f} ref mean abs {np.abs(ref).mean():.3f}")
    assert err.max() < 0.08 and err.mean() < 0.006
    # batch invariance: a stream encoded alone gives the same result
    alone = np.asarray(eng.encode(feats[1:2]))
    assert np.abs(alone[0] - got[1]).max() < 1e-3


@pytest.mark.parametrize("name,secs,seeds", [("micro.en", (6.0, 6.0), (1, 2)), ("tiny", (6.0, 6.0, 6.0, 14.0), (1, 2, 3, 7))])
def test_split_flash_kernel_on_the_decode_tests_inputs(name, secs, seeds):
    """The default encoder attention checked per query tile on the weights (seed 0) and inputs of the decode-level tests:
    the other encoder checks use seed-1 weights, and an attention error confined to some tiles shows up first as a decode
    divergence."""
    eng, orc = engine(name, seed=0)
    dims = eng.dims
    feats = np.stack([feats_for(dims, s, sd) for s, sd in zip(secs, seeds)])
    got = np.asarray(eng.encode(feats))
    ref = orc.encode(feats).enc.numpy()
    for b in range(len(secs)):
        for t in range(12):
            sl = slice(t * 128, min(1500, (t + 1) * 128))
            e = float(np.abs(got[b, sl] - ref[b, sl]).max())
            assert e < 0.08, (name, "stream", b, "query tile", t, e)


FUSED_ATTN_CHECK = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from oracle import mel as omel
from oracle.engine import OracleWhisper
from whisperlive_b200 import synth
from whisperlive_b200.config import dims_for
from whisperlive_b200.engine import B200Whisper
from whisperlive_b200.weights import random_init
worst, launches = 0.0, 0
for name, seed, secs, seeds in [("micro.en", 0, (6.0, 6.0), (1, 2)), ("tiny", 0, (6.0, 6.0, 6.0, 14.0), (1, 2, 3, 7)),
                                ("tiny", 1, (6.0, 29.0, 1.2), (1, 2, 3))]:
    dims = dims_for(name)
    w = random_init(dims, seed=seed)
    eng, orc = B200Whisper(dims, w, max_streams=4, max_beam=1), OracleWhisper(w, dims)
    feats = np.stack([omel.pad_or_trim(omel.log_mel(synth.speech_like(s, seed=sd), dims.n_mels)[:, :-1]) for s, sd in zip(secs, seeds)])
    n0 = eng.kernel_launches()
    enc = eng.encode(feats)
    if not launches:
        launches = eng.kernel_launches() - n0   # of the first encode: tells the two paths apart
    got = np.asarray(enc)
    ref = orc.encode(feats).enc.numpy()
    assert np.abs(got - ref).mean() < 0.006, (name, seed)
    for b in range(len(secs)):
        for t in range(12):
            sl = slice(t * 128, min(1500, (t + 1) * 128))
            e = float(np.abs(got[b, sl] - ref[b, sl]).max())
            assert e < 0.08, (name, seed, "stream", b, "query tile", t, e)
            worst = max(worst, e)
print("launches", launches, "worst tile error", worst)
"""


def test_fused_flash_attention_kernel_per_query_tile():
    """Both encoder attention paths against the oracle per query tile, on the decode tests' seed-0 weights and inputs and
    on the encoder test's seed-1 ones: the fused wgmma flash-attention kernel (the default) and the unfused scores GEMM +
    softmax + P V GEMM path (WLB200_FUSED_ATTN=0).  The switch is read once per process, hence one subprocess per path;
    that each took its own branch shows in the launch count of an encode (per layer the fused path launches one
    attention kernel, the unfused one a scores GEMM, a softmax kernel and a P V GEMM per attention sub-pass)."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    launches = {}
    for fused in ("1", "0"):
        out = subprocess.run([sys.executable, "-c", FUSED_ATTN_CHECK, root], capture_output=True, text=True, timeout=600,
                             env=dict(os.environ, WLB200_FUSED_ATTN=fused))
        assert out.returncode == 0, out.stderr[-3000:]
        print(f"WLB200_FUSED_ATTN={fused}:", out.stdout.strip())
        launches[fused] = int(out.stdout.split("launches")[1].split()[0])
    assert launches["1"] < launches["0"], launches


def test_encoder_golden_hf():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "model_hf.npz"))
    for name in ("micro.en", "tiny"):
        eng, _ = engine(name, seed=int(g[name + "__init_seed"][0]))
        dims = eng.dims
        wav = synth.speech_like(7.3, seed=int(g[name + "__wav_seed"][0]))
        feats = omel.pad_or_trim(omel.log_mel(wav, dims.n_mels)[:, :-1])
        enc = eng.encode(feats[None])
        got = np.asarray(enc)[0, ::25]
        assert np.abs(got - g[name + "__enc_sub"]).max() < 0.08
        logits = eng.decode_logits(enc, [g[name + "__tokens"][0].tolist()])[0]
        assert np.abs(logits[:, :512] - g[name + "__logits_head"]).max() < LOGIT_TOL
        assert np.abs(logits[:, -1700:] - g[name + "__logits_tail"]).max() < LOGIT_TOL


# --------------------------------------------------------------------------------------- K8-K12 decoder
@pytest.mark.parametrize("name", ["micro.en", "tiny"])
def test_teacher_forced_logits(name):
    eng, orc = engine(name, seed=2)
    dims = eng.dims
    feats = np.stack([feats_for(dims, 5.0, 4), feats_for(dims, 11.0, 5)])
    enc = eng.encode(feats)
    oenc = orc.encode(feats)
    rng = np.random.default_rng(3)
    toks = [[orc.spec.sot] + rng.integers(0, 50000, 17).tolist(), [orc.spec.sot] + rng.integers(0, 50000, 6).tolist()]
    got = eng.decode_logits(enc, toks)
    from oracle import model as om
    for b, t in enumerate(toks):
        xkv = [(k[b:b + 1], v[b:b + 1]) for k, v in oenc.xkv]
        with torch.no_grad():
            ref = om.decoder_forward(orc.w, torch.tensor([t]), xkv, om.DecoderState(dims.dec_layers), dims.n_heads,
                                     dims.dec_layers)[0].numpy()
        err = np.abs(got[b] - ref)
        print(f"logits {name} stream {b}: max err {err.max():.4f} mean {err.mean():.5f}")
        assert err.max() < LOGIT_TOL


def _oracle_rescore(orc, oenc, b, prompt, seq, kw):
    """Teacher-force the engine's hypothesis through the ORACLE (same logits processors) and return its
    length-normalised score as the oracle would have scored it."""
    from oracle.search import GenOptions, apply_processors, max_new_tokens, sample_begin
    spec = orc.spec
    opts = GenOptions(beam_size=kw.get("beam_size", 5), suppress_blank=kw.get("suppress_blank", True),
                      suppress_tokens=[t for t in kw.get("suppress_tokens", ()) if t >= 0],
                      max_initial_timestamp_index=kw.get("max_initial_timestamp_index", 50))
    sb = sample_begin(prompt, spec)
    prefix = list(prompt[sb:])
    use_ts = not (sb > 0 and prompt[sb - 1] == spec.no_timestamps)
    step = orc._stream_step_fn(oenc, b)
    if len(prompt) > 1:
        step(torch.tensor([prompt[:-1]]), None)
    n_new = max_new_tokens(len(prompt), kw.get("max_length", 448))
    cum, gen, cur = 0.0, [], prompt[-1]
    targets = list(seq) + ([spec.eot] if len(seq) < n_new else [])
    for tok in targets:
        logp = apply_processors(step(torch.tensor([[cur]]), None)[0, -1], gen, spec, opts, use_ts, prefix)
        cum += float(logp[tok])
        gen.append(tok)
        cur = tok
    lp = kw.get("length_penalty", 1)
    return cum / (max(len(seq), 1) ** lp) if lp else cum


def _oracle_cums(orc, oenc, b, prompt, seq, kw):
    """Cumulative oracle log-probability after each token of ``seq`` (teacher-forced through the oracle's network and
    logits processors)."""
    from oracle.search import GenOptions, apply_processors, sample_begin
    spec = orc.spec
    opts = GenOptions(beam_size=kw.get("beam_size", 5), suppress_blank=kw.get("suppress_blank", True),
                      suppress_tokens=[t for t in kw.get("suppress_tokens", ()) if t >= 0],
                      max_initial_timestamp_index=kw.get("max_initial_timestamp_index", 50))
    sb = sample_begin(prompt, spec)
    prefix = list(prompt[sb:])
    use_ts = not (sb > 0 and prompt[sb - 1] == spec.no_timestamps)
    step = orc._stream_step_fn(oenc, b)
    if len(prompt) > 1:
        step(torch.tensor([prompt[:-1]]), None)
    cum, gen, cur, out = 0.0, [], prompt[-1], []
    for tok in seq:
        logp = apply_processors(step(torch.tensor([[cur]]), None)[0, -1], gen, spec, opts, use_ts, prefix)
        cum += float(logp[tok])
        out.append(cum)
        gen.append(tok)
        cur = tok
    return out


def _beam_tie_tol(j):
    """Perturbation of a cumulative beam score after j tokens that fp16-sized logit errors can cause: the base tolerance
    plus 0.005 per token (4 % of the per-logit tolerance LOGIT_TOL; the rescoring assert in _compare_generation bounds the
    same drift on the engine's own path)."""
    return BEAM_TIE_TOL + 0.005 * j


def _boundary_tie(trace, beam, mine, j, eot):
    """First expansion step k < j at which the oracle let the prefix beam[:k+1] into its beam set by less than
    _beam_tie_tol(k + 1) over the best candidate it rejected (an EOT candidate finishes a hypothesis instead of competing
    for a beam, so it is not a rejection), or None.  Under an fp16-sized perturbation that candidate can take the
    place of beam[:k+1], and then nothing descending from beam[:k+1] is in the engine's beam set.  Only the steps after
    ``beam`` has parted from the engine's prefix ``mine`` count: a prefix the two share is held by the engine."""
    shared = next((q for q, (x, y) in enumerate(zip(beam, mine)) if x != y), min(len(beam), len(mine)))
    for k in range(shared, j):
        tr, nxt = trace[k], trace[k + 1]
        kept = set(nxt["alive"])
        pre = tuple(beam[:k])
        if pre not in tr["alive"]:
            return None
        bi = tr["alive"].index(pre)
        mine = next((v for (cb, ct, v) in tr["cand"] if cb == bi and ct == beam[k]), None)
        rejected = next((v for (cb, ct, v) in tr["cand"] if ct != eot and tr["alive"][cb] + (ct,) not in kept), None)
        if mine is not None and rejected is not None and mine - rejected < _beam_tie_tol(k + 1):
            return k, mine - rejected
    return None


def _explain_beam_divergence(eng, enc, orc, oenc, b, prompt, kw, got, ref, what):
    """A beam-search hypothesis that differs from the oracle's must be EXPLAINED, not waved through.  Walk the engine's
    hypothesis through the ORACLE's beam trace: the first step j at which its prefix P is no longer among the oracle's
    live beams is where the oracle pruned it -- at least K oracle beams outrank P there -- while the engine, whose logits
    differ from the oracle's by an fp16-sized perturbation, kept it, so at most K - 1 beams outranked P in the engine.
    That is legitimate only if, IN THE ORACLE'S OWN NUMBERS, enough of the outranking beams can be absent from the
    engine's set or fall below P under such a perturbation: a beam A can if
      * A and P are within _beam_tie_tol(j) of each other at step j (a direct near-tie), or
      * A's lineage entered the oracle's beam set at an earlier step k by less than _beam_tie_tol(k + 1) over the best
        candidate the oracle rejected there (a near-tie at the beam boundary: the engine may have kept that candidate
        instead, and then holds no descendant of A).
    The assertion: at most K - 1 of the outranking beams are neither.  (The search LOGIC itself is pinned exactly by
    test_search_logic_exact_on_engine_logits; the numerics of the engine's own path by the rescoring assert in
    _compare_generation.)"""
    from oracle.search import GenOptions, search_stream
    sp = orc.spec
    K = kw["beam_size"]
    sup = [t for t in kw.get("suppress_tokens", ()) if t >= 0]
    opts = GenOptions(beam_size=K, num_hypotheses=kw.get("num_hypotheses", 1), suppress_tokens=sup,
                      max_length=kw.get("max_length", 448), length_penalty=kw.get("length_penalty", 1),
                      suppress_blank=kw.get("suppress_blank", True), patience=kw.get("patience", 1),
                      max_initial_timestamp_index=kw.get("max_initial_timestamp_index", 50), trace=True)
    on_oracle = search_stream(orc._stream_step_fn(oenc, b), list(prompt), sp, opts, stream_index=b)
    assert on_oracle.sequences_ids[0] == ref.sequences_ids[0]
    gs = list(got.sequences_ids[0])
    cums = _oracle_cums(orc, oenc, b, list(prompt), gs, kw)
    for j in range(1, min(len(gs), len(on_oracle.trace) - 1) + 1):
        tr = on_oracle.trace[j]                    # live beams BEFORE expansion step j = after j generated tokens
        if tuple(gs[:j]) in tr["alive"]:
            continue
        above = [(a, c) for a, c in zip(tr["alive"], tr["alive_cum"]) if c > cums[j - 1]]
        firm = []
        for a, c in above:
            gap = c - cums[j - 1]
            tie = _boundary_tie(on_oracle.trace, a, gs, j, sp.eot)
            print(f"{what} stream {b}: after token {j} the oracle keeps a beam {gap:.4f} above the engine's prefix "
                  f"(cum {cums[j - 1]:.4f}); boundary near-tie in its lineage: {tie}")
            if gap >= _beam_tie_tol(j) and tie is None:
                firm.append(gap)
        assert len(firm) <= K - 1, (what, b, j, "beams firmly above the engine's prefix", firm)
        return
    # never pruned: the hypotheses differ only in when / how they were finalised or ranked
    assert abs(got.scores[0] - ref.scores[0]) < SCORE_TOL, (what, b, got.scores, ref.scores)


def _compare_generation(got, ref, what, orc=None, oenc=None, prompts=None, kw=None, eng=None, enc=None):
    """Token-exact, or an explained near-tie.  Greedy / sampling: the oracle's own decision margin at the first
    differing token is below MARGIN_TOL.  Beam search: see _explain_beam_divergence.  In every case the engine's
    score of its own tokens must agree with the oracle's score of the SAME tokens (the numerics are right)."""
    n_div = 0
    for b, (g, r) in enumerate(zip(got, ref)):
        gs, rs = g.sequences_ids[0], r.sequences_ids[0]
        assert abs(g.no_speech_prob - r.no_speech_prob) < 0.02
        if gs == rs:
            assert abs(g.scores[0] - r.scores[0]) < 0.02, (what, b, g.scores, r.scores)
            continue
        i = next((k for k, (x, y) in enumerate(zip(gs, rs)) if x != y), min(len(gs), len(rs)))
        n_div += 1
        beam = (kw or {}).get("beam_size", 5)
        if orc is None or beam == 1:
            margins = r.margins[max(0, i - 1): i + 2]
            print(f"{what} stream {b}: diverges at token {i} (oracle margins there {margins})")
            assert margins and min(margins) < MARGIN_TOL, (what, b, i, margins)
            if orc is None:
                continue
        rescored = _oracle_rescore(orc, oenc, b, list(prompts[b]), gs, kw) if not kw.get("sampling_temperature") else None
        if rescored is not None:
            print(f"{what} stream {b}: diverges at token {i}/{len(rs)}: engine score {g.scores[0]:.4f}, oracle score of the "
                  f"engine's tokens {rescored:.4f}, oracle best {r.scores[0]:.4f}")
            assert abs(rescored - g.scores[0]) < 0.03, (what, b, "engine score disagrees with the oracle on its own tokens")
        if beam > 1:
            assert eng is not None, "beam-search divergences must be explained: pass eng / enc"
            _explain_beam_divergence(eng, enc, orc, oenc, b, list(prompts[b]), kw, g, r, what)
    return n_div


@pytest.mark.parametrize("name,beam", [("micro.en", 1), ("micro.en", 5), ("micro", 4), ("tiny", 5)])
def test_generate_matches_oracle(name, beam):
    eng, orc = engine(name, seed=0)
    dims = eng.dims
    sp = orc.spec
    feats = np.stack([feats_for(dims, 6.0, 1), feats_for(dims, 6.0, 2), feats_for(dims, 6.0, 3), feats_for(dims, 14.0, 7)])
    enc, oenc = eng.encode(feats), orc.encode(feats)
    base = [sp.sot] if not dims.multilingual else [sp.sot, sp.sot + 1, sp.sot + 1 + dims.num_languages + 1]
    prompts = [base, base, [sp.timestamp_begin - 3, 400, 1234, 11] + base, base]
    sup = [1, 2, 3, 50]
    kw = dict(beam_size=beam, suppress_tokens=sup, return_scores=True, return_no_speech_prob=True)
    got = eng.generate(enc, prompts, **kw)
    ref = orc.generate(oenc, prompts, **kw)
    n_div = _compare_generation(got, ref, f"{name} beam{beam}", orc, oenc, prompts, kw, eng=eng, enc=enc)
    lens = [len(g.sequences_ids[0]) for g in got]
    print(f"generate {name} beam {beam}: lengths {lens} steps {[g.steps for g in got]} divergences {n_div}")


@pytest.mark.parametrize("beam", [1, 5])
def test_generate_with_prefix_matches_oracle(beam):
    """ADVICE r1: a ``prefix`` (transcriber_faster_whisper.py:1505-1511) puts <|0.00|> + text tokens AFTER the sot
    sequence.  CT2 ends the prompt at the sot sequence, so those tokens seed the timestamp rules' history (the first
    generated token is not forced to be a timestamp) and ``without_timestamps`` stays honoured with a prefix."""
    eng, orc = engine("micro.en", seed=0)
    dims, sp = eng.dims, orc.spec
    feats = np.stack([feats_for(dims, 6.0, 1), feats_for(dims, 9.0, 2), feats_for(dims, 5.0, 3)])
    enc, oenc = eng.encode(feats), orc.encode(feats)
    prompts = [[sp.sot, sp.timestamp_begin, 300, 4000, 77],                 # prefix with timestamps
               [sp.sot, sp.no_timestamps, 300, 4000],                       # prefix, without_timestamps
               [sp.timestamp_begin - 3, 999, sp.sot, sp.timestamp_begin, 512]]   # previous text + prefix
    kw = dict(beam_size=beam, suppress_tokens=[1, 2, 3], max_length=80)
    got = eng.generate(enc, prompts, **kw)
    ref = orc.generate(oenc, prompts, **kw)
    _compare_generation(got, ref, f"prefix beam{beam}", orc, oenc, prompts, kw, eng=eng, enc=enc)
    # stream 1: <|notimestamps|> sits INSIDE the prompt (a prefix follows it), so the timestamp rules must be off:
    # its first generated token is not forced to be a timestamp (random weights: text tokens dominate)
    assert got[1].sequences_ids[0][0] == ref[1].sequences_ids[0][0]
    # stream 0: the history already holds <|0.00|> + text, so the first generated token is free to be text


@pytest.mark.parametrize("name,beam", [("micro.en", 5), ("tiny", 1), ("micro", 4)])
def test_batched_prefill_equals_token_by_token(name, beam):
    """K8: prompts of 1 .. 230 tokens (sot_prev + previous text + sot sequence, transcriber_faster_whisper.py:1480-1513)
    prefilled in one batched pass give the hypotheses, scores and no-speech probabilities of feeding the prompt one
    decode step per token -- and the oracle's, which prefills like CT2 does."""
    eng, orc = engine(name, seed=0)
    dims, sp = eng.dims, orc.spec
    feats = np.stack([feats_for(dims, 6.0, 1), feats_for(dims, 9.0, 2), feats_for(dims, 5.0, 3), feats_for(dims, 12.0, 4)])
    enc, oenc = eng.encode(feats), orc.encode(feats)
    base = [sp.sot] if not dims.multilingual else [sp.sot, sp.sot + 1, sp.sot + 1 + dims.num_languages + 1]
    rng = np.random.default_rng(17)
    prev = lambda n: [sp.timestamp_begin - 3] + rng.integers(256, 40000, n).tolist()     # <|startofprev|> + text
    prompts = [base, prev(222) + base, prev(37) + base, prev(8) + base + [sp.no_timestamps]]
    kw = dict(beam_size=beam, suppress_tokens=[1, 2, 3], max_length=448)
    a = eng.generate(enc, prompts, prefill=True, **kw)
    b = eng.generate(enc, prompts, prefill=False, **kw)
    for x, y, p in zip(a, b, prompts):
        assert abs(x.no_speech_prob - y.no_speech_prob) < 5e-3
        if x.sequences_ids[0] == y.sequences_ids[0]:
            assert abs(x.scores[0] - y.scores[0]) < 5e-3
        else:   # different GEMM kernels feed the two paths (wgmma row tiles vs the decode path): a near-tie may flip,
            print("prefill vs stepwise differ:", x.scores, y.scores)   # and BOTH must then be explained against the oracle below
    ref = orc.generate(oenc, prompts, **kw)
    _compare_generation(a, ref, f"prefill {name} beam{beam}", orc, oenc, prompts, kw, eng=eng, enc=enc)
    _compare_generation(b, ref, f"stepwise {name} beam{beam}", orc, oenc, prompts, kw, eng=eng, enc=enc)


class _EngineStep:
    """oracle.search step function backed by the ENGINE's logits (teacher-forced wl_decode_logits over the
    full prefix of every live row): lets the oracle's search run on exactly the numbers the engine sees."""

    def __init__(self, eng, enc_b, prompt):
        self.eng, self.enc_b = eng, enc_b
        self.rows = [[]]
        self.prompt = list(prompt)

    def __call__(self, tokens, parents):
        if parents is not None:
            self.rows = [list(self.rows[int(p)]) for p in parents]
        t_new = tokens.shape[1]
        if tokens.shape[0] != len(self.rows):
            self.rows = [list(self.rows[0]) for _ in range(tokens.shape[0])]
        for r, row in enumerate(self.rows):
            row.extend(int(t) for t in tokens[r])
        out = []
        cap = self.eng.max_streams
        for r0 in range(0, len(self.rows), cap):      # at most max_streams rows per teacher-forced call
            rows = self.rows[r0:r0 + cap]
            out.extend(self.eng.decode_logits(self.enc_b.select([0] * len(rows)), rows))
        return torch.from_numpy(np.stack([o[-t_new:] for o in out]))


@pytest.mark.parametrize("beam", [1, 5])
def test_search_logic_exact_on_engine_logits(beam):
    """Search-logic parity isolated from numerics: the oracle's search driven by the engine's own logits must
    reproduce the engine's device-side search token for token (beam bookkeeping, timestamp rules, suppression,
    hypothesis finalisation, length normalisation)."""
    from oracle.search import GenOptions, search_stream
    eng, orc = engine("micro.en", seed=0, max_streams=8)
    dims = eng.dims
    sp = orc.spec
    feats = np.stack([feats_for(dims, 6.0, 1), feats_for(dims, 6.0, 2), feats_for(dims, 14.0, 7)])
    enc = eng.encode(feats)
    prompts = [[sp.sot], [sp.timestamp_begin - 3, 400, 1234, 11, sp.sot], [sp.sot]]
    sup = [1, 2, 3, 50]
    got = eng.generate(enc, prompts, beam_size=beam, num_hypotheses=min(beam, 3), suppress_tokens=sup, max_length=120)
    n_exact = 0
    for b, prompt in enumerate(prompts):
        opts = GenOptions(beam_size=beam, num_hypotheses=min(beam, 3), suppress_tokens=sup, max_length=120)
        ref = search_stream(_EngineStep(eng, enc.select([b]), prompt), list(prompt), sp, opts, stream_index=b)
        same = ref.sequences_ids == got[b].sequences_ids
        n_exact += same
        print(f"beam {beam} stream {b}: exact={same} steps {got[b].steps} vs {ref.steps + len(prompt) - 1} "
              f"min margin {min(ref.margins):.2e}")
        if same:
            np.testing.assert_allclose(got[b].scores, ref.scores, atol=2e-3)
            assert abs(got[b].no_speech_prob - ref.no_speech_prob) < 1e-3
        else:
            # only an exact-tie-sized margin (split-K summation order) may explain a difference
            assert min(ref.margins) < 2e-3, (b, got[b].sequences_ids[0][:8], ref.sequences_ids[0][:8])
    assert n_exact >= 2


def test_generate_sampling_matches_oracle():
    eng, orc = engine("micro.en", seed=0)
    dims = eng.dims
    feats = np.stack([feats_for(dims, 6.0, 1), feats_for(dims, 6.0, 2)])
    enc, oenc = eng.encode(feats), orc.encode(feats)
    sp = orc.spec
    kw = dict(beam_size=1, num_hypotheses=3, sampling_topk=0, sampling_temperature=0.6, suppress_tokens=[1, 2], seed=7)
    got = eng.generate(enc, [[sp.sot]] * 2, **kw)
    ref = orc.generate(oenc, [[sp.sot]] * 2, **kw)
    same = sum(g.sequences_ids[0] == r.sequences_ids[0] for g, r in zip(got, ref))
    print("sampling: identical best hypotheses:", same, "of", len(got))
    for g in got:
        assert len(g.sequences_ids) == 3 and g.scores == sorted(g.scores, reverse=True)
    # engine and oracle share the counter-based Gumbel noise (hash of seed, stream, row, step, token): EVERY sampled
    # hypothesis is identical unless the perturbed arg-max of its row was itself a near-tie at the diverging step
    for b, (g, r) in enumerate(zip(got, ref)):
        rows = [tuple(t) for t in r.row_tokens]
        for gs in g.sequences_ids:
            if tuple(gs) in rows:
                continue
            # closest oracle row = longest common prefix; its margin where they part must be tiny
            def lcp(t):
                return next((k for k, (x, y) in enumerate(zip(gs, t)) if x != y), min(len(gs), len(t)))
            j = max(range(len(rows)), key=lambda q: lcp(rows[q]))
            i = lcp(rows[j])
            m = r.row_margins[j][max(0, i - 1): i + 2]
            print(f"sampling stream {b}: a hypothesis leaves oracle row {j} at token {i}, key margins there {m}")
            assert m and min(m) < MARGIN_TOL, (b, j, i, m)


def test_generate_options_and_errors():
    eng, orc = engine("micro.en", seed=0)
    dims = eng.dims
    sp = orc.spec
    feats = feats_for(dims, 4.0, 9)[None]
    enc, oenc = eng.encode(feats), orc.encode(feats)
    # without timestamps + max_length cap + several hypotheses
    prompt = [sp.sot, sp.no_timestamps]
    kw = dict(beam_size=3, num_hypotheses=2, max_length=40, suppress_tokens=[5], length_penalty=0.0)
    got = eng.generate(enc, [prompt], **kw)
    ref = orc.generate(oenc, [prompt], **kw)
    assert len(got[0].sequences_ids) == len(ref[0].sequences_ids) == 2
    _compare_generation(got, ref, "options", orc, oenc, [prompt], kw, eng=eng, enc=enc)
    assert all(len(s) <= 20 for s in got[0].sequences_ids)
    with pytest.raises(RuntimeError):
        eng.generate(enc, [[sp.sot] * 448], beam_size=1)            # no room under max_length
    with pytest.raises(RuntimeError):
        eng.generate(enc, [[dims.vocab + 5]], beam_size=1)          # token out of range
    with pytest.raises(ValueError):
        eng.generate(enc, [[sp.sot], [sp.sot]], beam_size=1)        # prompt/stream count mismatch
    with pytest.raises(RuntimeError):
        eng.generate(enc, [[sp.sot]], beam_size=7)                  # exceeds max_beam


def test_slot_pool_accounting():
    import gc
    eng, _ = engine("micro.en", seed=0)
    gc.collect()
    free0 = eng.free_slots()
    enc = eng.encode(feats_for(eng.dims, 2.0, 1)[None])
    assert eng.free_slots() == free0 - 1
    sub = enc.select([0])
    del enc
    assert eng.free_slots() == free0 - 1      # still referenced by the view
    del sub
    import gc
    gc.collect()
    assert eng.free_slots() == free0


# --------------------------------------------------------------------------------------- N1 weight loading from disk
@pytest.mark.parametrize("fmt", ["safetensors", "ct2"])
def test_load_checkpoint_directory_from_disk(tmp_path, fmt):
    """N1: a model DIRECTORY in either on-disk format the reference's users have -- HF ``model.safetensors``
    (openai/whisper-*) or the CTranslate2 ``model.bin`` download_model fetches (faster_whisper_backend.py:133-178) --
    plus tokenizer.json / config.json, through the product constructors (no weights= / engine= injection): the engine
    built from disk encodes and decodes exactly like the one built from the same tensors in memory."""
    import json
    from whisperlive_b200.engine import B200Whisper
    from whisperlive_b200.transcriber import B200WhisperModel
    dims = dims_for("micro.en")
    w = random_init(dims, seed=4)
    d = tmp_path / "model"
    d.mkdir()
    if fmt == "safetensors":
        from safetensors.torch import save_file
        save_file({k: v.half().contiguous() for k, v in w.items()}, str(d / "model.safetensors"))
    else:
        from whisperlive_b200 import ct2_format
        ct2_format.save_ct2_model_bin(w, str(d / "model.bin"))
    heads = [[1, 0], [1, 1]]
    (d / "config.json").write_text(json.dumps({"alignment_heads": heads}))
    (d / "preprocessor_config.json").write_text(json.dumps({"feature_size": dims.n_mels, "sampling_rate": 16000, "hop_length": 160,
                                                            "chunk_length": 30, "n_fft": 400, "processor_class": "ignored"}))
    build_synthetic_tokenizer(dims.vocab).save(str(d / "tokenizer.json"))
    eng = B200Whisper.from_model(str(d), max_streams=2, max_beam=5)
    assert eng.dims.d_model == dims.d_model and eng.dims.vocab == dims.vocab and eng.alignment_heads == [(1, 0), (1, 1)]
    ref, _ = engine("micro.en", seed=4)
    feats = np.stack([feats_for(dims, 5.0, 1), feats_for(dims, 8.0, 2)])
    a, b = np.asarray(eng.encode(feats)), np.asarray(ref.encode(feats))
    assert np.array_equal(a, b), float(np.abs(a - b).max())
    model = B200WhisperModel(str(d), max_streams=2, max_beam=5)          # the call create_model makes (tokenizer.json from the dir)
    segs, info = model.transcribe(synth.speech_like(6.0, seed=3), beam_size=5, temperature=[0.0], log_prob_threshold=None)
    assert info.language == "en" and len(segs) > 0 and all(isinstance(s.text, str) for s in segs)


# --------------------------------------------------------------------------------------- K13 / K14
def test_detect_language_matches_oracle():
    eng, orc = engine("micro", seed=1)
    feats = np.stack([feats_for(eng.dims, 5.0, 3), feats_for(eng.dims, 9.0, 4)])
    got = eng.detect_language(eng.encode(feats))
    ref = orc.detect_language(orc.encode(feats))
    for g, r in zip(got, ref):
        gd, rd = dict(g), dict(r)
        assert max(abs(gd[k] - rd[k]) for k in rd) < 0.03
        assert g[0][0] == r[0][0] or abs(r[0][1] - r[1][1]) < 0.03


def test_align_matches_oracle():
    eng, orc = engine("micro.en", seed=3)
    dims = eng.dims
    feats = np.stack([feats_for(dims, 7.5, 5), feats_for(dims, 3.0, 6)])
    enc, oenc = eng.encode(feats), orc.encode(feats)
    rng = np.random.default_rng(5)
    text = [rng.integers(256, 50000, 14).tolist(), rng.integers(256, 50000, 5).tolist()]
    nf = [750, 300]
    got = eng.align(enc, [orc.spec.sot], text, nf)
    ref = orc.align(oenc, [orc.spec.sot], text, nf)
    for g, r, t in zip(got, ref, text):
        assert len(g.text_token_probs) == len(t)
        np.testing.assert_allclose(g.text_token_probs, r.text_token_probs, atol=0.02, rtol=0.05)
        _check_alignment(g.alignments, r.alignments, len(t))


# --------------------------------------------------------------------------------------- end to end (Boundary B)
def _compare_transcripts(got, ref):
    """(segments, info) pairs of the CUDA transcriber against the oracle-engine transcriber: identical, or identical up to
    an explained decode divergence (near-tie) after which only the average log-probs are comparable."""
    for (gs, gi), (rs, ri) in zip(got, ref):
        assert gi.language == ri.language and gi.duration == ri.duration
        same = [a.tokens == b.tokens for a, b in zip(gs, rs)]
        print("segments", len(gs), len(rs), "identical:", sum(same))
        assert len(gs) > 0
        if len(gs) == len(rs) and all(same):
            for a, b in zip(gs, rs):
                assert a.start == pytest.approx(b.start, abs=1e-6) and a.end == pytest.approx(b.end, abs=1e-6)
                # avg_logprob covers the whole window's hypothesis, including a tail after the last closed
                # timestamp pair that the segment split discards -- that tail may legitimately differ
                assert a.avg_logprob == pytest.approx(b.avg_logprob, abs=0.25)
        else:
            # a different segmentation is legal only as the consequence of an explained decode divergence: the first
            # window's hypothesis must then differ, and the generate-level tests bound such divergences
            first = next((k for k, (a, b) in enumerate(zip(gs, rs)) if a.tokens != b.tokens), min(len(gs), len(rs)))
            print("first differing segment", first, gs[first].tokens[:8] if first < len(gs) else None,
                  rs[first].tokens[:8] if first < len(rs) else None)
            assert first < min(len(gs), len(rs)) or len(gs) != len(rs)
            # everything BEFORE the divergence is identical, times included
            for a, b in zip(gs[:first], rs[:first]):
                assert a.tokens == b.tokens and a.start == pytest.approx(b.start, abs=1e-6) and a.end == pytest.approx(b.end, abs=1e-6)
            # and the divergence itself is a near-tie: the two transcripts' average log-probs agree
            if first < min(len(gs), len(rs)):
                assert gs[first].avg_logprob == pytest.approx(rs[first].avg_logprob, abs=0.3)



def test_transcribe_end_to_end_matches_oracle_pipeline():
    from whisperlive_b200.feature_extractor import FeatureExtractor
    from whisperlive_b200.transcriber import B200WhisperModel
    eng, orc = engine("micro.en", seed=0)
    dims = eng.dims
    hf = build_synthetic_tokenizer(dims.vocab)
    gpu = B200WhisperModel("micro.en", engine=eng, hf_tokenizer=hf, feature_extractor=FeatureExtractor(eng, dims.n_mels))
    cpu = B200WhisperModel("micro.en", engine=orc, hf_tokenizer=hf, feature_extractor=OracleFeatureExtractor(dims.n_mels))
    audios = [synth.speech_like(6.0, seed=1), synth.speech_like(33.0, seed=2)]
    kw = dict(temperature=[0.0], log_prob_threshold=None, beam_size=5)
    got = gpu.transcribe_batch(audios, [kw, kw])
    ref = [cpu.transcribe(a, **kw) for a in audios]
    _compare_transcripts(got, ref)


# --------------------------------------------------------------------------------------- BASELINE configs at full size
def test_small_en_greedy_30s_config2():
    """BASELINE config 2: small.en shape (d=768, 12 heads, 12+12 layers, 80 mels), ONE stream, a 30 s chunk, greedy.
    Exercises what the other sizes do not: a single decoder row (N tile 16, cross-attention with one query row),
    GEMM K = 768 / 3072 (12 and 48 k-blocks), 12 heads."""
    import time
    dims = dims_for("small.en")
    w = random_init(dims, seed=11)
    from whisperlive_b200.engine import B200Whisper
    eng = B200Whisper(dims, w, max_streams=1, max_beam=1, enc_slots=2)
    orc = OracleWhisper(w, dims)
    wav = synth.speech_like(30.0, seed=1234)
    got_mel = eng.mel([wav])[0]
    ref_mel = omel.log_mel(wav, dims.n_mels)
    assert np.abs(got_mel - ref_mel).max() < 2e-4
    feats = omel.pad_or_trim(ref_mel[:, :-1])[None]
    enc = eng.encode(feats)
    t0 = time.time()
    oenc = orc.encode(feats)
    print(f"oracle small.en encoder {time.time() - t0:.1f} s")
    ref = oenc.enc.numpy()
    err = np.abs(np.asarray(enc) - ref)
    rel_rms = float(np.sqrt((err ** 2).mean() / (ref ** 2).mean()))
    print(f"encoder small.en: max err {err.max():.4f} rel rms {rel_rms:.5f}")
    assert rel_rms < 0.008 and err.max() < 0.08
    kw = dict(beam_size=1, max_length=2 * 64, suppress_tokens=[-1], return_scores=True, return_no_speech_prob=True)
    prompts = [[orc.spec.sot]]
    got = eng.generate(enc, prompts, **kw)
    refg = orc.generate(oenc, prompts, **kw)
    n_div = _compare_generation(got, refg, "small.en greedy", orc, oenc, prompts, kw, eng=eng, enc=enc)
    print(f"small.en greedy 30 s: {len(got[0].sequences_ids[0])} tokens, divergences {n_div}, score {got[0].scores[0]:.4f} vs {refg[0].scores[0]:.4f}")
    assert len(got[0].sequences_ids[0]) >= 8
    del eng


_LARGE = {}


def _large_v3():
    """One large-v3-shaped engine + oracle shared by the full-size tests (init is the expensive part)."""
    if not _LARGE:
        import time
        t0 = time.time()
        dims = dims_for("large-v3")
        w = random_init(dims, seed=5)
        from whisperlive_b200.engine import B200Whisper
        # 10 alignment heads in the upper layers (the released large-v3 config lists 10); engine and oracle read them
        # from the same dims object
        dims.alignment_heads = [(dims.dec_layers - 1 - (i // 4), (3 * i) % dims.n_heads) for i in range(10)]
        _LARGE["eng"] = B200Whisper(dims, w, max_streams=8, max_beam=4, enc_slots=10)
        _LARGE["orc"] = OracleWhisper(w, dims)
        print(f"large-v3 init {time.time() - t0:.1f} s")
    return _LARGE["eng"], _LARGE["orc"]


def test_large_v3_b8_beam4_config3():
    """BASELINE config 3: large-v3, B = 8 streams with chunks U[5,30] s, beam 4, >= 40 decoded tokens.  All 8 streams
    run on the device in one batch (R = 32 decoder rows, N tile 32); the CPU oracle re-derives three of them (its
    encoder costs ~2.6 TFLOP per stream), token for token with the explained-divergence rule, and every stream is
    checked for batch invariance against a solo run of the engine."""
    import time
    eng, orc = _large_v3()
    dims, sp = eng.dims, orc.spec
    durs = synth.chunk_durations(8, 5.0, 30.0, seed=1234)
    feats = np.stack([feats_for(dims, d, 1234 + i) for i, d in enumerate(durs)])
    enc = eng.encode(feats)
    sot_seq = [sp.sot, sp.sot + 1, sp.sot + 1 + dims.num_languages + 1]
    kw = dict(beam_size=4, max_length=2 * 40, suppress_tokens=[-1], suppress_blank=True, return_scores=True)
    prompts = [sot_seq] * 8
    got = eng.generate(enc, prompts, **kw)
    assert all(len(g.sequences_ids[0]) >= 1 for g in got)
    print("config 3 lengths", [len(g.sequences_ids[0]) for g in got], "steps", [g.steps for g in got])
    check = [0, 3, 7]
    t0 = time.time()
    oenc = orc.encode(feats[check])
    refs = orc.generate(oenc, [sot_seq] * len(check), **kw)
    print(f"oracle: 3 streams encoder + beam-4 decode {time.time() - t0:.1f} s")
    sub = enc.select(check)
    n_div = _compare_generation([got[i] for i in check], refs, "large-v3 B8 beam4", orc, oenc, [sot_seq] * len(check), kw,
                                eng=eng, enc=sub)
    print("config 3 divergences (explained):", n_div)
    # batch invariance of the whole path: stream 5 decoded alone gives the same hypothesis
    solo = eng.generate(enc.select([5]), [sot_seq], **kw)[0]
    assert solo.sequences_ids[0] == got[5].sequences_ids[0] or abs(solo.scores[0] - got[5].scores[0]) < SCORE_TOL
    enc.release()


def test_large_v3_detect_language_and_align():
    """K13 / K14 at the architecture the metric is quoted on: 128 mels, 20 heads, 32 layers, 100 languages."""
    eng, orc = _large_v3()
    dims, sp = eng.dims, orc.spec
    feats = np.stack([feats_for(dims, 8.0, 31), feats_for(dims, 5.0, 32)])
    enc, oenc = eng.encode(feats), orc.encode(feats)
    got = eng.detect_language(enc)
    ref = orc.detect_language(oenc)
    for g, r in zip(got, ref):
        gd, rd = dict(g), dict(r)
        assert len(gd) == 100 and max(abs(gd[k] - rd[k]) for k in rd) < 0.03
        assert g[0][0] == r[0][0] or abs(r[0][1] - r[1][1]) < 0.03
    rng = np.random.default_rng(9)
    text = [rng.integers(256, 50000, 18).tolist(), rng.integers(256, 50000, 7).tolist()]
    nf = [800, 500]
    sot_seq = [sp.sot, sp.sot + 1, sp.sot + 1 + dims.num_languages + 1]
    ga = eng.align(enc, sot_seq, text, nf)
    ra = orc.align(oenc, sot_seq, text, nf)
    for g, r, t in zip(ga, ra, text):
        np.testing.assert_allclose(g.text_token_probs, r.text_token_probs, atol=0.02, rtol=0.05)
        _check_alignment(g.alignments, r.alignments, len(t))
    enc.release()


def _check_alignment(got, ref, n_text):
    """DTW paths are monotone staircases from (0,0) to the same corner; an fp16-sized perturbation of the attention
    weights may move a jump, by a bounded number of frames: every token's first frame within ALIGN_MAX_SHIFT frames of
    the oracle's, the median within 1."""
    ga, ra = np.array(got), np.array(ref)
    assert ga[0].tolist() == [0, 0] and ga[-1].tolist() == ra[-1].tolist()
    assert (np.diff(ga[:, 0]) >= 0).all() and (np.diff(ga[:, 1]) >= 0).all() and (np.abs(np.diff(ga, axis=0)).sum(1) >= 1).all()
    jump_g = [int(ga[ga[:, 0] == i, 1].min()) for i in range(n_text + 1)]
    jump_r = [int(ra[ra[:, 0] == i, 1].min()) for i in range(n_text + 1)]
    diff = np.abs(np.array(jump_g) - np.array(jump_r))
    print("align jump diffs", diff.tolist())
    assert np.median(diff) <= 1 and diff.max() <= ALIGN_MAX_SHIFT, diff.tolist()


def test_transcribe_batch_more_streams_than_slots():
    """ADVICE r1 (medium): n > max_streams streams, audio longer than one window -- the transcriber encodes in groups
    of max_streams and hands every group's encoder slots back explicitly, so the pool (2 x max_streams) never runs dry
    and every slot is free again afterwards."""
    import gc
    from whisperlive_b200.engine import B200Whisper
    from whisperlive_b200.feature_extractor import FeatureExtractor
    from whisperlive_b200.transcriber import B200WhisperModel
    dims = dims_for("micro.en")
    eng = B200Whisper(dims, random_init(dims, seed=0), max_streams=2, max_beam=5)
    m = B200WhisperModel("micro.en", engine=eng, hf_tokenizer="synthetic", feature_extractor=FeatureExtractor(eng, dims.n_mels))
    audios = [synth.speech_like(33.0 if i % 2 else 6.0, seed=40 + i) for i in range(5)]
    kw = dict(temperature=[0.0], beam_size=5, log_prob_threshold=None, compression_ratio_threshold=None)
    out = m.transcribe_batch(audios, [kw] * 5)
    assert len(out) == 5 and all(segs is not None and len(segs) > 0 for segs, _ in out)
    solo = m.transcribe(audios[3], **kw)      # no sampling rungs: batched and solo runs are comparable token for token
    assert [s.tokens for s in solo[0]] == [s.tokens for s in out[3][0]]
    gc.collect()
    assert eng.free_slots() == eng.enc_slots


# --------------------------------------------------------------------------------------- full size (BASELINE config)
def test_full_size_large_v3_single_stream():
    """The architecture BASELINE.json's metric is quoted on (large-v3: d=1280, 20 heads, 32+32 layers, 128 mels,
    51866 tokens) at a batch the CPU oracle finishes in seconds: one 9 s stream.  Checks K1 (128-mel filterbank),
    K2-K7 (encoder output), K8-K12 (teacher-forced logits and the beam-4 hypothesis, re-scored by the oracle) and two
    size-independent properties: batch invariance of the encoder and run-to-run bit-reproducibility of generate
    (deterministic split-K, no atomics)."""
    import time
    eng, orc = _large_v3()
    dims = eng.dims
    wav = synth.speech_like(9.0, seed=21)
    ref_mel = omel.log_mel(wav, dims.n_mels)
    got_mel = eng.mel([wav])[0]
    assert got_mel.shape == ref_mel.shape == (128, len(wav) // 160 + 1)
    assert np.abs(got_mel - ref_mel).max() < 2e-4
    feats = omel.pad_or_trim(ref_mel[:, :-1])[None]
    enc = eng.encode(feats)
    got = np.asarray(enc)
    t1 = time.time()
    oenc = orc.encode(feats)
    ref = oenc.enc.numpy()
    print(f"oracle encoder {time.time() - t1:.1f} s")
    err = np.abs(got - ref)
    rel_rms = float(np.sqrt((err ** 2).mean() / (ref ** 2).mean()))
    print(f"encoder large-v3: max err {err.max():.4f} mean err {err.mean():.5f} rel rms {rel_rms:.5f} ref mean abs {np.abs(ref).mean():.3f}")
    assert rel_rms < 0.008 and err.mean() < 0.006 and err.max() < 0.06
    # batch invariance: the same stream next to a different one gives the same encoder output
    other = feats_for(dims, 21.0, 22)[None]
    pair = np.asarray(eng.encode(np.concatenate([other, feats])))
    assert np.abs(pair[1] - got[0]).max() < 2e-3
    # teacher-forced logits over a short token sequence
    rng = np.random.default_rng(8)
    toks = [[orc.spec.sot] + rng.integers(0, 50000, 5).tolist()]
    lg = eng.decode_logits(enc, toks)[0]
    from oracle import model as om
    with torch.no_grad():
        ref_lg = om.decoder_forward(orc.w, torch.tensor(toks), oenc.xkv, om.DecoderState(dims.dec_layers), dims.n_heads,
                                    dims.dec_layers)[0].numpy()
    lerr = np.abs(lg - ref_lg)
    print(f"logits large-v3: max err {lerr.max():.4f} mean {lerr.mean():.5f} (logit std {ref_lg.std():.2f})")
    assert lerr.max() < LOGIT_TOL and lerr.mean() < 0.015                      # measured: 0.024 / 0.0034
    # beam-4 generate, a few tokens: the engine's hypothesis, teacher-forced through the oracle, scores what the engine says
    sot_seq = [orc.spec.sot, orc.spec.sot + 1, orc.spec.sot + 1 + dims.num_languages + 1]
    kw = dict(beam_size=4, max_length=2 * 8, suppress_tokens=[-1], suppress_blank=True)
    a = eng.generate(enc, [sot_seq], **kw)[0]
    b = eng.generate(enc, [sot_seq], **kw)[0]
    assert a.sequences_ids == b.sequences_ids and a.scores == b.scores, "generate is not bit-reproducible"
    rescored = _oracle_rescore(orc, oenc, 0, sot_seq, a.sequences_ids[0], kw)
    print(f"generate large-v3 beam 4: {len(a.sequences_ids[0])} tokens, engine score {a.scores[0]:.4f}, oracle score of the same tokens {rescored:.4f}")
    assert abs(rescored - a.scores[0]) < 0.02                                    # measured: 0.0013


# --------------------------------------------------------------------------------------- BASELINE config 1 input
def test_config1_jfk_chunk():
    """BASELINE config 1's input -- the reference's only audio asset, assets/jfk.flac (its WER test, tests/test_server.py:
    92-118), decoded + resampled to 16 kHz by tests/golden/make_golden_jfk.py into a committed fixture: 176 000 samples of
    REAL speech (everything else here is synthetic).  K1 on it against the oracle, then the whole single-client path at
    the tiny.en shape (random weights: no checkpoint offline, so this pins the arithmetic, not the transcript)."""
    from whisperlive_b200.feature_extractor import FeatureExtractor
    from whisperlive_b200.transcriber import B200WhisperModel
    pcm = np.load(os.path.join(os.path.dirname(__file__), "golden", "jfk_16k_i16.npy")).astype(np.float32) / 32768.0
    assert pcm.shape == (176000,)
    eng, orc = engine("tiny.en", seed=0)
    dims = eng.dims
    feats = FeatureExtractor(eng, dims.n_mels)(pcm)
    ref = omel.log_mel(pcm, dims.n_mels)
    assert feats.shape == ref.shape == (dims.n_mels, 1101)
    print("jfk mel max err", float(np.abs(feats - ref).max()))
    assert float(np.abs(feats - ref).max()) < 2e-4
    hf = build_synthetic_tokenizer(dims.vocab)
    gpu = B200WhisperModel("tiny.en", engine=eng, hf_tokenizer=hf, feature_extractor=FeatureExtractor(eng, dims.n_mels))
    cpu = B200WhisperModel("tiny.en", engine=orc, hf_tokenizer=hf, feature_extractor=OracleFeatureExtractor(dims.n_mels))
    kw = dict(temperature=[0.0], log_prob_threshold=None, beam_size=5)       # the live path's defaults (beam 5)
    got = [gpu.transcribe(pcm, **kw)]
    refs = [cpu.transcribe(pcm, **kw)]
    assert got[0][1].duration == pytest.approx(11.0)
    _compare_transcripts(got, refs)


# --------------------------------------------------------------------------------------- N2: decode session
def _same_hypotheses(a, b, what):
    """Two runs of the ENGINE over the same stream.  The decode steps use the same kernels row for row; the batched
    prefill does not (its GEMM / cross-attention splits depend on how many prompt rows share the pass), so the cached
    prompt K/V may differ in the last fp16 bit: hypotheses agree, or the two runs sit on a near-tie."""
    assert abs(a.no_speech_prob - b.no_speech_prob) < 2e-3, what
    if a.sequences_ids[0] == b.sequences_ids[0]:
        assert abs(a.scores[0] - b.scores[0]) < 2e-3, (what, a.scores, b.scores)
    else:
        print("near-tie between two engine runs:", what, a.scores[0], b.scores[0])
        assert abs(a.scores[0] - b.scores[0]) < SCORE_TOL, (what, a.sequences_ids[0][:12], b.sequences_ids[0][:12])


@pytest.mark.parametrize("name,beam", [("micro.en", 5), ("micro", 4), ("tiny", 1)])
def test_decode_session_step_level_admission(name, beam):
    """N2 (include/wlb200.h, wl_session_*): streams admitted into the RUNNING device-side decode loop at different token
    steps, decoded in bounded slices, collected one by one with their indices refilled -- and one-shot calls
    (generate / align) interleaved between the slices -- give exactly the hypotheses of a one-shot ``generate`` over the
    same streams (reference: batches run to completion, whisper_live/batch_inference.py:155-187)."""
    eng, orc = engine(name, seed=0)
    dims, sp = eng.dims, orc.spec
    durs = [6.0, 9.0, 5.0, 12.0, 7.0, 4.0]
    feats = np.stack([feats_for(dims, d, 60 + i) for i, d in enumerate(durs)])
    enc_a, enc_b = eng.encode(feats[:4]), eng.encode(feats[4:])
    views = [enc_a.select([i]) for i in range(4)] + [enc_b.select([i]) for i in range(2)]
    base = [sp.sot] if not dims.multilingual else [sp.sot, sp.sot + 1, sp.sot + 1 + dims.num_languages + 1]
    rng = np.random.default_rng(23)
    prev = lambda n: [sp.timestamp_begin - 3] + rng.integers(256, 40000, n).tolist()
    prompts = [base, prev(40) + base, base, prev(150) + base, base + [sp.no_timestamps], prev(9) + base]
    lengths = [2 * 30, 448, 2 * 18, 448, 2 * 25, 2 * 40]
    kw = dict(beam_size=beam, suppress_tokens=[1, 2, 3], return_scores=True, return_no_speech_prob=True)
    # reference: one-shot generate, 4 streams per call like the session's capacity (same kernels for every row)
    ref = eng.generate(enc_a, prompts[:4], max_length=448, max_length_per_stream=lengths[:4], **kw)
    ref += eng.generate(enc_b.join([views[4], views[5], views[0], views[1]]), prompts[4:] + prompts[:2], max_length=448,
                        max_length_per_stream=lengths[4:] + lengths[:2], **kw)[:2]
    sess = eng.open_decode_session(capacity=4, **kw)
    where, got, joined_at = {}, {}, {}
    order = [0, 1, 2, 3, 4, 5]
    queue = list(order)

    def admit(n):
        take = [queue.pop(0) for _ in range(min(n, len(queue), len(sess.free_indices())))]
        if take:
            idx = sess.admit([views[i] for i in take], [prompts[i] for i in take], [lengths[i] for i in take])
            for i, ix in zip(take, idx):
                where[ix] = i
                joined_at[i] = sess.steps
    admit(2)                                           # streams 0, 1 start the loop
    for ix in sess.run(max_steps=3):                   # 3 token steps (fewer only if somebody already finished)
        got[where.pop(ix)] = sess.collect(ix)
    assert 1 <= sess.last_steps <= 3
    admit(1)                                           # stream 2 joins a loop that has already run for a few steps
    # one-shot calls between two slices of the session leave it alone (own decode state + self-attention cache)
    side = eng.generate(views[5], [prompts[5]], max_length=lengths[5], **kw)[0]
    if eng.alignment_heads:
        eng.align(views[0], base, [[300, 301, 302]], [200])
    guard = 0
    while sess.live or queue:
        guard += 1
        assert guard < 400
        for ix in sess.run(max_steps=7):
            got[where.pop(ix)] = sess.collect(ix)
        admit(4)                                       # refill whatever is free
    sess.close()
    assert sorted(got) == order
    assert joined_at[0] == 0 and joined_at[2] > 0 and all(joined_at[i] > joined_at[2] for i in (4, 5))
    for i in order:
        _same_hypotheses(got[i], ref[i], f"{name} beam{beam} stream {i}")
    _same_hypotheses(side, ref[5], "interleaved one-shot generate")
    print(f"decode session {name} beam {beam}: joined at steps {joined_at}, lengths {[len(got[i].sequences_ids[0]) for i in order]}, "
          f"{sess.steps} steps in {sess.runs} slices")
    enc_a.release(); enc_b.release()


def test_decode_session_errors():
    eng, orc = engine("micro.en", seed=0)
    dims, sp = eng.dims, orc.spec
    enc = eng.encode(np.stack([feats_for(dims, 5.0, 1), feats_for(dims, 5.0, 2)]))
    v0, v1 = enc.select([0]), enc.select([1])
    with pytest.raises(ValueError):
        eng.open_decode_session(beam_size=1, sampling_topk=0, sampling_temperature=0.7)
    sess = eng.open_decode_session(capacity=2, beam_size=5)
    with pytest.raises(Exception, match="has not finished"):
        sess.collect(0)
    (i0,) = sess.admit([v0], [[sp.sot]], [20])
    with pytest.raises(Exception, match="still holds a stream"):
        sess.admit([v1], [[sp.sot]], [20], indices=[i0])
    with pytest.raises(Exception, match="out of range|no room"):
        sess.admit([v1], [[sp.sot] * 30], [20])
    (i1,) = sess.admit([v1], [[sp.sot]], [20])          # the failed admission left index 1 free
    with pytest.raises(RuntimeError):
        sess.admit([v1], [[sp.sot]], [20])               # no free index
    done = set()
    for _ in range(40):
        done |= set(sess.run(max_steps=4))
        if len(done) == 2:
            break
    assert done == {i0, i1}
    r = sess.collect(i0)
    assert 1 <= len(r.sequences_ids[0]) <= 10
    sess.close()
    enc.release()


def test_step_rounds_equal_transcribe_batch():
    """The transcriber on step-level rounds (``TranscribeSession.step_round``: streams added while others are in the
    middle of their decode, multi-window audio, word timestamps) gives the segments of the run-to-completion
    ``transcribe_batch``."""
    from whisperlive_b200.feature_extractor import FeatureExtractor
    from whisperlive_b200.transcriber import B200WhisperModel
    eng, _ = engine("micro.en", seed=0)
    dims = eng.dims
    m = B200WhisperModel("micro.en", engine=eng, hf_tokenizer=build_synthetic_tokenizer(dims.vocab),
                         feature_extractor=FeatureExtractor(eng, dims.n_mels))
    audios = [synth.speech_like(33.0, seed=70), synth.speech_like(6.0, seed=71), synth.speech_like(14.0, seed=72),
              synth.speech_like(8.0, seed=73), synth.speech_like(5.0, seed=74)]
    kws = [dict(temperature=[0.0], beam_size=5, log_prob_threshold=None, compression_ratio_threshold=None,
                word_timestamps=(i == 2)) for i in range(5)]
    ref = m.transcribe_batch(audios, kws)
    sess = m.open_session()
    handles = sess.add_streams(audios[:2], kws[:2])
    results, rounds = {}, 0
    late = [(2, 2), (4, 3), (6, 4)]                      # (round, stream): admitted while the others are mid-decode
    while sess.pending() or late:
        while late and late[0][0] <= rounds:
            handles += sess.add_streams([audios[late[0][1]]], [kws[late[0][1]]])
            late.pop(0)
        sess.step_round(max_steps=5)
        rounds += 1
        for e in sess.pop_finished():
            results[e.handle] = sess.result_of(e)
        assert rounds < 500
    sess.close()
    assert any(a > 0 for a in sess.admitted_steps)       # somebody joined a loop that was already running
    for h, (segs_ref, _info) in zip(handles, ref):
        segs, _ = results[h]
        assert [s.tokens for s in segs] == [s.tokens for s in segs_ref]
        assert [(s.start, s.end) for s in segs] == [(s.start, s.end) for s in segs_ref]
        for a, b in zip(segs, segs_ref):
            assert (a.words is None) == (b.words is None)
            if a.words is not None:
                assert [(w.word, w.start, w.end) for w in a.words] == [(w.word, w.start, w.end) for w in b.words]
    print(f"step rounds: {rounds} rounds, admissions at session steps {sess.admitted_steps}")
