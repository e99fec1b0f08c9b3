"""The decode-step kernels of the default path above 16 decoder rows, one by one, at the batch the benchmark decodes
(large-v3, 32 streams x beam 4 = 128 rows) and at the edges of every template instance:

  * the split-K decode GEMM (csrc/dec_gemm.cu), every K range checked against the float64 product over exactly its
    k-blocks;
  * the cross-attention kernel + the combine kernel (K11) at every key split, against a float64 softmax(q K^T / 8) V;
  * the cross-attention pool layout from both ends: the head-split GEMM epilogue that writes it and the kernel that
    reads it;
  * the self-attention kernel (K10): beam indirection, the new position's k / v and the cache append;
  * the consumers that fold split-K partials: layernorm_update_rows and gelu_cast;
  * and one whole beam-4 decode of 32 streams (R = 128) against the oracle, the only test here that runs the kernels as
    programmatic dependents inside the captured decode graph.

Every reference is float64 numpy over the exact fp16 inputs; where the kernel defines an fp32 intermediate (q = bias +
the K ranges in index order), the reference forms it the same way in fp32 first."""
import zlib

import numpy as np
import pytest
from scipy.special import erf

from whisperlive_b200.config import dims_for

pytestmark = pytest.mark.gpu

S_ENC, T_MAX = 1500, 448

_ENG = []


def engine():
    """A small context: the hooks only borrow its stream."""
    if not _ENG:
        from whisperlive_b200.engine import B200Whisper
        from whisperlive_b200.weights import random_init
        dims = dims_for("micro.en")
        _ENG.append(B200Whisper(dims, random_init(dims, seed=0), max_streams=1, max_beam=1))
    return _ENG[0]


def f32_sum(bias, parts):
    """bias + parts[0] + parts[1] + ... in fp32, in index order (what the consumers of split-K partials compute)."""
    acc = np.zeros(parts.shape[1:], np.float32) if bias is None else np.broadcast_to(bias.astype(np.float32), parts.shape[1:])
    for p in parts:
        acc = (acc + p).astype(np.float32)
    return acc


# --------------------------------------------------------------------------------------- split-K decode GEMM
DG_ROWS = [1, 16, 17, 32, 33, 64, 65, 100, 128, 256]    # every row-tile width (16 / 32 / 64 / 128) and its edges
DG_SHAPES = {   # (n_out, K) of the decoder linears: QKV, O / cross-O / q-cross, FC1, FC2
    "tiny_qkv": (1152, 384), "tiny_o": (384, 384), "tiny_fc1": (1536, 384), "tiny_fc2": (384, 1536),
    "v3_qkv": (3840, 1280), "v3_o": (1280, 1280), "v3_fc1": (5120, 1280), "v3_fc2": (1280, 5120),
    "ragged": (200, 64),
}


def dg_inputs(n_out, K, R, seed):
    rng = np.random.default_rng(seed)
    w = (rng.standard_normal((n_out, K), dtype=np.float32) / np.sqrt(K)).astype(np.float16)
    x = rng.standard_normal((R, K), dtype=np.float32).astype(np.float16)
    return w, x


def check_partials(parts, w, x, nsplit):
    """Partial s must be the float64 product over exactly k-blocks [s * kbs, min((s + 1) * kbs, total)) -- the range
    boundaries and the short last range are pinned, not only the sum."""
    K = w.shape[1]
    kb = -(-K // 64)
    kbs = -(-kb // nsplit)
    assert parts.shape[0] == nsplit
    w64, x64 = w.astype(np.float64), x.astype(np.float64)
    for s in range(nsplit):
        k0, k1 = s * kbs * 64, min((s + 1) * kbs * 64, K)
        assert k0 < k1, (s, nsplit, K)
        ref = x64[:, k0:k1] @ w64[:, k0:k1].T
        err = np.abs(parts[s] - ref).max()
        assert err < 1e-4, (f"K range {s}/{nsplit} (k {k0}..{k1})", err)


@pytest.mark.parametrize("shape", list(DG_SHAPES))
@pytest.mark.parametrize("R", DG_ROWS)
def test_dec_gemm_engine_split(R, shape):
    n_out, K = DG_SHAPES[shape]
    w, x = dg_inputs(n_out, K, R, seed=R * 7919 + K + n_out)
    parts, ns = engine().test_dec_gemm(w, x, 0)
    if R == 128:
        print(f"dec_gemm R=128 {shape} ({n_out}x{K}): {ns} K ranges")
    assert 1 <= ns <= 8
    check_partials(parts, w, x, ns)
    again, ns2 = engine().test_dec_gemm(w, x, ns)
    assert ns2 == ns and np.array_equal(parts.view(np.uint32), again.view(np.uint32)), "two launches differ"


def valid_splits(kb):
    return [s for s in range(1, kb + 1) if -(-kb // -(-kb // s)) == s]


@pytest.mark.parametrize("R", [17, 65, 128, 256])
def test_dec_gemm_every_split_of_k1280(R):
    """Every K split of 20 k-blocks the kernel can form, including those beyond the plan's cap of 8 and the 7-range
    split whose last range is 2 k-blocks of 3 (the O projections at the benchmark batch)."""
    w, x = dg_inputs(1280, 1280, R, seed=R)
    splits = valid_splits(20)
    assert splits == [1, 2, 3, 4, 5, 7, 10, 20]
    for s in splits:
        parts, used = engine().test_dec_gemm(w, x, s)
        assert used == s
        check_partials(parts, w, x, s)


@pytest.mark.parametrize("R", [65, 128])
def test_dec_gemm_fc2_k5120_eight_ranges(R):
    w, x = dg_inputs(1280, 5120, R, seed=5120 + R)
    parts, used = engine().test_dec_gemm(w, x, 8)
    assert used == 8
    check_partials(parts, w, x, 8)


@pytest.mark.parametrize("R", [17, 128])
def test_dec_gemm_vocabulary_projection(R):
    """The logits GEMM: one K range, 406 feature tiles, the last one 26 features wide."""
    w, x = dg_inputs(51866, 1280, R, seed=51866 + R)
    parts, used = engine().test_dec_gemm(w, x, 1)
    assert used == 1
    check_partials(parts, w, x, 1)


def test_dec_gemm_refuses_impossible_splits():
    from whisperlive_b200._lib import WlError
    w, x = dg_inputs(384, 1280, 17, seed=1)
    for bad in (6, 8, 9, 21, -1):          # 20 k-blocks: 6 / 8 / 9 ranges leave the last one empty, 21 > 20
        with pytest.raises(WlError, match="bad arguments|cannot be formed"):
            engine().test_dec_gemm(w, x, bad)
    w, x = dg_inputs(200, 64, 17, seed=2)
    with pytest.raises(WlError, match="cannot be formed"):
        engine().test_dec_gemm(w, x, 2)


# --------------------------------------------------------------------------------------- cross attention (K11)
def swizzle(kv):
    """Logical [..., 1500, 64] -> the pool layout: the 16-byte piece p of key s stored at piece p ^ (s & 7)."""
    lead = kv.shape[:-2]
    pieces = kv.reshape(*lead, S_ENC, 8, 8)
    s = np.arange(S_ENC)[:, None]
    perm = np.arange(8)[None, :] ^ (s & 7)     # an involution: stored piece q holds logical piece q ^ (s & 7)
    return np.ascontiguousarray(pieces[..., s, perm, :]).reshape(kv.shape)


def cross_ref(q_part, q_bias, K, V, slot, rps):
    """float64 softmax(q K^T) V per (stream, head) with q = fp32(bias + the K ranges in order) * 0.125."""
    q = (f32_sum(q_bias, q_part) * np.float32(0.125)).astype(np.float64)
    R, d = q.shape
    H = d // 64
    B = R // rps
    out = np.empty((R, d))
    probs = np.empty((R, H, S_ENC))
    for b in range(B):
        qb = q[b * rps:(b + 1) * rps].reshape(rps, H, 64).transpose(1, 0, 2)          # [H, rps, 64]
        Kb, Vb = K[slot[b]].astype(np.float64), V[slot[b]].astype(np.float64)        # [H, 1500, 64]
        s = qb @ Kb.transpose(0, 2, 1)
        p = np.exp(s - s.max(-1, keepdims=True))
        p /= p.sum(-1, keepdims=True)
        out[b * rps:(b + 1) * rps] = (p @ Vb).transpose(1, 0, 2).reshape(rps, d)
        probs[b * rps:(b + 1) * rps] = p.transpose(1, 0, 2)
    return out, probs


def done_pattern(kind, B):
    if kind == "none":
        return np.zeros(B, np.int32)
    if kind == "alternate":
        return (np.arange(B) % 2).astype(np.int32)
    if kind == "all_but_last":
        return (np.arange(B) != B - 1).astype(np.int32)
    if kind == "all_but_first":
        return (np.arange(B) != 0).astype(np.int32)
    raise ValueError(kind)


def cross_inputs(B, rps, H, q_nsplit, keys, seed):
    """Scores spanning about +-30.  keys = "peak": row 0 of every stream has a planted maximum (score ~45) at key 1499
    (the 92-key tail chunk), 127, 128 or a random key; "peak_high": the same with score ~100, beyond where exp() of a
    raw score overflows fp32; "negative": every score is negative, so that a key the kernel must not count (a zero row
    past the tail) would dominate the softmax."""
    rng = np.random.default_rng(seed)
    d, R = H * 64, B * rps
    n_slots = B + 3
    slot = rng.permutation(n_slots)[:B].astype(np.int32)     # a non-identity map into a larger pool
    q_bias = rng.standard_normal(d, dtype=np.float32)
    q_part = (rng.standard_normal((q_nsplit, R, d), dtype=np.float32) * np.float32(10 / np.sqrt(q_nsplit)))
    K = rng.standard_normal((n_slots, H, S_ENC, 64), dtype=np.float32)
    V = rng.standard_normal((n_slots, H, S_ENC, 64), dtype=np.float32).astype(np.float16)
    if keys == "negative":
        q_bias = np.abs(q_bias)
        q_part = np.abs(q_part)
        K = -np.abs(K) * np.float32(0.6)
    K = K.astype(np.float16)
    if keys.startswith("peak"):
        top = 100.0 if keys == "peak_high" else 45.0
        q = f32_sum(q_bias, q_part) * np.float32(0.125)
        for b in range(B):
            star = [1499, 127, 128, int(rng.integers(S_ENC))][b % 4]
            for h in range(H):
                qh = q[b * rps, h * 64:(h + 1) * 64].astype(np.float64)
                K[slot[b], h, star] = (qh * (top / (qh @ qh))).astype(np.float16)
    return q_part, q_bias, K, V, slot


XA_SPLITS = [0, 1, 2, 3, 4, 6, 12]
XA_CASES = [
    # B, rows per stream, H, q K ranges, done pattern, keys
    (1, 1, 2, 1, "none", "negative"),
    (1, 8, 20, 4, "none", "peak"),
    (4, 2, 6, 2, "alternate", "negative"),
    (4, 3, 20, 3, "all_but_last", "peak_high"),
    (4, 5, 2, 4, "all_but_first", "negative"),
    (32, 4, 20, 2, "alternate", "peak"),           # the benchmark step: large-v3, 32 streams, beam 4
    (32, 6, 6, 1, "all_but_first", "peak"),
    (32, 1, 20, 3, "all_but_last", "negative"),
    (32, 7, 2, 4, "alternate", "peak"),
    (40, 4, 6, 1, "alternate", "negative"),        # B > 32: the second ballot round of the live list
    (40, 8, 2, 2, "all_but_last", "peak_high"),
    (40, 2, 20, 3, "all_but_first", "peak"),
    (40, 7, 20, 4, "alternate", "negative"),
]


@pytest.mark.parametrize("case", XA_CASES, ids=lambda c: "B{}_rows{}_H{}_q{}_{}_{}".format(*c))
def test_cross_attention_every_key_split(case):
    B, rps, H, q_ns, pattern, keys = case
    eng = engine()
    q_part, q_bias, K, V, slot = cross_inputs(B, rps, H, q_ns, keys, seed=zlib.crc32(repr(case).encode()))
    Kp, Vp = swizzle(K), swizzle(V)
    ref, ref_probs = cross_ref(q_part, q_bias, K, V, slot, rps)
    vmax = float(np.abs(V).max())
    done = done_pattern(pattern, B)
    live_rows = np.repeat(done == 0, rps)
    sentinel = -7.5
    for ns in XA_SPLITS:
        out, _, used = eng.test_cross_attn(q_part, q_bias, Kp, Vp, slot, np.zeros(B, np.int32), rps, nsplit=ns,
                                           sentinel=sentinel)
        if ns == 0:
            assert used in XA_SPLITS[1:], used
            print(f"cross attention B={B} H={H} rows/stream={rps}: picked key split {used}")
        else:
            assert used == ns
        err = np.abs(out - ref).max()
        np.testing.assert_allclose(out, ref, atol=2e-3 * vmax, rtol=2e-3, err_msg=f"key split {used}")
        if pattern != "none":
            part, _, _ = eng.test_cross_attn(q_part, q_bias, Kp, Vp, slot, done, rps, nsplit=used, sentinel=sentinel)
            assert np.all(part[~live_rows] == sentinel), f"key split {used}: a done stream's rows were written"
            assert np.array_equal(part[live_rows].view(np.uint32), out[live_rows].view(np.uint32)), \
                f"key split {used}: a live stream's output depends on which other streams are done"
        print(f"  split {used}: max err {err:.2e} (atol {2e-3 * vmax:.2e})")
    out, probs, used = eng.test_cross_attn(q_part, q_bias, Kp, Vp, slot, done, rps, nsplit=1, probs=True)
    np.testing.assert_allclose(probs[live_rows], ref_probs[live_rows], atol=2e-5, rtol=2e-4)
    assert np.all(probs[~live_rows] == 0)
    print(f"  probabilities: max err {np.abs(probs[live_rows] - ref_probs[live_rows]).max():.2e}")


def test_cross_attention_refuses_impossible_key_splits():
    from whisperlive_b200._lib import WlError
    q_part, q_bias, K, V, slot = cross_inputs(2, 1, 2, 1, "peak", seed=3)
    for bad in (5, 7, 13):   # 12 chunks: 5 and 7 ranges leave an empty one
        with pytest.raises(WlError, match="cannot be formed"):
            engine().test_cross_attn(q_part, q_bias, swizzle(K), swizzle(V), slot, [0, 0], 1, nsplit=bad)


def test_headsplit_pool_layout_writer_and_reader():
    """The cross-KV GEMM epilogue writes the pool in the layout the cross-attention kernel reads.  Writer: the
    head-split output equals the numpy layout of the exact product (small integers: every sum is exact in fp32 and
    fp16), slots in reverse stream order.  Reader: that very pool as K, against the float64 reference on the logical K."""
    eng = engine()
    rng = np.random.default_rng(11)
    ns, H, Kdim = 2, 2, 128
    N = H * 64
    a = rng.integers(-3, 4, (ns * S_ENC, Kdim)).astype(np.float16)
    b = rng.integers(-3, 4, (N, Kdim)).astype(np.float16)
    bias = rng.integers(-8, 9, N).astype(np.float32)
    got = eng.test_gemm(a, b, bias, out="headsplit", hs_rows=S_ENC).reshape(ns, H, S_ENC, 64)
    exact = a.astype(np.float64) @ b.astype(np.float64).T + bias
    assert np.abs(exact).max() < 2048
    logical = exact.reshape(ns, S_ENC, H, 64).transpose(0, 2, 1, 3).astype(np.float16)   # [stream][h][s][64]
    want = swizzle(logical)[::-1]                                                          # slot = ns - 1 - stream
    assert np.array_equal(got.astype(np.float16).view(np.uint16), want.view(np.uint16)), "head-split layout differs"
    slot = np.arange(ns)[::-1].astype(np.int32)
    V = rng.standard_normal((ns, H, S_ENC, 64), dtype=np.float32).astype(np.float16)
    q_part = (rng.standard_normal((1, ns, N), dtype=np.float32) * np.float32(0.25))
    K_logical = np.empty_like(logical)
    K_logical[slot] = logical
    ref, _ = cross_ref(q_part, None, K_logical, V, slot, 1)
    out, _, _ = eng.test_cross_attn(q_part, None, got.astype(np.float16), swizzle(V), slot, [0] * ns, 1, nsplit=0)
    np.testing.assert_allclose(out, ref, atol=2e-3 * np.abs(V).max(), rtol=2e-3)


# --------------------------------------------------------------------------------------- self attention (K10)
SA_POS = [0, 1, 31, 32, 33, 63, 200, 447]   # 31..33 straddle the 32 positions fetched before the dependency wait


def self_inputs(R, H, form, rng, rot, n_rows):
    """form: "plain" (final q / k / v, no bias) or the number of K ranges (with a bias)."""
    d = H * 64
    pos = np.array([SA_POS[(r + rot) % len(SA_POS)] for r in range(R)], np.int32)
    active = np.array([0 if (R > 1 and r % 5 == 3) else 1 for r in range(R)], np.int32)
    wrow = rng.permutation(n_rows)[:R].astype(np.int32) if rot % 2 else None
    wr = np.arange(R) if wrow is None else wrow
    written = {(int(wr[r]), int(pos[r])) for r in range(R) if active[r]}
    # beam-style indirection: the later half of a row's history is its own, earlier positions come from other rows --
    # never from a (row, position) this launch writes
    src = np.zeros((R, T_MAX), np.int16)
    for r in range(R):
        for p in range(pos[r]):
            c = r if p >= pos[r] // 2 else int(rng.integers(n_rows))
            while (c, p) in written:
                c = int(rng.integers(n_rows))
            src[r, p] = c
    scale = np.concatenate([np.full(d, 8.0), np.ones(2 * d)]).astype(np.float32)   # q, k, v
    if form == "plain":
        part = (rng.standard_normal((1, R, 3 * d), dtype=np.float32) * scale)
        bias = None
    else:
        part = (rng.standard_normal((form, R, 3 * d), dtype=np.float32) * (scale / np.float32(np.sqrt(form))))
        bias = (rng.standard_normal(3 * d, dtype=np.float32) * np.float32(0.3))
    return part.astype(np.float32), bias, src, pos, active, wrow


def self_ref(part, bias, kc, vc, src, pos, active, H):
    qkv = f32_sum(bias, part)
    d = H * 64
    q = (qkv[:, :d] * np.float32(0.125)).astype(np.float64)
    k, v = qkv[:, d:2 * d].astype(np.float64), qkv[:, 2 * d:].astype(np.float64)
    out = np.full((len(pos), d), np.nan)
    for r in np.flatnonzero(active):
        n = pos[r]
        for h in range(H):
            sl = slice(h * 64, (h + 1) * 64)
            Kc = kc[src[r, :n], h, np.arange(n)].astype(np.float64)
            Vc = vc[src[r, :n], h, np.arange(n)].astype(np.float64)
            s = np.append(Kc @ q[r, sl], q[r, sl] @ k[r, sl])   # the new position: the unrounded fp32 k
            p = np.exp(s - s.max())
            p /= p.sum()
            out[r, sl] = p[:n] @ Vc + p[n] * v[r, sl]
    return out, qkv


@pytest.mark.parametrize("R,H", [(1, 6), (1, 20), (20, 6), (20, 20), (128, 6), (128, 20)])
def test_self_attention(R, H):
    eng = engine()
    rng = np.random.default_rng(R * 100 + H)
    d = H * 64
    sentinel = 5.25
    n_rows = R + 2
    kc = rng.standard_normal((n_rows, H, T_MAX, 64), dtype=np.float32).astype(np.float16)
    vc = rng.standard_normal((n_rows, H, T_MAX, 64), dtype=np.float32).astype(np.float16)
    for i, form in enumerate(["plain", 1, 2, 3, 4, 5, 6, 7, 8]):
        part, bias, src, pos, active, wrow = self_inputs(R, H, form, rng, i, n_rows)
        out, kc2, vc2 = eng.test_self_attn(part, bias, kc, vc, src, pos, active, wrow, sentinel=sentinel)
        ref, qkv = self_ref(part, bias, kc, vc, src, pos, active, H)
        on = active.astype(bool)
        vmax = max(float(np.abs(vc).max()), float(np.abs(qkv[:, 2 * d:]).max()))
        np.testing.assert_allclose(out[on], ref[on], atol=2e-3 * vmax, rtol=2e-3, err_msg=f"form {form}")
        assert np.all(out[~on] == sentinel), f"form {form}: an inactive row's output was written"
        # the cache append: fp16(k), fp16(v) of the new position, exactly, at (write row, pos); nothing else changes
        kw, vw = kc.copy(), vc.copy()
        wr = np.arange(R) if wrow is None else wrow
        for r in np.flatnonzero(on):
            kw[wr[r], :, pos[r]] = qkv[r, d:2 * d].astype(np.float16).reshape(H, 64)
            vw[wr[r], :, pos[r]] = qkv[r, 2 * d:].astype(np.float16).reshape(H, 64)
        assert np.array_equal(kc2.view(np.uint16), kw.view(np.uint16)), f"form {form}: K cache"
        assert np.array_equal(vc2.view(np.uint16), vw.view(np.uint16)), f"form {form}: V cache"
        print(f"self attention R={R} H={H} form {form}: max err {np.abs(out[on] - ref[on]).max():.2e}")


# --------------------------------------------------------------------------------------- folding split-K partials
@pytest.mark.parametrize("d", [128, 384, 1280])
@pytest.mark.parametrize("rows", [1, 128, 256])
def test_layernorm_update(rows, d):
    eng = engine()
    rng = np.random.default_rng(rows * 10 + d)
    gamma = (1 + 0.1 * rng.standard_normal(d)).astype(np.float32)
    beta = (0.1 * rng.standard_normal(d)).astype(np.float32)
    for ns in range(9):
        x = rng.standard_normal((rows, d), dtype=np.float32)
        x[::2] += np.float32(1e3)   # a large mean: a variance taken as E[x^2] - E[x]^2 would cancel away
        part = rng.standard_normal((ns, rows, d), dtype=np.float32) if ns else None
        bias = rng.standard_normal(d, dtype=np.float32) if ns else None
        xn, y = eng.test_layernorm_update(x, part, bias, gamma, beta)
        terms = [x.astype(np.float64)] + ([bias.astype(np.float64)[None]] + list(part.astype(np.float64)) if ns else [])
        ref_x = sum(terms)
        mag = sum(np.abs(t) for t in terms)
        assert np.all(np.abs(xn - ref_x) <= 1e-6 * mag), f"{ns} K ranges: updated x"
        mu = ref_x.mean(-1, keepdims=True)
        ref_y = (ref_x - mu) / np.sqrt(((ref_x - mu) ** 2).mean(-1, keepdims=True) + 1e-5) * gamma + beta
        np.testing.assert_allclose(y, ref_y, atol=4e-3, rtol=2e-3, err_msg=f"{ns} K ranges: y")


@pytest.mark.parametrize("rows,cols", [(1, 384), (17, 1536), (128, 5120), (256, 1536)])
def test_gelu_cast(rows, cols):
    """1..8 K ranges: up to 4 are summed unrolled, more in the rolled loop (tiny's FC1 at 17..32 rows gets 6)."""
    eng = engine()
    rng = np.random.default_rng(rows + cols)
    for ns in range(1, 9):
        part = (rng.standard_normal((ns, rows, cols), dtype=np.float32) * np.float32(3 / np.sqrt(ns)))
        bias = rng.standard_normal(cols, dtype=np.float32)
        y = eng.test_gelu_cast(part, bias)
        z = bias.astype(np.float64) + part.astype(np.float64).sum(0)
        ref = 0.5 * z * (1 + erf(z / np.sqrt(2)))
        np.testing.assert_allclose(y, ref, atol=1e-3, rtol=2e-3, err_msg=f"{ns} K ranges")


# --------------------------------------------------------------------------------------- the whole step at R = 128
def test_beam4_32_streams_against_oracle():
    """tiny (d = 384, H = 6) at 32 streams x beam 4: every decoder linear takes the BN = 128 split-K GEMM and the
    kernels run as programmatic dependents in the captured decode graph.  The oracle re-derives four streams (explained
    divergences only); one stream decoded alone gives the same hypothesis."""
    from oracle.engine import OracleWhisper
    from whisperlive_b200 import synth
    from whisperlive_b200.engine import B200Whisper
    from whisperlive_b200.weights import random_init
    from tests.test_gpu_parity import SCORE_TOL, _compare_generation, feats_for
    dims = dims_for("tiny")
    w = random_init(dims, seed=0)
    eng, orc = B200Whisper(dims, w, max_streams=32, max_beam=4), OracleWhisper(w, dims)
    sp = orc.spec
    durs = synth.chunk_durations(32, 5.0, 30.0, seed=4321)
    feats = np.stack([feats_for(dims, t, 4321 + i) for i, t in enumerate(durs)])
    enc = eng.encode(feats)
    sot_seq = [sp.sot, sp.sot + 1, sp.sot + 1 + dims.num_languages + 1]
    kw = dict(beam_size=4, max_length=2 * 40, suppress_tokens=[-1], suppress_blank=True, return_scores=True)
    got = eng.generate(enc, [sot_seq] * 32, **kw)
    assert all(len(g.sequences_ids[0]) >= 1 for g in got)
    print("R=128 lengths", [len(g.sequences_ids[0]) for g in got])
    check = [0, 13, 26, 31]
    oenc = orc.encode(feats[check])
    refs = orc.generate(oenc, [sot_seq] * len(check), **kw)
    n_div = _compare_generation([got[i] for i in check], refs, "tiny B32 beam4", orc, oenc, [sot_seq] * len(check), kw,
                                eng=eng, enc=enc.select(check))
    print("R=128 divergences (explained):", n_div)
    solo = eng.generate(enc.select([13]), [sot_seq], **kw)[0]
    assert solo.sequences_ids[0] == got[13].sequences_ids[0] or abs(solo.scores[0] - got[13].scores[0]) < SCORE_TOL
    enc.release()
