"""The encoder-pass kernels one by one, at the batch the benchmark encodes (large-v3, passes of 16 streams = 24000 rows)
and at the edges where they could go wrong unnoticed under the end-to-end encoder bounds:

  * self-attention on both paths -- the fused flash-attention kernel (csrc/flash_attn.cu) and the unfused scores GEMM
    + softmax_rows + P V GEMM in sub-passes of AB streams -- against a float64 softmax(Q K^T / 8) V, with inputs that
    drive the ragged 12th key tile, the online-softmax rescale, the max subtraction and the V^T pad columns;
  * the conv stem (prep_features, conv1 + GELU, conv2 + GELU + positions) against float64 convolutions;
  * layernorm_rows against a float64 LayerNorm;
  * and the whole encoder of a 2-layer large-v3-shaped model at a 16-stream pass followed by a 1-stream pass.

Every reference is float64 numpy over the exact fp16 (or fp32) inputs the kernel sees.  Each check prints its
measured maximum error; the tolerances below are set from the error sources and from those measurements (H100)."""
import os
import zlib

import numpy as np
import pytest
from scipy.special import erf

from whisperlive_b200.config import WhisperDims, dims_for

pytestmark = pytest.mark.gpu

S_ENC, S_PAD = 1500, 1536
U16 = 2.0 ** -11           # fp16 unit roundoff (half an ulp, relative)
NAN16 = np.uint16(0x7E5A)  # the NaN pattern output buffers are filled with before a launch

_ENG = []


def engine():
    """A small context: the attention and LayerNorm hooks only borrow its stream."""
    if not _ENG:
        from whisperlive_b200.engine import B200Whisper
        from whisperlive_b200.weights import random_init
        dims = dims_for("micro.en")
        _ENG.append(B200Whisper(dims, random_init(dims, seed=0), max_streams=1, max_beam=1))
    return _ENG[0]


# --------------------------------------------------------------------------------------- self-attention
# Tolerances, in units of U16 * max|V| of the case.  The output is a convex combination of V rows, so every error
# source scales with max|V|: the fp16 rounding of the output (at most U16 |out|), the fp16 rounding of P (each
# probability within U16 relative; the fused kernel normalises by the fp32 sum of the unrounded ones, the unfused path
# rounds the already normalised P), ex2.approx / __expf (~2^-22 relative) and fp32 accumulation (~2^-24 per term).
# Worst case ~1.5 units: half an ulp of output rounding plus U16 of P on a row dominated by one or two keys (the large
# magnitudes case).  Largest measured on an H100 (700 W), over both paths, every H and nb, in U16 * max|V| units:
# typical 0.13, sharp 0.025, uniform 0.21, late maximum 0.39, large magnitudes 1.17, offset V 0.94 (of which 0.84 is
# the output rounding at 300); each tolerance is 1.7x to 4x its measurement.
ATTN_TOL = {"typical": 0.4, "sharp": 0.1, "uniform": 0.6, "late_max": 1.0, "large": 2.0, "offset_v": 2.0}
ATTN_CASES = list(ATTN_TOL)
SHARP_KEYS = [0, 127, 128, 1407, 1408, 1499]            # both sides of every key-tile edge, the last key
SHARP_ROWS = [3, 700, 1407, 1408, 1450, 1499]           # three query rows inside the ragged last query tile


def attn_inputs(case, nb, H, seed):
    """Q, K, V [nb, H, 1500, 64] as fp16, plus the planted (row, key) pairs of the sharp case."""
    rng = np.random.default_rng(seed)
    shape = (nb, H, S_ENC, 64)
    Q = rng.standard_normal(shape, dtype=np.float32)
    K = rng.standard_normal(shape, dtype=np.float32)
    V = rng.standard_normal(shape, dtype=np.float32)
    planted = []
    if case == "sharp":
        # small background scores (|s| < ~3); row r_i of every (stream, head) has all its q in coordinate c_i and key
        # k_i a matching entry: scaled score 0.125 * 16 * 20 = 40 against at most a few for every other key
        Q *= 0.25
        K *= 0.25
        for b in range(nb):
            for h in range(H):
                rot = (b + h) % 6
                for i, r in enumerate(SHARP_ROWS):
                    k = SHARP_KEYS[(i + rot) % 6]
                    c = (7 * i + h) % 64
                    Q[b, h, r] = 0.0
                    Q[b, h, r, c] = 16.0
                    K[b, h, k, c] = 20.0
                    planted.append((b, h, r, k))
    elif case == "uniform":
        Q[:] = 0.0                                       # every score 0: the output is the mean of the 1500 V rows
        V += 1.0
    elif case == "late_max":
        # even rows: coordinate 0 adds a scaled score of 0.125 * 8 * 20 = 20 to the keys of the 12th tile only, so the
        # running maximum of tiles 0-10 is ~20 below the one that first shows up in the last tile
        Q[:, :, ::2, 0] = 8.0
        Q[:, :, 1::2, 0] = 0.0
        K[..., 0] = 0.0
        K[:, :, 1408:, 0] = 20.0
    elif case == "large":
        # scaled scores of std ~60 (beyond +-200 at the tails); every third row has all scores negative (~ -250)
        Q *= 8.0
        K = np.abs(K) * 7.5
        Q[:, :, ::3] = -np.abs(Q[:, :, ::3])
    elif case == "offset_v":
        V += 300.0                                       # fp16-P vs fp32-sum normalisation bias shows as 300 x it
    return Q.astype(np.float16), K.astype(np.float16), V.astype(np.float16), planted


def attn_pack(Q, K, V, pad=1e4):
    """qk [nb][1500][2d] (Q | K, head h in columns 64 h ..), vt [nb][d][1536] with the 36 pad columns set to `pad`, and
    the output buffer [nb * 1500 + 128][d] filled with the NaN pattern."""
    nb, H = Q.shape[:2]
    d = 64 * H
    qk = np.concatenate([Q.transpose(0, 2, 1, 3).reshape(nb, S_ENC, d), K.transpose(0, 2, 1, 3).reshape(nb, S_ENC, d)], -1)
    vt = np.full((nb, d, S_PAD), pad, np.float16)
    vt[:, :, :S_ENC] = V.transpose(0, 1, 3, 2).reshape(nb, d, S_ENC)
    out = np.full((nb * S_ENC + 128, d), NAN16, np.uint16).view(np.float16)
    return np.ascontiguousarray(qk), vt, out


def attn_unpack(out, nb, H):
    return out[:nb * S_ENC].reshape(nb, S_ENC, H, 64).transpose(0, 2, 1, 3)


def attn_ref(Q, K, V, b, h):
    q, k, v = (a[b, h].astype(np.float64) for a in (Q, K, V))
    s = 0.125 * (q @ k.T)
    p = np.exp(s - s.max(-1, keepdims=True))
    return (p / p.sum(-1, keepdims=True)) @ v


def check_buffer(out, nb, what):
    """Every row of every stream finite; the 128 guard rows after the last stream untouched."""
    body = out[:nb * S_ENC].astype(np.float32)
    bad = np.flatnonzero(~np.isfinite(body).all(-1))
    assert bad.size == 0, f"{what}: {bad.size} output rows not finite / not written, first (stream, row) {divmod(int(bad[0]), S_ENC)}"
    assert np.all(out[nb * S_ENC:].view(np.uint16) == NAN16), f"{what}: the guard rows after the last stream were written"


def ref_streams(nb, H):
    return list(range(nb)) if nb * H <= 96 else [0, 7, nb - 1]


@pytest.mark.parametrize("nb", [1, 3, 16])
@pytest.mark.parametrize("H", [2, 6, 20])
def test_encoder_attention(H, nb):
    eng = engine()
    d = 64 * H
    rule = 2 if d >= 1024 else 4
    runs = [(0, 0), (1, 0)] + ([(1, 2)] if nb == 3 and rule != 2 else [])   # (path, ab): nb 3 at ab 2 -> ragged chunk
    for case in ATTN_CASES:
        Q, K, V, planted = attn_inputs(case, nb, H, seed=zlib.crc32(f"{case}/{nb}/{H}".encode()))
        qk, vt, buf = attn_pack(Q, K, V)
        unit = U16 * float(np.abs(V.astype(np.float32)).max())
        tol = ATTN_TOL[case] * unit
        streams = ref_streams(nb, H)
        refs = {(b, h): attn_ref(Q, K, V, b, h) for b in streams for h in range(H)}
        outs = {}
        for path, ab in runs:
            what = f"{case} H={H} nb={nb} path={'fused' if path == 0 else f'unfused ab={ab or rule}'}"
            raw = eng.test_enc_attn(qk, vt, buf, path, ab)
            check_buffer(raw, nb, what)
            got = attn_unpack(raw, nb, H)
            outs[(path, ab)] = got
            err = max(float(np.abs(got[b, h].astype(np.float64) - r).max()) for (b, h), r in refs.items())
            print(f"attention {what}: max err {err:.3e} = {err / unit:.3f} U16 max|V| (tol {ATTN_TOL[case]})")
            for (b, h), r in refs.items():
                e = np.abs(got[b, h].astype(np.float64) - r)
                assert e.max() <= tol, f"{what}: stream {b} head {h}: max err {e.max():.3e} at row {int(e.max(1).argmax())} (tol {tol:.3e})"
            for b, h, r, k in planted:      # P is exactly 1 at the planted key and underflows to 0 everywhere else
                assert np.array_equal(got[b, h, r].view(np.uint16), V[b, h, k].view(np.uint16)), \
                    f"{what}: stream {b} head {h} row {r}: not bit-identical to V row {k}"
        if nb > 1:
            fused = outs[(0, 0)]
            # the fused kernel: one CTA per (query tile, head, stream), so a stream's output cannot depend on its batch
            for b in range(nb):
                qs, vs, bs = attn_pack(Q[b:b + 1], K[b:b + 1], V[b:b + 1])
                alone = attn_unpack(eng.test_enc_attn(qs, vs, bs, 0, 0), 1, H)[0]
                assert np.array_equal(alone.view(np.uint16), fused[b].view(np.uint16)), \
                    f"{case} H={H} nb={nb}: fused stream {b} differs from the same stream launched alone"
            # the unfused path on streams without a float64 reference: within the tolerance of the fused result
            # (which the bit-identity above ties to the stream's own solo launch)
            rest = [b for b in range(nb) if b not in streams]
            for key, got in outs.items():
                if key[0] == 1 and rest:
                    e = np.abs(got[rest].astype(np.float64) - fused[rest].astype(np.float64)).max()
                    assert e <= 2 * tol, f"{case} H={H} nb={nb} unfused ab={key[1]}: {e:.3e} from the fused result"


def test_encoder_attention_refuses_bad_arguments():
    from whisperlive_b200._lib import WlError
    Q, K, V, _ = attn_inputs("typical", 1, 2, seed=1)
    qk, vt, buf = attn_pack(Q, K, V)
    for path, ab in ((2, 0), (-1, 0), (1, -1)):
        with pytest.raises(WlError, match="bad arguments"):
            engine().test_enc_attn(qk, vt, buf, path, ab)


# --------------------------------------------------------------------------------------- conv stem
# Tolerance, relative to sum_k |conv2 input x weight| of the output element: the fp32 accumulation over K = 3d terms
# (<= ~K 2^-24 in the worst case, ~sqrt(K) 2^-24 typically) plus the occasional 1-ulp flip of an fp16 conv1 output whose
# fp32 value sat at a rounding midpoint (one term off by U16 relative).  Largest measured on an H100 (700 W): 2.2e-5 at
# d 384, 7.4e-6 at d 1280 (in those units); set at about 3x the larger.
STEM_TOL = 6e-5
_STEM = {}


def stem_engine(n_mels, d):
    if (n_mels, d) not in _STEM:
        from whisperlive_b200.engine import B200Whisper
        from whisperlive_b200.weights import random_init
        dims = WhisperDims(f"stem{n_mels}", d, d // 64, 1, 1, n_mels, 51866 if n_mels == 128 else 51864)
        w = random_init(dims, seed=3)
        _STEM[(n_mels, d)] = (B200Whisper(dims, w, max_streams=1, max_beam=1), w)
    return _STEM[(n_mels, d)]


def stem_windows(n_mels, nb):
    """log-mel windows of speech-like audio (1.2 s, 7.3 s, 30 s) and one with a strong impulse in frames 0 and 2999."""
    from oracle import mel as omel
    from whisperlive_b200 import synth
    out = []
    for i in range(nb):
        kind = i % 4
        secs = (1.2, 7.3, 30.0, 7.3)[kind]
        f = omel.pad_or_trim(omel.log_mel(synth.speech_like(secs, seed=60 + i), n_mels)[:, :-1])
        if kind == 3:
            f = f.copy()
            f[:, 0] = 6.0
            f[:, 2999] = -5.0 + 3.0 * np.sin(np.arange(n_mels))
        out.append(f.astype(np.float32))
    return np.stack(out)


def gelu(z):
    return 0.5 * z * (1 + erf(z / np.sqrt(2)))


def conv_k3(x, w, stride):
    """conv1d, kernel 3, padding 1: x [T][C] (float64), w [out][C][3] -> ([T_out][out], sum |terms|)."""
    T = x.shape[0]
    xp = np.zeros((T + 2, x.shape[1]))
    xp[1:T + 1] = x
    n = (T - 1) // stride + 1
    cols = np.concatenate([xp[k:k + stride * (n - 1) + 1:stride] for k in range(3)], 1)    # [n][3 C]: tap-major
    wk = w.transpose(0, 2, 1).reshape(w.shape[0], -1)                                      # [out][3 C]
    return cols @ wk.T, np.abs(cols) @ np.abs(wk).T


@pytest.mark.parametrize("nb", [1, 16])
@pytest.mark.parametrize("n_mels,d", [(80, 384), (128, 1280)])
def test_conv_stem(n_mels, d, nb):
    eng, w = stem_engine(n_mels, d)
    # the conv weights as the engine holds them (fp16); biases and the positional table stay fp32
    w1, w2 = (w[f"model.encoder.{k}.weight"].numpy().astype(np.float16).astype(np.float64) for k in ("conv1", "conv2"))
    b1, b2 = (w[f"model.encoder.{k}.bias"].numpy().astype(np.float32).astype(np.float64) for k in ("conv1", "conv2"))
    pos = w["model.encoder.embed_positions.weight"].numpy().astype(np.float32).astype(np.float64)
    feats = stem_windows(n_mels, nb)
    got = eng.test_enc_stem(feats)
    worst = 0.0
    for b in range(nb):
        y1, _ = conv_k3(feats[b].astype(np.float16).astype(np.float64).T, w1, 1)
        c1 = gelu(y1 + b1).astype(np.float16).astype(np.float64)        # conv1o is fp16
        y2, mag = conv_k3(c1, w2, 2)
        ref = gelu(y2 + b2) + pos
        rel = np.abs(got[b].astype(np.float64) - ref) / mag
        worst = max(worst, float(rel.max()))
        for name, sl in (("frame 0", slice(0, 1)), ("frame 1499", slice(1499, 1500)), ("interior", slice(1, 1499))):
            e = float(rel[sl].max())
            assert e <= STEM_TOL, f"n_mels {n_mels} d {d} nb {nb} stream {b} {name}: {e:.2e} (tol {STEM_TOL})"
    print(f"conv stem n_mels {n_mels} d {d} nb {nb}: max err {worst:.2e} of sum |terms|")


# --------------------------------------------------------------------------------------- layernorm_rows
# y16: within one fp16 ulp of fp16(float64 LN) -- the kernel rounds its fp32 result once.  y32: within 1e-5 of the
# magnitude of its terms (|gamma z| + |beta|); rsqrtf and the fp32 arithmetic are ~1e-7 relative.  On top of both, the
# conditioning of the input: the row mean is summed in fp32, so it is off by a few 2^-24 mean|x|, which LayerNorm
# divides by the row's std.  For rows of mean 1e3 and std 0.1 that is ~1e-3 absolute, whatever the kernel does short
# of wider sums; LN_COND bounds it in units of 2^-24 |gamma| mean|x| / std (largest measured on an H100 (700 W): 3.1,
# at d 1280 and 24000 rows; set at about 2x).  For the N(0, 1) and 1e4-magnitude rows the term is ~1e-7 and the 1-ulp / 1e-5 criteria bind.
LN_COND = 6.0
LN_ROWS = [1, 7, 8, 9, 24000]        # 24000 = the encoder's 16 streams x 1500 rows
LN_D = [128, 384, 512, 768, 1024, 1280]


def ln_inputs(rows, d, rng):
    """Row kinds by index: 0 N(0, 1); 1 mean 1e3, std 0.1; 2 magnitude 1e4; 3 exactly constant (sums exact in fp32)."""
    x = rng.standard_normal((rows, d), dtype=np.float32)
    kind = np.arange(rows) % 4
    x[kind == 1] = np.float32(1e3) + np.float32(0.1) * x[kind == 1]
    x[kind == 2] *= np.float32(1e4)
    consts = np.array([2.5, -1024.0, 0.0, 7.0], np.float32)
    x[kind == 3] = consts[(np.arange(rows)[kind == 3] // 4) % 4][:, None]
    return x, kind


@pytest.mark.parametrize("d", LN_D)
@pytest.mark.parametrize("rows", LN_ROWS)
def test_layernorm_rows(rows, d):
    eng = engine()
    rng = np.random.default_rng(rows * 7 + d)
    x, kind = ln_inputs(rows, d, rng)
    gamma = (1 + 0.3 * rng.standard_normal(d)).astype(np.float32)
    beta = (0.5 * rng.standard_normal(d)).astype(np.float32)
    nan = np.full((rows + 8, d), np.nan, np.float32)
    y16, y32 = eng.test_layernorm(x, gamma, beta, nan, nan)
    for name, y in (("y16", y16), ("y32", y32)):
        assert np.all(np.isnan(y[rows:])), f"{name}: the guard rows after the last row were written"
        assert np.all(np.isfinite(y[:rows])), f"{name}: rows not written"
    y16, y32 = y16[:rows].astype(np.float64), y32[:rows].astype(np.float64)
    x64 = x.astype(np.float64)
    mu = x64.mean(-1, keepdims=True)
    sd = np.sqrt(((x64 - mu) ** 2).mean(-1, keepdims=True))
    z = (x64 - mu) / np.sqrt(sd ** 2 + 1e-5)
    ref = z * gamma + beta
    cond = LN_COND * 2.0 ** -24 * np.abs(gamma) * np.abs(x64).mean(-1, keepdims=True) / np.maximum(sd, 1e-30)
    cond[kind == 3] = 0.0
    r16 = ref.astype(np.float16)
    ulp = np.spacing(np.abs(r16)).astype(np.float64)
    e16 = np.abs(y16 - r16.astype(np.float64)) - cond
    e32 = np.abs(y32 - ref) - cond
    mag = np.abs(gamma * z) + np.abs(beta)
    big = kind == 1
    cond_units = float((np.abs(y32 - ref)[big] / (cond[big] / LN_COND)).max()) if big.any() else 0.0
    print(f"layernorm rows {rows} d {d}: y16 max {float((np.abs(y16 - r16)[~big] / ulp[~big]).max()):.1f} ulp, "
          f"y32 max rel {float((np.abs(y32 - ref) / mag)[~big].max()):.2e}; rows of mean 1e3: {cond_units:.2f} (LN_COND units)")
    assert np.all(e16 <= ulp), f"y16 more than 1 ulp off, row {int(np.argmax((e16 - ulp).max(1)))}"
    assert np.all(e32 <= 1e-5 * mag), f"y32 beyond 1e-5 relative, row {int(np.argmax((e32 - 1e-5 * mag).max(1)))}"
    const = kind == 3
    assert np.array_equal(y32[const], np.broadcast_to(beta, (int(const.sum()), d))), "a constant row's y32 is not beta"
    assert np.array_equal(y16[const].astype(np.float16).view(np.uint16),
                          np.broadcast_to(beta.astype(np.float16), (int(const.sum()), d)).view(np.uint16)), \
        "a constant row's y16 is not fp16(beta)"
    if rows == 9:   # either output alone
        a16, none = eng.test_layernorm(x, gamma, beta, nan, None)
        none2, a32 = eng.test_layernorm(x, gamma, beta, None, nan)
        assert none is None and none2 is None
        assert np.array_equal(a16[:rows], y16.astype(np.float32)) and np.array_equal(a32[:rows], y32.astype(np.float32))


def test_layernorm_rows_refuses_unsupported_widths():
    from whisperlive_b200._lib import WlError
    for d in (130, 1284, 1536):
        x = np.ones((2, d), np.float32)
        g = np.ones(d, np.float32)
        with pytest.raises(WlError, match="unsupported width"):
            engine().test_layernorm(x, g, g, np.zeros((10, d), np.float32), None)


# --------------------------------------------------------------------------------------- the encoder at the benchmark's batch
def test_encoder_at_the_benchmark_encoder_batch():
    """A 2-layer large-v3-shaped model (d 1280, 20 heads, 128 mels) with max_streams=17: 17 windows encode as a pass of
    16 streams (M = 24000 rows per GEMM, a 12 x 20 x 16 flash-attention grid) and a pass of 1.  Every stream is held to
    the large-v3 encoder bounds against the oracle; streams 0, 15 and 16 encoded alone agree with the batched result."""
    if os.environ.get("WLB200_ENC_BATCH"):
        pytest.skip("WLB200_ENC_BATCH is set: the encoder batch is read once per process and this test needs the default 16")
    from oracle.engine import OracleWhisper
    from whisperlive_b200 import synth
    from whisperlive_b200.engine import B200Whisper
    from whisperlive_b200.weights import random_init
    from tests.test_gpu_parity import feats_for
    dims = WhisperDims("large-v3-2L", 1280, 20, 2, 1, 128, 51866)
    w = random_init(dims, seed=6)
    eng, orc = B200Whisper(dims, w, max_streams=17, max_beam=1), OracleWhisper(w, dims)
    durs = [1.0 + 29.0 * i / 16 for i in range(17)]
    feats = np.stack([feats_for(dims, t, 700 + i) for i, t in enumerate(durs)])
    enc = eng.encode(feats)
    got = np.asarray(enc)
    enc.release()
    ref = orc.encode(feats).enc.numpy()
    for b in range(17):
        err = np.abs(got[b] - ref[b])
        rel_rms = float(np.sqrt((err ** 2).mean() / (ref[b] ** 2).mean()))
        tiles = [float(err[t * 128:(t + 1) * 128].max()) for t in range(12)]
        print(f"encoder 16+1 stream {b} ({durs[b]:.1f} s): max err {err.max():.4f} rel rms {rel_rms:.5f}")
        assert err.max() < 0.06 and rel_rms < 0.008, (b, float(err.max()), rel_rms)
        assert max(tiles) < 0.08, (b, tiles)
    for b in (0, 15, 16):
        alone = eng.encode(feats[b:b + 1])
        e = float(np.abs(np.asarray(alone)[0] - got[b]).max())
        alone.release()
        print(f"stream {b} alone vs batched: {e:.2e}")
        assert e < 2e-3, (b, e)
