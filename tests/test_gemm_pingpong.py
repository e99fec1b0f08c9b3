"""The ping-pong wgmma GEMM (csrc/gemm.cu::gemm_pingpong_kernel) against the CUDA-core checker and against the classic
kernel, forced through the test hook on the same inputs.  The two tensor-core kernels run the same m64n128k16
sequence and the same epilogue arithmetic for every output element, so their results must be bit-identical."""
import numpy as np
import pytest
import torch

from whisperlive_b200.config import dims_for

pytestmark = pytest.mark.gpu

_ENG = []


def engine():
    if not _ENG:
        from whisperlive_b200.engine import B200Whisper
        from whisperlive_b200.weights import random_init
        dims = dims_for("micro.en")
        _ENG.append(B200Whisper(dims, random_init(dims, seed=0), max_streams=1, max_beam=1))
    return _ENG[0]


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def tiles(M, N, Z=1):
    return -(-M // 128) * -(-N // 128) * Z


def cases():
    s = sms()
    return [
        # id, Z, M, N, K, hook kwargs (besides the operands)
        ("qk_f16_bias", 1, 6000, 2560, 1280, dict(out="f16", bias="n")),
        ("fc2_f32_resid", 1, 4500, 1280, 5120, dict(out="resid", bias="n")),
        ("fc1_f16_gelu", 1, 2000, 2560, 640, dict(out="f16", bias="n", gelu=True)),
        # 3 tiles per CTA (one warpgroup gets one tile fewer), ragged M tail and an N tail of whole 8-column pieces
        ("odd_tiles_ragged", 1, 128 * s - 37, 360, 256, dict(out="f32", bias="n")),
        # N not a multiple of 8: element-wise (column) epilogue
        ("ragged_col_store", 1, 128 * s - 5, 357, 192, dict(out="f32", bias="n")),
        # V^T of the encoder: W shared by the batch, bias on m, rows of the batch entries
        ("vt_batched_bias_m", 3, 1280, 1500, 1280, dict(out="f16", bias="m", a_shared=True)),
        # conv stem: batched activations, weight shared, bias + GELU
        ("conv_batched", 2, 3000, 1280, 384, dict(out="f16", bias="n", gelu=True, b_shared=True)),
        # cross-attention K/V straight into the slot pool
        ("cross_kv_headsplit", 1, 4 * 1500, 1280, 1280, dict(out="headsplit", bias="n", hs_rows=1500)),
    ]


CASE_IDS = ["qk_f16_bias", "fc2_f32_resid", "fc1_f16_gelu", "odd_tiles_ragged", "ragged_col_store", "vt_batched_bias_m",
            "conv_batched", "cross_kv_headsplit"]


@pytest.mark.parametrize("case_id", CASE_IDS)
def test_pingpong_matches_classic_and_simt(case_id):
    eng = engine()
    _, Z, M, N, K, kw = next(c for c in cases() if c[0] == case_id)
    kw = dict(kw)
    rng = np.random.default_rng(sum(map(ord, case_id)))
    a_shared, b_shared = kw.pop("a_shared", False), kw.pop("b_shared", False)
    a = rng.standard_normal((M, K) if a_shared else (Z, M, K)).astype(np.float16)
    b = rng.standard_normal((N, K) if b_shared else (Z, N, K)).astype(np.float16)
    bias_kind = kw.pop("bias")
    bias = rng.standard_normal(M if bias_kind == "m" else N).astype(np.float32)
    if kw["out"] == "resid":
        kw["resid"] = rng.standard_normal((Z, M, N)).astype(np.float32)
    kw.update(bias_on_m=bias_kind == "m", batch=Z if (a_shared or b_shared) else None)
    assert tiles(M, N, Z) >= 2 * sms() and eng.gemm_variant(M, N, K, Z) == "pingpong"
    simt = eng.test_gemm(a, b, bias, use_simt=True, **kw)
    classic = eng.test_gemm(a, b, bias, variant="classic", **kw)
    pp = eng.test_gemm(a, b, bias, variant="pingpong", **kw)
    auto = eng.test_gemm(a, b, bias, **kw)
    tol = dict(atol=2e-3 * np.sqrt(K), rtol=1e-3)
    print(f"{case_id}: max |pingpong - simt| {np.abs(pp - simt).max():.3e}")
    np.testing.assert_allclose(pp, simt, **tol)
    np.testing.assert_allclose(classic, simt, **tol)
    assert np.array_equal(pp.view(np.uint32), classic.view(np.uint32)), "ping-pong and classic kernels differ"
    assert np.array_equal(auto.view(np.uint32), pp.view(np.uint32))
    if kw["out"] == "headsplit":   # every element of every slot was written
        assert np.count_nonzero(pp) > 0.99 * pp.size


def test_encoder_shapes_select_pingpong():
    """Every GEMM of a 16-stream large-v3 encoder pass (and the cross-KV projections) takes the ping-pong kernel;
    small problems keep the classic one."""
    eng = engine()
    d, ff, S, nb, nm = 1280, 5120, 1500, 16, 128
    M = nb * S
    encoder = [(3000, d, 3 * nm, nb), (S, d, 3 * d, nb), (M, 2 * d, d, 1), (d, S, d, nb), (M, d, d, 1), (M, ff, d, 1),
               (M, d, ff, 1)]
    for shape in encoder:
        assert eng.gemm_variant(*shape) == "pingpong", shape
    for shape in [(384, 3 * d, d, 1), (3840, 16, 1280, 1), (1500, 64, 1536, 40), (128, 128, 64, 1)]:
        assert eng.gemm_variant(*shape) == "classic", shape
