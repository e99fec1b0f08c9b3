"""ctypes binding of libwlb200.so (the C ABI in include/wlb200.h).

There is no CPU fallback: if the shared library cannot be loaded (or built with nvcc) the import
of anything that needs it raises."""
from __future__ import annotations

import ctypes as C
import os
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libwlb200.so")
ABI_VERSION = 14

c_i32p = C.POINTER(C.c_int32)
c_i64p = C.POINTER(C.c_int64)
c_f32p = C.POINTER(C.c_float)
c_u16p = C.POINTER(C.c_uint16)


class WlConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("device", C.c_int32),
        ("d_model", C.c_int32), ("n_heads", C.c_int32), ("enc_layers", C.c_int32), ("dec_layers", C.c_int32),
        ("n_mels", C.c_int32), ("vocab", C.c_int32),
        ("eot", C.c_int32), ("sot", C.c_int32), ("no_speech", C.c_int32), ("no_timestamps", C.c_int32),
        ("timestamp_begin", C.c_int32), ("blank", C.c_int32), ("lang_begin", C.c_int32), ("n_lang", C.c_int32),
        ("max_streams", C.c_int32), ("max_beam", C.c_int32), ("enc_slots", C.c_int32),
        ("n_align_heads", C.c_int32), ("align_heads", c_i32p),
    ]


class WlGenOpts(C.Structure):
    _fields_ = [
        ("beam_size", C.c_int32), ("patience", C.c_float), ("num_hypotheses", C.c_int32), ("length_penalty", C.c_float),
        ("max_length", C.c_int32), ("suppress_blank", C.c_int32), ("max_initial_timestamp_index", C.c_int32),
        ("sampling_topk", C.c_int32), ("sampling_temperature", C.c_float), ("seed", C.c_uint32),
        ("suppress_tokens", c_i32p), ("n_suppress", C.c_int32), ("use_cuda_graph", C.c_int32),
        ("max_length_per_stream", c_i32p), ("prefill", C.c_int32),
    ]


class WlStreamSearch(C.Structure):
    _fields_ = [
        ("sample", C.c_int32), ("num_hypotheses", C.c_int32), ("temperature", C.c_float), ("seed", C.c_uint32),
        ("noise_key", C.c_int32),
    ]


class WlStreamRules(C.Structure):
    _fields_ = [
        ("rules", C.c_int32), ("beam_size", C.c_int32), ("patience", C.c_float), ("length_penalty", C.c_float),
        ("suppress_blank", C.c_int32), ("max_initial_timestamp_index", C.c_int32), ("suppress_tokens", c_i32p),
        ("n_suppress", C.c_int32),
    ]


class WlMtConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("d_model", C.c_int32), ("n_heads", C.c_int32), ("enc_layers", C.c_int32),
        ("dec_layers", C.c_int32), ("ffn", C.c_int32), ("vocab", C.c_int32), ("max_positions", C.c_int32),
        ("pad_id", C.c_int32), ("embed_scale", C.c_float), ("max_src_tokens", C.c_int32),
    ]


class WlMtOpts(C.Structure):
    _fields_ = [
        ("num_beams", C.c_int32), ("max_length", C.c_int32), ("length_penalty", C.c_float), ("early_stopping", C.c_int32),
        ("decoder_start", C.c_int32), ("eos", C.c_int32), ("forced_bos", C.c_int32), ("forced_eos", C.c_int32),
        ("use_cuda_graph", C.c_int32),
    ]


class WlSearchScript(C.Structure):
    _fields_ = [("seed", C.c_uint32), ("pattern", C.c_int32)]


# name -> (restype, argtypes); every symbol include/wlb200.h declares
SIGNATURES = {
    "wl_init": (C.c_int, [C.POINTER(WlConfig), C.POINTER(C.c_void_p)]),
    "wl_destroy": (None, [C.c_void_p]),
    "wl_last_error": (C.c_char_p, [C.c_void_p]),
    "wl_device_bytes": (C.c_int, [C.c_void_p, c_i64p]),
    "wl_mem_info": (C.c_int, [C.c_int32, c_i64p, c_i64p]),
    "wl_load_tensor": (C.c_int, [C.c_void_p, C.c_char_p, c_f32p, c_i64p, C.c_int32]),
    "wl_load_tensor_typed": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int32, c_i64p, C.c_int32, C.c_void_p,
                                       C.c_int32]),
    "wl_finalize_weights": (C.c_int, [C.c_void_p]),
    "wl_mel": (C.c_int, [C.c_void_p, c_f32p, c_i64p, C.c_int32, c_f32p, c_i64p]),
    "wl_encode": (C.c_int, [C.c_void_p, c_f32p, C.c_int32, c_i32p]),
    "wl_slots_release": (C.c_int, [C.c_void_p, c_i32p, C.c_int32]),
    "wl_slots_free_count": (C.c_int, [C.c_void_p]),
    "wl_encoder_output": (C.c_int, [C.c_void_p, C.c_int32, c_f32p]),
    "wl_generate": (C.c_int, [C.c_void_p, c_i32p, C.c_int32, c_i32p, c_i32p, C.POINTER(WlGenOpts), c_i32p, c_i32p, c_f32p,
                              c_f32p, c_i32p]),
    "wl_session_open": (C.c_int, [C.c_void_p, C.POINTER(WlGenOpts), C.c_int32]),
    "wl_session_admit": (C.c_int, [C.c_void_p, C.c_int32, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p]),
    "wl_session_admit_ex": (C.c_int, [C.c_void_p, C.c_int32, c_i32p, c_i32p, c_i32p, c_i32p, c_i32p,
                                      C.POINTER(WlStreamSearch), C.POINTER(WlStreamRules)]),
    "wl_session_run": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, c_i32p, c_i32p]),
    "wl_session_collect": (C.c_int, [C.c_void_p, C.c_int32, c_i32p, c_i32p, c_f32p, c_f32p, c_i32p]),
    "wl_session_peek": (C.c_int, [C.c_void_p, C.c_int32, c_i32p, c_i32p, c_i32p, c_f32p, c_f32p, c_i32p, c_i32p]),
    "wl_session_cancel": (C.c_int, [C.c_void_p, C.c_int32, c_i32p]),
    "wl_session_close": (C.c_int, [C.c_void_p]),
    "wl_detect_language": (C.c_int, [C.c_void_p, c_i32p, C.c_int32, c_f32p]),
    "wl_align": (C.c_int, [C.c_void_p, c_i32p, C.c_int32, c_i32p, C.c_int32, c_i32p, c_i32p, c_i32p, C.c_int32, c_i32p,
                           C.c_int32, c_i32p, c_f32p]),
    "wl_decode_logits": (C.c_int, [C.c_void_p, c_i32p, C.c_int32, c_i32p, c_i32p, c_f32p]),
    "wl_test_gemm": (C.c_int, [C.c_void_p, c_u16p, c_u16p, c_f32p, c_f32p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                               C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "wl_gemm_variant": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, c_i32p]),
    "wl_test_wgemm": (C.c_int, [C.c_void_p, c_u16p, c_u16p, c_f32p, c_f32p, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "wl_test_dec_gemm": (C.c_int, [C.c_void_p, c_u16p, c_u16p, c_f32p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, c_i32p]),
    "wl_test_cross_attn": (C.c_int, [C.c_void_p, c_f32p, c_f32p, C.c_int32, c_u16p, c_u16p, C.c_int32, c_i32p, c_i32p,
                                     C.c_int32, C.c_int32, C.c_int32, C.c_int32, c_i32p, C.c_float, c_f32p, c_f32p]),
    "wl_test_self_attn": (C.c_int, [C.c_void_p, c_f32p, c_f32p, C.c_int32, c_u16p, c_u16p, C.c_int32, C.POINTER(C.c_int16),
                                    c_i32p, c_i32p, c_i32p, C.c_int32, C.c_int32, C.c_float, c_f32p]),
    "wl_test_fold": (C.c_int, [C.c_void_p, C.c_int32, c_f32p, c_f32p, C.c_int32, c_f32p, c_f32p, c_f32p, c_f32p,
                               C.c_int32, C.c_int32]),
    "wl_test_enc_attn": (C.c_int, [C.c_void_p, c_u16p, c_u16p, c_u16p, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "wl_test_enc_stem": (C.c_int, [C.c_void_p, c_f32p, c_f32p, C.c_int32]),
    "wl_test_read_weight": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p]),
    "wl_test_layernorm": (C.c_int, [C.c_void_p, c_f32p, c_f32p, c_f32p, c_f32p, c_f32p, C.c_int32, C.c_int32]),
    "wl_test_search": (C.c_int, [C.c_void_p, C.c_int32, c_i32p, c_i32p, C.POINTER(WlGenOpts), C.POINTER(WlSearchScript),
                                 c_i32p, c_i32p, c_f32p, c_f32p, c_i32p, c_i32p, c_f32p]),
    "wl_test_session_script": (C.c_int, [C.c_void_p, C.POINTER(WlSearchScript)]),
    "wl_bench_gemm": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, c_f32p]),
    "wl_kernel_launches": (C.c_int64, [C.c_void_p]),
    "wl_last_device_ms": (C.c_float, [C.c_void_p, C.c_int32]),
    "wl_profile_cross_attn": (C.c_int, [C.c_void_p, C.c_int32]),
    "wl_mel_device": (C.c_int, [C.c_void_p, c_f32p, c_i64p, C.c_int32, c_i32p]),
    "wl_encode_windows": (C.c_int, [C.c_void_p, C.c_int32, c_i32p, c_i32p, c_i32p, c_i32p]),
    "wl_mel_resident": (C.c_int, [C.c_void_p]),
    "wl_encode_resident": (C.c_int, [C.c_void_p, C.c_int32, c_i32p]),
    "wl_vad_load_tensor": (C.c_int, [C.c_void_p, C.c_char_p, c_f32p, c_i64p, C.c_int32]),
    "wl_vad": (C.c_int, [C.c_void_p, c_f32p, c_i64p, C.c_int32, c_f32p, c_i64p]),
    "wl_spk_load_tensor": (C.c_int, [C.c_void_p, C.c_char_p, c_f32p, c_i64p, C.c_int32]),
    "wl_spk_embed": (C.c_int, [C.c_void_p, c_f32p, c_i64p, C.c_int32, c_f32p]),
    "wl_test_spk_fbank": (C.c_int, [C.c_void_p, c_f32p, c_i64p, C.c_int32, c_f32p]),
    "wl_test_spk_conv": (C.c_int, [C.c_void_p, c_u16p, c_i64p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                   C.c_int32, c_u16p, c_f32p, c_u16p, C.c_int32, c_u16p]),
    "wl_mt_init": (C.c_int, [C.POINTER(WlMtConfig), C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]),
    "wl_mt_destroy": (None, [C.c_void_p]),
    "wl_mt_last_error": (C.c_char_p, [C.c_void_p]),
    "wl_mt_load_tensor": (C.c_int, [C.c_void_p, C.c_char_p, c_f32p, c_i64p, C.c_int32]),
    "wl_mt_finalize": (C.c_int, [C.c_void_p]),
    "wl_mt_device_bytes": (C.c_int, [C.c_void_p, c_i64p]),
    "wl_mt_translate": (C.c_int, [C.c_void_p, c_i32p, c_i32p, C.c_int32, C.POINTER(WlMtOpts), c_i32p, c_i32p, c_f32p]),
    "wl_test_mt_attn": (C.c_int, [C.c_void_p, c_u16p, c_i32p, C.c_int32, C.c_int32, c_u16p]),
    "wl_test_mt_cross_attn": (C.c_int, [C.c_void_p, c_f32p, c_u16p, C.c_int32, C.c_int32, C.c_int32, c_i32p, C.c_int32,
                                        C.c_int32, C.c_int32, c_u16p]),
    "wl_test_mt_logits": (C.c_int, [C.c_void_p, c_i32p, c_i32p, C.c_int32, c_i32p, C.c_int32, c_f32p]),
    "wl_test_mt_search": (C.c_int, [C.c_void_p, c_f32p, C.c_int32, C.c_int32, C.POINTER(WlMtOpts), c_i32p, c_i32p, c_f32p,
                                    c_i32p]),
}

_lock = threading.Lock()
_lib = None


def load(build_if_missing: bool = True) -> C.CDLL:
    """Load (building first if the .so is absent and nvcc is available). Raises on failure."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            if not build_if_missing:
                raise RuntimeError(f"{LIB_PATH} is missing: run `python -m whisperlive_b200.build`")
            from . import build as _build
            _build.build()
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = lib
        return lib


class WlError(RuntimeError):
    pass


def check(lib, ctx, rc: int, what: str) -> None:
    if rc != 0:
        msg = lib.wl_last_error(ctx)
        raise WlError(f"{what} failed ({rc}): {msg.decode() if msg else '?'}")


def ptr(arr, ctype):
    return arr.ctypes.data_as(C.POINTER(ctype))
