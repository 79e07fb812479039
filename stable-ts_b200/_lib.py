"""ctypes binding of libstablets_b200.so (declared in include/stablets_b200.h).

There is NO fallback: if the CUDA library is missing or a call fails, this raises.  PyTorch is used only to own
device memory and streams.
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int32, c_longlong, c_size_t, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libstablets_b200.so")

STB_PREC_FP16, STB_PREC_FP16X3 = 1, 3
STB_ACT_NONE, STB_ACT_GELU = 0, 1
N_FRAMES, N_AUDIO_CTX, KPAD = 3000, 1500, 1504

# tensor ids (include/stablets_b200.h)
(T_ENC_CONV1_W, T_ENC_CONV1_B, T_ENC_CONV2_W, T_ENC_CONV2_B, T_ENC_POS, T_ENC_LNPOST_G, T_ENC_LNPOST_B,
 T_DEC_TOKEMB_F32, T_DEC_TOKEMB, T_DEC_POS, T_DEC_LN_G, T_DEC_LN_B) = range(12)
T_LAYER_BASE = 32
(L_ATTN_LN_G, L_ATTN_LN_B, L_QKV_W, L_QKV_B, L_OUT_W, L_OUT_B, L_MLP_LN_G, L_MLP_LN_B, L_FC1_W, L_FC1_B, L_FC2_W,
 L_FC2_B, L_CROSS_LN_G, L_CROSS_LN_B, L_CQ_W, L_CQ_B, L_CKV_W, L_CKV_B, L_COUT_W, L_COUT_B, L_COUNT) = range(21)


class Operand(ctypes.Structure):
    _fields_ = [("hi", c_void_p), ("lo", c_void_p), ("rows", c_int), ("k", c_int), ("row_stride", c_longlong),
                ("h_stride", c_longlong), ("b_stride", c_longlong)]


class Epilogue(ctypes.Structure):
    _fields_ = [("out_f32", c_void_p), ("out_hi", c_void_p), ("out_lo", c_void_p), ("ld_out", c_longlong),
                ("out_h_stride", c_longlong), ("out_b_stride", c_longlong), ("transposed", c_int), ("bias", c_void_p),
                ("bias_per_row", c_int), ("residual", c_void_p), ("ld_res", c_longlong), ("res_h_stride", c_longlong),
                ("res_b_stride", c_longlong), ("alpha", c_float), ("act", c_int)]


class Dims(ctypes.Structure):
    _fields_ = [(n, c_int) for n in ("n_mels", "n_audio_ctx", "n_audio_state", "n_audio_head", "n_audio_layer",
                                     "n_vocab", "n_text_ctx", "n_text_state", "n_text_head", "n_text_layer")]


_SIGS = {
    "stb_last_error": (c_char_p, []),
    "stb_abi_version": (c_int, []),
    "stb_launch_count": (ctypes.c_ulonglong, []),
    "stb_prof_enable": (None, [c_int]),
    "stb_prof_report": (c_int, [ctypes.c_char_p, c_size_t]),
    "stb_logmel": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                           c_size_t, c_void_p]),
    "stb_gemm": (c_int, [POINTER(Operand), POINTER(Operand), c_int, c_int, POINTER(Epilogue), c_void_p]),
    "stb_attention": (c_int, [POINTER(Operand), POINTER(Operand), POINTER(Operand), c_int, c_int, c_int, c_int, c_void_p,
                              c_void_p, c_longlong, c_longlong, c_longlong, c_void_p]),
    "stb_silence_mask": (c_int, [c_void_p, c_int, c_int, c_longlong, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                 c_void_p, c_void_p]),
    "stb_resample_mono": (c_int, [c_void_p, c_int, c_int, c_longlong, c_int, c_int, c_void_p, c_int, c_void_p, c_longlong, c_int,
                                  c_void_p]),
    "stb_gemv": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_longlong,
                         c_void_p, c_void_p, c_void_p, c_longlong, c_void_p]),
    "stb_decode_linear": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p,
                                  c_longlong, c_void_p, c_void_p, c_void_p, c_longlong, c_void_p]),
    "stb_decode_linear_split": (c_int, [c_int, c_int]),
    "stb_split_f16": (c_int, [c_void_p, c_longlong, c_int, c_longlong, c_void_p, c_void_p, c_longlong, c_void_p]),
    "stb_model_create": (c_int, [POINTER(Dims), c_int, POINTER(c_void_p)]),
    "stb_model_destroy": (None, [c_void_p]),
    "stb_model_set_tensor": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "stb_encoder_ws_bytes": (c_size_t, [c_void_p, c_int]),
    "stb_encoder_forward": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "stb_cross_kv_bytes": (c_size_t, [c_void_p, c_int]),
    "stb_cross_kv": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "stb_decoder_ws_bytes": (c_size_t, [c_void_p, c_int, c_int]),
    "stb_decoder_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_longlong, c_void_p,
                                    POINTER(c_int32), c_int, c_void_p, c_size_t, c_void_p]),
    "stb_token_probs": (c_int, [c_void_p, c_longlong, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "stb_softmax_probs": (c_int, [c_void_p, c_longlong, c_int, c_int, c_void_p, c_longlong, c_void_p]),
    "stb_qkpost_ws_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "stb_qk_postprocess": (c_int, [c_void_p, c_int, c_int, c_int, c_longlong, c_int, c_int, c_int, c_float, c_int, c_void_p,
                                   c_longlong, c_void_p, c_size_t, c_void_p]),
    "stb_decode_state_bytes": (c_size_t, [c_void_p, c_int]),
    "stb_decode_ws_bytes": (c_size_t, [c_void_p, c_int]),
    "stb_decode_step": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_void_p,
                                c_size_t, c_void_p]),
    "stb_sample_greedy": (c_int, [c_void_p, c_longlong, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                  c_longlong, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "stb_decode_state_bytes_rows": (c_size_t, [c_void_p, c_int, c_int]),
    "stb_decode_step_ragged": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                       c_longlong, c_void_p, c_size_t, c_void_p]),
    "stb_decode_self_attn": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p]),
    "stb_decode_cross_attn": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_void_p]),
    "stb_decode_cross_splits": (c_int, []),
    "stb_layernorm": (c_int, [c_void_p, c_longlong, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "stb_softmax_rows": (c_int, [c_void_p, c_longlong, c_int, c_longlong, c_int, c_int, c_void_p, c_void_p, c_longlong,
                                 c_void_p]),
    "stb_sample": (c_int, [c_void_p, c_longlong, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                           c_longlong, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_void_p,
                           c_void_p, c_void_p]),
    "stb_qkpost_dynamic_ws_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "stb_qk_postprocess_dynamic": (c_int, [c_void_p, c_int, c_int, c_int, c_longlong, c_int, c_int, c_int, c_float, c_int, c_int,
                                           c_void_p, c_int, c_void_p, c_longlong, c_void_p, c_size_t, c_void_p]),
    "stb_qkpost_new_ws_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "stb_qk_postprocess_new": (c_int, [c_void_p, c_int, c_int, c_int, c_longlong, c_int, c_int, c_int, c_float, c_int, c_int,
                                       c_float, c_float, c_float, c_void_p, c_longlong, c_void_p, c_size_t, c_void_p]),
    "stb_axpby": (c_int, [c_void_p, c_void_p, c_float, c_float, c_longlong, c_void_p]),
    "stb_dtw_smem_bytes": (c_size_t, [c_int, c_int]),
    "stb_dtw_ws_bytes": (c_size_t, [c_int, c_int, c_int]),
    "stb_dtw": (c_int, [c_void_p, c_int, c_int, c_int, c_longlong, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                        c_void_p]),
}

_lib = None


def exported_symbols():
    """Names include/stablets_b200.h declares (used by the CPU-side ABI test)."""
    return sorted(_SIGS)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python stable-ts_b200/build.py` (there is no CPU fallback)")
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


class StbError(RuntimeError):
    pass


def check(rc: int):
    if rc != 0:
        raise StbError(f"libstablets_b200 error {rc}: {lib().stb_last_error().decode(errors='replace')}")


def get_option(name: str) -> int:
    """-1 for every name: the library has no kernel-variant switches; kept for callers that report option values."""
    return -1


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    return None if t is None else c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def prof_report() -> dict:
    """Per-kernel event-timed totals since the last call (see stb_prof_report)."""
    import json
    buf = ctypes.create_string_buffer(1 << 16)
    check(lib().stb_prof_report(buf, len(buf)))
    return json.loads(buf.value.decode())


def device_ctx(device):
    """``torch.cuda.device(device)`` for a CUDA device; a no-op context for anything else (the CPU stand-in of the tests)."""
    import contextlib
    import torch
    device = torch.device(device)
    return torch.cuda.device(device) if device.type == "cuda" else contextlib.nullcontext()
