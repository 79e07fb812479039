"""CPU-side checks of the drop-in boundary: the C-ABI library builds for sm_90a, loads without a GPU and exports
every symbol include/stablets_b200.h declares (no compute calls here)."""
import ctypes
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "stablets_b200.h")).read()
    return sorted(set(re.findall(r"STB_API[^;(]*?\b(stb_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_declared_symbols():
    import importlib.util
    spec = importlib.util.spec_from_file_location("stb_build", os.path.join(ROOT, "stable-ts_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    so = mod.build()
    assert os.path.exists(so)
    lib = ctypes.CDLL(so)
    names = _declared()
    assert len(names) >= 19
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/stablets_b200.h but not exported"
    lib.stb_abi_version.restype = ctypes.c_int
    assert lib.stb_abi_version() >= 1


def test_python_binding_covers_header():
    from stable_ts_b200 import _lib
    assert sorted(_lib.exported_symbols()) == _declared()


def test_sass_has_hopper_tensor_and_tma_instructions():
    so = os.path.join(ROOT, "stable-ts_b200", "libstablets_b200.so")
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    assert "HGMMA" in out and "UTMALDG" in out and "sm_90a" in out


def test_product_path_fails_loudly_without_cuda():
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from stable_ts_b200.model import B200Whisper
    with pytest.raises(RuntimeError):
        B200Whisper(None, {}, device="cuda")


def test_error_reporting_without_a_gpu():
    """stb_last_error works without a device: argument errors are reported with a message before any CUDA call.  The library
    has no kernel-variant switches; _lib.get_option reads -1 for every name, the removed "decode_fused_ln" and the older
    "xattn_tc", "decode_splitk_legacy" and "decode_lin_priority" among them (bench.py reports these)."""
    from stable_ts_b200 import _lib as L
    lib = L.lib()
    assert lib.stb_abi_version() >= 7
    for name in ("decode_fused_ln", "no_such_option", "xattn_tc", "decode_splitk_legacy", "decode_lin_priority"):
        assert L.get_option(name) == -1
    # argument validation happens before any CUDA call
    assert lib.stb_decode_state_bytes(None, 4) == 0 and lib.stb_decode_ws_bytes(None, 4) == 0
    assert lib.stb_axpby(None, None, 1.0, 0.0, 8, None) != 0 and b"stb_axpby" in lib.stb_last_error()
    assert lib.stb_decode_linear(None, None, 48, 100, None, None, 1280, None, 0, None, 0, None, None, None, 1280,
                                 None) != 0 and b"K=100" in lib.stb_last_error()
    assert lib.stb_decode_self_attn(None, None, None, 4, 0, 448, None, None, None, None, None, None) != 0
    assert b"stb_decode_self_attn: H=0" in lib.stb_last_error()
    assert lib.stb_decode_cross_attn(None, None, None, 0, 20, None, None, None, None, None, None) != 0
    assert b"stb_decode_cross_attn: B=0" in lib.stb_last_error()
    assert lib.stb_decode_cross_splits() >= 1
    assert lib.stb_layernorm(None, 8, 1408, None, None, None, None, None, None) != 0
    assert b"stb_layernorm: d=1408" in lib.stb_last_error()
    assert lib.stb_softmax_rows(None, 8, 1500, 1504, 1, 0, None, None, 1496, None) != 0
    assert b"stb_softmax_rows: ld_p=1496" in lib.stb_last_error()
