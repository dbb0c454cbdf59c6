"""CPU: the C-ABI library loads and exports every symbol include/mvb200.h declares (no compute calls)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "mvb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mvb_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_boundary():
    names = _declared()
    for must in ("mvb_s1_create", "mvb_s1_forward", "mvb_s1_sample", "mvb_s1_generate", "mvb_s1_decode",
                 "mvb_last_error"):
        assert must in names


def test_library_exports_every_declared_symbol():
    from mvb200 import _lib
    if not os.path.isfile(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in _declared():
        assert hasattr(lib, name), f"{name} declared in include/mvb200.h but not exported"
    assert set(_declared()) == set(_lib.SIGNATURES), "python binding table out of sync with the header"
    for hook in ("mvb_gemm_test", "mvb_mbd_conv_test", "mvb_s2_attn_test", "mvb_s2_sample_test", "mvb_voc_op_test",
                 "mvb_audio_post_test"):
        assert hook in _lib.SIGNATURES and hasattr(lib, hook), f"test hook {hook} missing"
    assert lib.mvb_abi_version() == _lib.ABI_VERSION == 2


def test_config_validation_without_gpu():
    from mvb200 import _lib
    lib = _lib.load()
    ok = _lib.S1Config(24, 16, 128, 2048, 5632, 2562, 2048, 256, 1e-5, 1, 0, 2048)
    # 24 layers x {K,V} x 2 rows x 16 heads x 2048 slots x 128 x 2 B = 805,306,368 (SURVEY.md D5)
    assert lib.mvb_s1_kv_bytes(ctypes.byref(ok)) == 805306368
    assert lib.mvb_s1_workspace_bytes(ctypes.byref(ok)) > 0
    bad = _lib.S1Config(24, 16, 64, 1024, 5632, 2562, 2048, 256, 1e-5, 1, 0, 2048)
    assert lib.mvb_s1_kv_bytes(ctypes.byref(bad)) == 0
    assert b"head_dim" in lib.mvb_last_error()


def test_missing_library_fails_loudly(monkeypatch):
    from mvb200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libmvb200.so")
    with pytest.raises(_lib.MvbError, match="no CPU or PyTorch fallback"):
        _lib.load()
