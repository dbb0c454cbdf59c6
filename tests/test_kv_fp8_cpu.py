"""CPU: the fp8 KV cache's size, config validation, Python mapping and quantiser (kv_dtype="fp8", include/mvb200.h at
mvb_s1_kv_bytes).  No device calls."""
import ctypes

import pytest
import torch

from mvb200 import _lib, synth
from mvb200 import quantize as Q


def _cfg(max_utts, kv, d=synth.FULL):
    return _lib.S1Config(d.n_layer, d.n_head, d.head_dim, d.dim, d.intermediate_size, d.vocab_size, d.block_size,
                         d.speaker_emb_dim, d.norm_eps, max_utts, kv, d.block_size)


@pytest.mark.parametrize("max_utts", [1, 8, 64])
def test_kv_bytes_is_the_documented_formula(max_utts):
    lib = _lib.load()
    d = synth.FULL
    n_vec = d.n_layer * 2 * (2 * max_utts) * d.n_head * d.block_size
    got = lib.mvb_s1_kv_bytes(ctypes.byref(_cfg(max_utts, _lib.MVB_KV_FP8)))
    assert got == 128 * n_vec + 2 * n_vec                          # e4m3 codes, then one bf16 scale per head vector
    assert got == 408944640 * max_utts
    bf16 = lib.mvb_s1_kv_bytes(ctypes.byref(_cfg(max_utts, _lib.MVB_KV_BF16)))
    assert bf16 == 805306368 * max_utts


@pytest.mark.parametrize("max_utts", [1, 8, 64])
def test_workspace_bytes_do_not_depend_on_kv_dtype(max_utts):
    lib = _lib.load()
    for fn in (lib.mvb_s1_workspace_bytes, lib.mvb_s1_int4_workspace_bytes, lib.mvb_s1_int8_workspace_bytes,
               lib.mvb_s1_fp8_workspace_bytes):
        a = fn(ctypes.byref(_cfg(max_utts, _lib.MVB_KV_BF16)))
        assert a > 0 and fn(ctypes.byref(_cfg(max_utts, _lib.MVB_KV_FP8))) == a, fn.__name__


def test_validate_accepts_fp8_and_rejects_3():
    lib = _lib.load()
    assert _lib.MVB_KV_FP8 == 2
    assert lib.mvb_s1_kv_bytes(ctypes.byref(_cfg(1, 2))) > 0
    assert lib.mvb_s1_kv_bytes(ctypes.byref(_cfg(1, 3))) == 0
    assert b"kv_dtype" in lib.mvb_last_error()
    assert lib.mvb_s1_workspace_bytes(ctypes.byref(_cfg(1, 3))) == 0


def test_setup_caches_maps_fp8_and_rejects_other_strings(monkeypatch):
    """setup_caches passes "fp8" as MVB_KV_FP8 (the engine creation is intercepted: no device here) and raises ValueError
    for a string it does not know instead of creating a bf16 cache."""
    from mvb200.fast_model import ModelArgs, Transformer
    d = synth.TINY
    m = Transformer.__new__(Transformer)
    m.config = ModelArgs(block_size=d.block_size, vocab_size=d.vocab_size, n_layer=d.n_layer, n_head=d.n_head, dim=d.dim)
    m.quantisation_mode, m._h, m.kv_dtype, m.max_batch_size, m.max_seq_length = None, None, "bf16", -1, -1
    m._lib = _lib.load()
    seen = []
    monkeypatch.setattr(Transformer, "close", lambda self: None)
    monkeypatch.setattr(Transformer, "_create", lambda self, create, destroy, cfg, *a: seen.append(cfg.kv_dtype))
    for s, want in (("fp8", _lib.MVB_KV_FP8), ("bf16", _lib.MVB_KV_BF16), ("fp32", _lib.MVB_KV_FP32)):
        m.setup_caches(2, d.block_size, kv_dtype=s, tensor_core_path=True)
        assert seen[-1] == want and m.kv_dtype == s
    for bad in ("fp16", "FP8", "float8", ""):
        with pytest.raises(ValueError, match="kv_dtype"):
            m.setup_caches(2, d.block_size, kv_dtype=bad, tensor_core_path=True)
    assert len(seen) == 3


def _e4m3_values():
    """Every finite e4m3 value (both zeros included), float64."""
    codes = torch.arange(256, dtype=torch.uint8)
    v = codes.view(torch.float8_e4m3fn).double()
    return v[torch.isfinite(v)]


@pytest.mark.parametrize("e", [-23, -7, -1, 0, 3, 20])
def test_round_trip_is_exact_for_e4m3_times_a_power_of_two(e):
    """A vector of e4m3 values times 2^e that contains +-448 2^e has scale exactly 2^e (for 2^e >= FLT_EPSILON, the
    scale's floor), and every element comes back."""
    vals = _e4m3_values()
    g = torch.Generator().manual_seed(e + 100)
    for sign in (1.0, -1.0):
        for _ in range(20):
            x = vals[torch.randint(0, vals.numel(), (128,), generator=g)].clone()
            x[int(torch.randint(0, 128, (1,), generator=g))] = sign * 448.0
            x = (x * 2.0 ** e).float()
            codes, s = Q.quantize_kv_fp8(x)
            assert float(s) == 2.0 ** e
            assert torch.equal(Q.dequantize_kv_fp8(codes, s), x)


def test_quantiser_definition_and_non_finite_encoding():
    """The expression of the definition on finite rows; zero rows take FLT_EPSILON; NaN and inf have the one encoding the
    device store uses."""
    g = torch.Generator().manual_seed(1)
    x = torch.randn(16, 128, generator=g) * torch.exp2(torch.randint(-20, 20, (16, 1), generator=g).float())
    codes, s = Q.quantize_kv_fp8(x)
    want_s = torch.clamp(x.abs().amax(-1) / 448, min=torch.finfo(torch.float32).eps).to(torch.bfloat16)
    assert torch.equal(s.view(torch.int16), want_s.view(torch.int16))
    want_q = torch.clamp(x / want_s.float()[:, None], -448, 448).to(torch.float8_e4m3fn)
    assert torch.equal(codes.view(torch.uint8), want_q.view(torch.uint8))
    c0, s0 = Q.quantize_kv_fp8(torch.zeros(128))
    assert float(s0) == float(torch.tensor(torch.finfo(torch.float32).eps).to(torch.bfloat16)) and not c0.view(torch.uint8).any()
    y = torch.ones(3, 128)
    y[0, 5] = float("nan")
    y[1, 7] = float("inf")
    y[2, 9] = -float("inf")
    c, s = Q.quantize_kv_fp8(y)
    cb = c.view(torch.uint8)
    assert int(s.view(torch.int16)[0]) == 0x7FC0 and bool((cb[0] == 0x7F).all())
    for r, i in ((1, 7), (2, 9)):
        assert float(s[r]) == float("inf") and int(cb[r, i]) == 0x7F
        assert bool((cb[r, torch.arange(128) != i] == 0).all())
