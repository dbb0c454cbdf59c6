"""CPU: the fp8 (e4m3) per-channel quantiser (mvb200/quantize.py) against the torch expression that defines it, on random
and adversarial rows; the fp8 matrix layout (fragment-native code order, 256-byte scale alignment); the quantised key set
and model size; the NaN / Inf check; the mode's argument checks; and the fp8 engine's workspace size.  The reference has
no fp8 mode, so torch's own float8_e4m3fn cast is the oracle."""
import ctypes as C
import dataclasses

import pytest
import torch

from mvb200 import quantize as Q
from mvb200 import synth

FLT_EPS = torch.finfo(torch.float32).eps


def _expr(w):
    """The definition: s = bf16(max(amax / 448, eps)), q = e4m3(clamp(w / fp32(s), -448, 448))."""
    wf = w.to(torch.bfloat16).float()
    s = torch.clamp(wf.abs().amax(1) / 448, min=FLT_EPS).to(torch.bfloat16)
    return torch.clamp(wf / s.float()[:, None], -448, 448).to(torch.float8_e4m3fn), s


def _same(a, b):
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def _tiny():
    from mvb200.fast_model import ModelArgs
    d = synth.TINY
    cfg = ModelArgs(block_size=d.block_size, vocab_size=d.vocab_size, n_layer=d.n_layer, n_head=d.n_head, dim=d.dim)
    return d, synth.stage1_state_dict(d, 0), cfg


@pytest.mark.parametrize("M,K,std", [(64, 256, 0.02), (48, 2048, 1.0), (18, 5632, 3e-4)])
def test_quantiser_bit_identical_random(M, K, std):
    w = (torch.randn(M, K, generator=torch.Generator().manual_seed(M + K)) * std).to(torch.bfloat16)
    q, s = Q.quantize_fp8_per_channel(w)
    q0, s0 = _expr(w)
    assert q.dtype == torch.float8_e4m3fn and s.dtype == torch.bfloat16
    assert _same(q, q0) and torch.equal(s.view(torch.int16), s0.view(torch.int16))


def test_quantiser_adversarial_rows():
    K = 256
    rows = torch.zeros(4, K)
    # row 0: all zero -> scale eps, codes +0
    # row 1: amax just above a bf16 rounding boundary of amax / 448, so the stored scale rounds down and w / s > 448
    amax = 512.0                                # 512 / 448 = 1.1429 rounds down to bf16 1.1406: w / s = 448.9
    rows[1, 0], rows[1, 1] = amax, -amax
    rows[1, 2:] = torch.linspace(-1, 1, K - 2)
    # row 2: values that land on e4m3 subnormals (below 2^-6 s) and values that round to zero (below 2^-10 s)
    rows[2, 0] = 448.0
    rows[2, 1:8] = torch.tensor([2 ** -7, 3 * 2 ** -9, 2 ** -9, -2 ** -8, 2 ** -11, -2 ** -12, 2 ** -10 * 1.5])
    rows[3] = torch.randn(K, generator=torch.Generator().manual_seed(3))
    w = rows.to(torch.bfloat16)
    q, s = Q.quantize_fp8_per_channel(w)
    q0, s0 = _expr(w)
    assert _same(q, q0) and torch.equal(s.view(torch.int16), s0.view(torch.int16))
    assert float(s[0]) == FLT_EPS and not q[0].float().any()
    assert float(w[1, 0].float() / s[1].float()) > 448, "row 1 does not exercise the clamp"
    assert float(q[1, 0].float()) == 448 and float(q[1, 1].float()) == -448
    qv = q[2, 1:8].float()
    assert ((qv.abs() > 0) & (qv.abs() < 2 ** -6)).any() and (qv == 0).any(), "row 2 reaches no subnormal or no zero"
    # torch's cast does not saturate: what the clamp guards against
    assert torch.isnan(torch.tensor([500.0]).to(torch.float8_e4m3fn).float()).all()


def test_nan_and_inf_rejected():
    d, sd, _ = _tiny()
    for bad in (float("nan"), float("inf"), -float("inf")):
        sdb = dict(sd)
        w = sd["transformer.h.1.attn.c_proj.weight"].clone()
        w[3, 7] = bad
        sdb["transformer.h.1.attn.c_proj.weight"] = w
        with pytest.raises(ValueError, match="NaN or Inf"):
            Q.pack_arena_fp8(sdb, d.n_layer)


@pytest.mark.parametrize("M,K", [(2562, 256), (34, 512), (16, 256), (2, 768)])
def test_layout(M, K):
    """Codes at f8_code_offset's position (include/mvb200.h), the scales at the next 256-byte boundary, and the round trip."""
    q, s = Q.quantize_fp8_per_channel(torch.randn(M, K, generator=torch.Generator().manual_seed(M)).to(torch.bfloat16))
    buf = Q.pack_fp8_matrix(q, s)
    so = (M * K + 255) // 256 * 256
    assert buf.numel() == Q.int8_matrix_bytes(M, K) == so + 2 * M
    assert torch.equal(buf[so:].view(torch.bfloat16).view(torch.int16), s.view(torch.int16))
    assert not buf[M * K:so].any()
    u = q.view(torch.uint8)
    M16 = M // 16 * 16
    g = torch.Generator().manual_seed(K)
    for j, k in zip(torch.randint(0, M, (500,), generator=g).tolist(), torch.randint(0, K, (500,), generator=g).tolist()):
        if j >= M16:
            off = j * K + k
        else:
            r, kk = j % 16, k % 32
            lane = (r % 8) * 4 + (kk % 8) // 2
            word = (kk // 16) * 2 + (kk // 8) % 2
            byte = (kk % 2) * 2 + r // 8
            off = ((j // 16) * (K // 32) + k // 32) * 512 + lane * 16 + word * 4 + byte
        assert int(buf[off]) == int(u[j, k]), (j, k)
    q1, s1 = Q.unpack_fp8_matrix(buf, M, K)
    assert _same(q1, q) and torch.equal(s1.view(torch.int16), s.view(torch.int16))


def test_arena_key_set_and_model_size():
    from mvb200.fast_model import ModelArgs, Transformer
    d, sd, cfg = _tiny()
    arena, offs, payload = Q.pack_arena_fp8(sd, d.n_layer)
    assert len(offs) == 5 + 7 * d.n_layer and all(o % 256 == 0 for o in offs)
    linear = [k for k, lin, _ in Q._keys(d.n_layer) if lin]
    assert sorted(linear) == sorted(["speaker_cond_pos.weight", "lm_heads.0.weight"] +
                                    [f"transformer.h.{i}.{k}.weight" for i in range(d.n_layer)
                                     for k in ("attn.c_attn", "attn.c_proj", "mlp.swiglu.w1", "mlp.swiglu.w3", "mlp.c_proj")])
    for i, (k, lin, _) in enumerate(Q._keys(d.n_layer)):
        t = sd[k]
        if lin:
            q, s = Q.unpack_fp8_matrix(arena[offs[i]:], *t.shape)
            q0, s0 = Q.quantize_fp8_per_channel(t)
            assert _same(q, q0) and torch.equal(s.view(torch.int16), s0.view(torch.int16)), k
        else:
            b = t.to(torch.bfloat16).contiguous().reshape(-1).view(torch.uint8)
            assert torch.equal(arena[offs[i]:offs[i] + b.numel()], b), k
    m = object.__new__(Transformer)
    m.config, m.quantisation_mode = cfg, "fp8"
    assert payload == m.model_size_bytes() == Transformer.int8_model_size_bytes(cfg)
    full = ModelArgs.from_name("metavoice-1B")
    m.config = full
    print(f"metavoice-1B: fp8 arena {m.model_size_bytes() / 1e9:.3f} GB")
    assert 1.25e9 < m.model_size_bytes() < 1.27e9


def test_dequantized_state_dict_is_s_times_q():
    d, sd, _ = _tiny()
    sdq = Q.fp8_dequantized_state_dict(sd, d.n_layer)
    k = "transformer.h.0.mlp.swiglu.w1.weight"
    q, s = Q.quantize_fp8_per_channel(sd[k])
    assert torch.equal(sdq[k].view(torch.int16), (q.double() * s.double()[:, None]).to(torch.bfloat16).view(torch.int16))


def test_mode_argument_checks(tmp_path, monkeypatch):
    from mvb200 import fast_inference_utils as U
    from mvb200.fast_model import ModelArgs, Transformer
    with pytest.raises(Exception, match="Invalid quantisation mode"):
        U._load_model(tmp_path / "missing.pt", None, "cuda", torch.bfloat16, "fp16")
    with pytest.raises(NotImplementedError):
        U._load_model(tmp_path / "missing.pt", None, "cpu", torch.bfloat16, "fp8")
    d = dataclasses.replace(synth.TINY, norm_type="layernorm", nonlinearity_type="gelu", bias=True, intermediate_size=None)
    d.__post_init__()
    path = tmp_path / "first_stage.pt"
    torch.save(synth.stage1_checkpoint(d, 0, tie_head=True), str(path))

    def no_read(*a, **k):
        raise AssertionError("weights read")
    monkeypatch.setattr(Transformer, "from_state_dict", classmethod(no_read))
    with pytest.raises(NotImplementedError, match="production architecture"):
        U._load_model(path, None, "cuda", torch.bfloat16, quantisation_mode="fp8")
    with pytest.raises(NotImplementedError, match="production architecture"):
        Transformer.__init__(object.__new__(Transformer), ModelArgs(n_layer=2, n_head=2, dim=256, norm_type="layernorm"),
                             torch.zeros(1, dtype=torch.uint8), [0], "cpu", "fp8")


@pytest.mark.parametrize("max_utts,want", [(1, 180869632), (8, 185481216)])
def test_fp8_workspace_bytes(max_utts, want):
    """The int8 workspace plus speaker_cond_pos's widened q (dim x spk_dim bf16) for the production config."""
    from mvb200 import _lib
    lib = _lib.load()
    d = synth.FULL
    cfg = _lib.S1Config(d.n_layer, d.n_head, d.head_dim, d.dim, d.intermediate_size, d.vocab_size, d.block_size,
                        d.speaker_emb_dim, d.norm_eps, max_utts, _lib.MVB_KV_BF16, d.block_size)
    i8, f8 = lib.mvb_s1_int8_workspace_bytes(C.byref(cfg)), lib.mvb_s1_fp8_workspace_bytes(C.byref(cfg))
    assert f8 == want == i8 + d.dim * d.speaker_emb_dim * 2
