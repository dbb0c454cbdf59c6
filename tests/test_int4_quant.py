"""CPU: the int4 group quantiser (mvb200/quantize.py) against the reference's own group_quantize_tensor /
group_dequantize_tensor_from_qparams (tests/golden/int4_quant.npz, written by tools/make_golden_int4.py), the packed
layout, the tensor-selection rule, the int4 model size and the quantisation_mode errors."""
import os

import numpy as np
import pytest
import torch

from mvb200 import quantize as Q

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "int4_quant.npz")
CASES = ["k256", "k2048", "k5632", "edge"]


def _bf16(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(a.astype(np.uint16).view(np.int16).copy()).view(torch.bfloat16)


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("case", CASES)
def test_quantiser_bit_identical(golden, case):
    w = _bf16(golden[f"{case}_w"])
    assert torch.isfinite(w.float()).all()
    q, s, z = Q.group_quantize(w)
    assert torch.equal(q, torch.from_numpy(golden[f"{case}_q"]))
    assert torch.equal(s.view(torch.int16), _bf16(golden[f"{case}_scales"]).view(torch.int16))
    assert torch.equal(z.view(torch.int16), _bf16(golden[f"{case}_zeros"]).view(torch.int16))


def _ulp(a: torch.Tensor) -> torch.Tensor:
    """One bf16 ulp of |a| (float64 in, float64 out; 0 for 0)."""
    mag = a.abs()
    return torch.where(mag > 0, 2.0 ** (torch.floor(torch.log2(mag.clamp(min=1e-300))) - 7), torch.zeros_like(mag))


@pytest.mark.parametrize("case", CASES)
def test_dequant_against_reference(golden, case):
    """W_deq (the exact value rounded once) against the reference's dequantiser, which rounds to bf16 after the multiply and
    again after the add.  Where its product rounding is exact the two are equal; in general the gap is at most half an ulp
    of the product (the reference's first rounding, which cancellation against z can make larger than an ulp of the
    result) plus one ulp of the result."""
    q = torch.from_numpy(golden[f"{case}_q"])
    s, z = _bf16(golden[f"{case}_scales"]), _bf16(golden[f"{case}_zeros"])
    ref = _bf16(golden[f"{case}_deq"])
    got = Q.dequantize(q, s, z)
    M, K = q.shape
    qd = q.double().reshape(M, K // 128, 128) - 8
    prod = qd * s.double()[..., None]
    prod_r = prod.to(torch.bfloat16).double()
    prod_exact = (prod_r == prod).reshape(M, K)
    total = prod + z.double()[..., None]
    sum_exact = ((prod_r + z.double()[..., None]).to(torch.bfloat16).double() == total).reshape(M, K)
    exact = prod_exact & sum_exact
    g, r = got.double(), ref.double()
    diff = (g - r).abs()
    one_ulp = _ulp(torch.maximum(g.abs(), r.abs()))
    assert torch.equal(got[prod_exact].view(torch.int16), ref[prod_exact].view(torch.int16))
    assert bool((diff <= one_ulp + 0.5 * _ulp(prod).reshape(M, K)).all())
    print(f"{case}: {int(exact.sum())}/{exact.numel()} exact in the reference, "
          f"{int((diff > 0).sum())} differ, {int((diff > one_ulp).sum())} by more than one ulp")


@pytest.mark.parametrize("M,K", [(16, 256), (24, 768), (8, 5632)])
def test_pack_round_trip(M, K):
    g = torch.Generator().manual_seed(M + K)
    w = (torch.randn(M, K, generator=g) * 0.03).to(torch.bfloat16)
    q, s, z = Q.group_quantize(w)
    buf = Q.pack_matrix(q, s, z)
    assert buf.numel() == Q.packed_bytes(M, K)
    q2, s2, z2 = Q.unpack_matrix(buf, M, K)
    assert torch.equal(q, q2) and torch.equal(s.view(torch.int16), s2.view(torch.int16))
    assert torch.equal(z.view(torch.int16), z2.view(torch.int16))
    # word layout: the first 32-bit word of a row holds k = 0, 2, 4, 6 in bits 0-15 and k = 1, 3, 5, 7 in bits 16-31
    w0 = int(buf[:4].clone().view(torch.int32)) & 0xFFFFFFFF
    assert [(w0 >> (4 * n)) & 0xF for n in range(8)] == [int(q[0, k]) for k in (0, 2, 4, 6, 1, 3, 5, 7)]


def test_selection_rule():
    assert Q.is_quantised(6144, 2048) and Q.is_quantised(2048, 5632) and Q.is_quantised(2048, 256)
    assert not Q.is_quantised(2562, 2048)           # lm_head of MetaVoice-1B stays bf16
    with pytest.raises(ValueError, match="in_features"):
        Q.is_quantised(2048, 200, "w_bad")


def _tiny_sd():
    from mvb200 import synth
    return synth.TINY, synth.stage1_state_dict(synth.TINY, 0)


def test_arena_layout_and_selection():
    d, sd = _tiny_sd()
    arena, offs, payload = Q.pack_arena_int4(sd, d.n_layer)
    assert len(offs) == 5 + 7 * d.n_layer and all(o % 256 == 0 for o in offs)
    # lm_head (vocab 2562 outputs) is the bf16 checkpoint tensor, byte for byte
    lm = sd["lm_heads.0.weight"].to(torch.bfloat16).contiguous().reshape(-1).view(torch.uint8)
    assert torch.equal(arena[offs[4]:offs[4] + lm.numel()], lm)
    # speaker_cond_pos is stored as W_deq
    spk = sd["speaker_cond_pos.weight"]
    want = Q.dequantize(*Q.group_quantize(spk)).reshape(-1).view(torch.uint8)
    assert torch.equal(arena[offs[2]:offs[2] + want.numel()], want)
    # w2 of layer 1 is a packed matrix that decodes to the quantiser's output
    w2 = sd["transformer.h.1.mlp.c_proj.weight"]
    M, K = w2.shape
    q, s, z = Q.unpack_matrix(arena[offs[5 + 7 + 6]:], M, K)
    q0, s0, z0 = Q.group_quantize(w2)
    assert torch.equal(q, q0) and torch.equal(s.view(torch.int16), s0.view(torch.int16))


def test_bad_in_features_rejected():
    d, sd = _tiny_sd()
    sd = dict(sd)
    sd["speaker_cond_pos.weight"] = torch.zeros(d.dim, 200)
    with pytest.raises(ValueError, match="in_features"):
        Q.pack_arena_int4(sd, d.n_layer)


def test_model_size_is_int4_arena():
    from mvb200.fast_model import ModelArgs, Transformer
    d, sd = _tiny_sd()
    cfg = ModelArgs(block_size=d.block_size, vocab_size=d.vocab_size, n_layer=d.n_layer, n_head=d.n_head, dim=d.dim)
    D, F, V = cfg.dim, cfg.intermediate_size, cfg.vocab_size
    per_layer = (4 * D * D + 3 * D * F) // 2 + (4 * D * D + 3 * D * F) // 128 * 4 + 2 * D * 2
    want = cfg.n_layer * per_layer + (2 * V * D + cfg.block_size * D + cfg.speaker_emb_dim * D + D) * 2
    _, _, payload = Q.pack_arena_int4(sd, d.n_layer)
    assert payload == want
    assert Transformer.int4_model_size_bytes(cfg) == want
    full = ModelArgs.from_name("metavoice-1B")
    i4, b16 = Transformer.int4_model_size_bytes(full), Transformer.bf16_model_size_bytes(full)
    print(f"metavoice-1B: int4 arena {i4 / 1e9:.3f} GB, bf16 {b16 / 1e9:.3f} GB")
    assert 0.6e9 < i4 < 0.7e9 and i4 < 0.3 * b16


def test_modes_raise(tmp_path):
    from mvb200 import fast_inference_utils as U
    p = tmp_path / "missing.pt"
    with pytest.raises(NotImplementedError):
        U._load_model(p, None, "cpu", torch.bfloat16, "int8")
    with pytest.raises(Exception, match="Invalid quantisation mode"):
        U._load_model(p, None, "cpu", torch.bfloat16, "int2")
