"""CPU: the int8 per-channel quantiser (mvb200/quantize.py) against the reference's own dynamically_quantize_per_channel and
WeightOnlyInt8QuantHandler (tests/golden/int8_quant.npz, written by oracle/make_golden_int8.py), the int8 matrix layout, the
quantised key set, the int8 model size and the NaN check."""
import os

import numpy as np
import pytest
import torch

from mvb200 import quantize as Q

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "int8_quant.npz")
CASES = ["k256", "k2048", "k5632", "head", "edge"]


def _bf16(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(a.astype(np.uint16).view(np.int16).copy()).view(torch.bfloat16)


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("case", CASES)
def test_quantiser_bit_identical(golden, case):
    w = _bf16(golden[f"{case}_w"])
    q, s = Q.quantize_per_channel(w)
    assert q.dtype == torch.int8 and s.dtype == torch.bfloat16
    assert torch.equal(q, torch.from_numpy(golden[f"{case}_q"]))
    assert torch.equal(s.view(torch.int16), _bf16(golden[f"{case}_scales"]).view(torch.int16))


def test_minus_128_reachable():
    """q is computed with the fp32 scale s32 = amax / 127.5, so a row's minimum -amax lands near -127.5 and can round to
    -128; the stored bf16 scale differs from s32 by at most half a bf16 ulp (2^-8 relative)."""
    g = torch.Generator().manual_seed(0)
    w = (torch.randn(2048, 2048, generator=g) * 0.02).to(torch.bfloat16)
    q, s = Q.quantize_per_channel(w)
    s32 = torch.clamp(torch.maximum(-w.float().amin(1).clamp(max=0), w.float().amax(1).clamp(min=0)) / 127.5,
                      min=torch.finfo(torch.float32).eps)
    rel = float(((s.float() - s32) / s32).abs().max())
    print(f"2048 x 2048: {int((q == -128).sum())} elements at -128; bf16 vs fp32 scale up to {rel:.2e} relative")
    assert int((q == -128).sum()) > 0 and 0 < rel <= 2.0 ** -8


@pytest.mark.parametrize("M,K", [(16, 256), (24, 768), (8, 5632), (3, 100)])
def test_pack_round_trip(M, K):
    g = torch.Generator().manual_seed(M + K)
    w = (torch.randn(M, K, generator=g) * 0.03).to(torch.bfloat16)
    q, s = Q.quantize_per_channel(w)
    buf = Q.pack_int8_matrix(q, s)
    assert buf.numel() == Q.int8_matrix_bytes(M, K)
    q2, s2 = Q.unpack_int8_matrix(buf, M, K)
    assert torch.equal(q, q2) and torch.equal(s.view(torch.int16), s2.view(torch.int16))
    # layout: int8 row-major, then the bf16 scales at the next 256-byte boundary
    assert torch.equal(buf[:M * K].view(torch.int8).reshape(M, K), q)
    so = (M * K + 255) // 256 * 256
    assert torch.equal(buf[so:so + 2 * M].view(torch.bfloat16).view(torch.int16), s.view(torch.int16))


def _tiny():
    from mvb200 import synth
    from mvb200.fast_model import ModelArgs
    d = synth.TINY
    cfg = ModelArgs(block_size=d.block_size, vocab_size=d.vocab_size, n_layer=d.n_layer, n_head=d.n_head, dim=d.dim)
    return d, synth.stage1_state_dict(d, 0), cfg


def test_quantised_key_set_is_the_reference_handlers(golden):
    from oracle.ref_harness import rename_to_fast
    d, sd, _ = _tiny()
    ours = [k for k, linear, _ in Q._keys(d.n_layer) if linear]
    fast = sorted(k[:-len(".weight")] for k in rename_to_fast({k: None for k in ours}))
    assert fast == sorted(str(n) for n in golden["tiny_quantised_modules"])


def test_arena_layout():
    d, sd, _ = _tiny()
    arena, offs, _ = Q.pack_arena_int8(sd, d.n_layer)
    assert len(offs) == 5 + 7 * d.n_layer and all(o % 256 == 0 for o in offs)
    # every Linear is an int8 matrix that decodes to the quantiser's output; embeddings and norms are the bf16 tensors
    for i, (k, linear, _) in enumerate(Q._keys(d.n_layer)):
        t = sd[k]
        if linear:
            q, s = Q.unpack_int8_matrix(arena[offs[i]:], *t.shape)
            q0, s0 = Q.quantize_per_channel(t)
            assert torch.equal(q, q0) and torch.equal(s.view(torch.int16), s0.view(torch.int16)), k
        else:
            b = t.to(torch.bfloat16).contiguous().reshape(-1).view(torch.uint8)
            assert torch.equal(arena[offs[i]:offs[i] + b.numel()], b), k


def test_model_size_is_the_reference_model_size(golden):
    from mvb200.fast_model import ModelArgs, Transformer
    d, sd, cfg = _tiny()
    _, _, payload = Q.pack_arena_int8(sd, d.n_layer)
    assert payload == int(golden["tiny_model_size"]) == Transformer.int8_model_size_bytes(cfg)
    full = ModelArgs.from_name("metavoice-1B")
    D, F, V, L = full.dim, full.intermediate_size, full.vocab_size, full.n_layer
    want = (L * (4 * D * D + 3 * D * F + 2 * (5 * D + 2 * F) + 4 * D) + full.speaker_emb_dim * D + 2 * D + V * D + 2 * V
            + 2 * (V * D + full.block_size * D + D))
    i8, b16 = Transformer.int8_model_size_bytes(full), Transformer.bf16_model_size_bytes(full)
    print(f"metavoice-1B: int8 arena {i8 / 1e9:.3f} GB, bf16 {b16 / 1e9:.3f} GB")
    assert i8 == want and 1.25e9 < i8 < 1.27e9 and 2.49e9 < b16 < 2.51e9


def test_dequantized_state_dict_is_s_times_q():
    d, sd, _ = _tiny()
    sdq = Q.int8_dequantized_state_dict(sd, d.n_layer)
    k = "transformer.h.0.mlp.swiglu.w1.weight"
    q, s = Q.quantize_per_channel(sd[k])
    assert torch.equal(sdq[k].view(torch.int16), (q.double() * s.double()[:, None]).to(torch.bfloat16).view(torch.int16))
    assert torch.equal(sdq["transformer.wpe.weight"], sd["transformer.wpe.weight"])


def test_nan_weight_rejected():
    d, sd, _ = _tiny()
    sd = dict(sd)
    w = sd["transformer.h.1.attn.c_proj.weight"].clone()
    w[3, 7] = float("nan")
    sd["transformer.h.1.attn.c_proj.weight"] = w
    with pytest.raises(ValueError, match="NaN"):
        Q.pack_arena_int8(sd, d.n_layer)


def test_int8_needs_the_cuda_engine(tmp_path):
    from mvb200 import fast_inference_utils as U
    with pytest.raises(NotImplementedError):
        U._load_model(tmp_path / "missing.pt", None, "cpu", torch.bfloat16, "int8")
