"""CPU: voice overlays of last-N-block finetunes (Transformer.add_voice): the first overlaid block, rejection of
checkpoints that are not such a finetune, and the overlay's tensor order against include/mvb200.h's offset rule."""
import dataclasses

import pytest
import torch

from mvb200 import synth
from mvb200.fast_model import ModelArgs, Transformer, overlay_first_layer, overlay_keys, stage1_keys

D4 = dataclasses.replace(synth.TINY, n_layer=4)


def finetune(d, base_seed, n_blocks, seed=99):
    """The base state dict with ln_f and the last n_blocks blocks redrawn from another seed (what finetune.py changes)."""
    sd = dict(synth.stage1_state_dict(d, base_seed))
    other = synth.stage1_state_dict(d, seed)
    for k in other:
        if k.startswith("transformer.ln_f.") or any(k.startswith(f"transformer.h.{i}.") for i in range(d.n_layer - n_blocks, d.n_layer)):
            sd[k] = other[k]
    return sd


def _config(d):
    return ModelArgs(block_size=d.block_size, vocab_size=d.vocab_size, n_layer=d.n_layer, n_head=d.n_head, dim=d.dim,
                     intermediate_size=d.intermediate_size, norm_eps=d.norm_eps, norm_type=d.norm_type,
                     nonlinearity_type=d.nonlinearity_type, bias=d.bias)


@pytest.mark.parametrize("n_blocks", [1, 2, 4])
def test_first_layer_is_the_first_finetuned_block(n_blocks):
    base = synth.stage1_state_dict(D4, 0)
    assert overlay_first_layer(base, finetune(D4, 0, n_blocks), _config(D4)) == D4.n_layer - n_blocks


def test_only_ln_f_changed_overlays_the_last_block():
    base = synth.stage1_state_dict(D4, 0)
    sd = dict(base)
    sd["transformer.ln_f.weight"] = synth.stage1_state_dict(D4, 5)["transformer.ln_f.weight"]
    assert overlay_first_layer(base, sd, _config(D4)) == D4.n_layer - 1


@pytest.mark.parametrize("key", ["transformer.h.0.attn.c_attn.weight", "transformer.h.1.ln_2.weight",
                                 "transformer.wtes.0.weight", "transformer.wpe.weight", "speaker_cond_pos.weight",
                                 "lm_heads.0.weight"])
def test_a_change_outside_ln_f_and_the_last_blocks_is_rejected(key):
    base = synth.stage1_state_dict(D4, 0)
    sd = finetune(D4, 0, 1)
    sd[key] = sd[key].clone()
    sd[key].view(-1)[0] += 1
    with pytest.raises(ValueError, match=key.replace(".", r"\.")):
        overlay_first_layer(base, sd, _config(D4))


def test_add_voice_strips_compile_prefix_and_checks_the_architecture():
    base = synth.stage1_state_dict(synth.TINY, 0)
    m = Transformer.from_state_dict(base, _config(synth.TINY), device="cpu")
    ft = finetune(synth.TINY, 0, 1)
    ck = dict(model={"_orig_mod." + k: v for k, v in ft.items()}, model_args=synth.stage1_model_args(synth.TINY))
    assert m.add_voice(ck) == 1 and m.n_voices == 2
    overlay, offsets, first = m._voices[0]
    assert first == 1 and len(offsets) == 7 + 1
    bad = dict(ck, model_args=dict(ck["model_args"], norm_type="layernorm"))
    with pytest.raises(ValueError, match="architecture"):
        m.add_voice(bad)
    with pytest.raises(ValueError, match="n_layer"):
        m.add_voice(dict(ck, model_args=dict(ck["model_args"], n_layer=3)))
    with pytest.raises(KeyError):
        m.voice_id(2)
    assert m.voice_id(None) == 0 and m.voice_id(1) == 1


def test_quantised_engine_refuses_voices_before_reading_weights():
    base = synth.stage1_state_dict(synth.TINY, 0)
    m = Transformer.from_state_dict(base, _config(synth.TINY), device="cpu", quantisation_mode="int8")
    with pytest.raises(NotImplementedError):
        m.add_voice(None)     # nothing is read: the mode is checked first


@pytest.mark.parametrize("norm,mlp,bias", [("rmsnorm", "swiglu", False), ("layernorm", "gelu", True),
                                           ("rmsnorm", "swiglu", True), ("layernorm", "swiglu", False)])
def test_overlay_order_follows_the_header(norm, mlp, bias):
    """Per overlaid layer its tensors in mvb_s1_create_ex's order -- the layer's weights as the arena lists them, then
    its biases as the arena's bias block lists them -- then ln_f.weight and (LayerNorm with bias) ln_f.bias."""
    n_layer, first = 4, 2
    keys = overlay_keys(n_layer, first, norm, mlp, bias)
    full = stage1_keys(n_layer, norm, mlp, bias)
    n_w = 6 if mlp == "gelu" else 7
    n_b = ((2 if norm == "layernorm" else 0) + 3 + (1 if mlp == "gelu" else 2)) if bias else 0
    assert len(keys) == (n_layer - first) * (n_w + n_b) + 1 + (1 if bias and norm == "layernorm" else 0)
    for j, l in enumerate(range(first, n_layer)):
        block = keys[j * (n_w + n_b):(j + 1) * (n_w + n_b)]
        weights = [k for k in full if k.startswith(f"transformer.h.{l}.") and k.endswith(".weight")]
        biases = [k for k in full if k.startswith(f"transformer.h.{l}.") and k.endswith(".bias")]
        assert block == weights + biases
    assert keys[(n_layer - first) * (n_w + n_b)] == "transformer.ln_f.weight"
    if bias and norm == "layernorm":
        assert keys[-1] == "transformer.ln_f.bias"


@pytest.mark.parametrize("norm,mlp,bias", [("rmsnorm", "swiglu", False), ("layernorm", "gelu", True),
                                           ("rmsnorm", "swiglu", True), ("layernorm", "swiglu", False)])
def test_base_tensors_read_back_from_the_arena(norm, mlp, bias):
    """add_voice compares against the base read back from the engine's arena (no host copy of the checkpoint is kept):
    every tensor, with its shape, equals the state dict's."""
    d = dataclasses.replace(synth.TINY, norm_type=norm, nonlinearity_type=mlp, bias=bias, intermediate_size=None)
    d.__post_init__()
    sd = synth.stage1_state_dict(d, 0)
    m = Transformer.from_state_dict(sd, _config(d), device="cpu")
    base = m._base_tensors()
    assert list(base) == stage1_keys(d.n_layer, norm, mlp, bias)
    for k, t in base.items():
        assert t.shape == sd[k].shape and torch.equal(t, sd[k]), k
