"""CPU: the stage-2 architectures beyond rmsnorm / swiglu / no bias -- the oracle against golden vectors from the reference's
own GPT (and the live reference where it is mounted), SecondStage's reading of model_args, and the library's host-side
validation of mvb_s2_create_ex (offset count, arch fields, workspace size)."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from mvb200 import _lib, synth
from mvb200.second_stage import stage2_arch, stage2_keys
from oracle import make_golden_stage2_arch as G, ref_harness, stage2_arch_port as A, stage2_port as P

VARIANTS = G.variants()
IDS = [v[0] for v in VARIANTS]


def _oracle(d, sd):
    return A.Stage2ArchOracle(sd, d.n_head, d.rmsnorm_eps, norm_type=d.norm_type, nonlinearity_type=d.nonlinearity_type,
                              bias=d.bias)


@pytest.mark.parametrize("tag,dims,frames,drop", VARIANTS, ids=IDS)
def test_stage2_arch_oracle_matches_reference_golden(golden_dir, tag, dims, frames, drop):
    g = np.load(f"{golden_dir}/stage2_arch.npz")
    sd = synth.stage2_state_dict(dims, 1)
    assert synth.state_dict_checksum(sd) == pytest.approx(float(g[f"{tag}_checksum"]), abs=1e-9)
    logits = _oracle(dims, sd).forward(torch.from_numpy(g[f"{tag}_idx"]).long(), torch.from_numpy(g[f"{tag}_spk"]))
    keep = g[f"{tag}_keep"]
    got = torch.stack([logits[h][0, keep] for h in G.HEADS])
    ref = torch.from_numpy(g[f"{tag}_logits"])
    assert float((got - ref).abs().max() / ref.abs().max()) < 1e-5
    torch.manual_seed(4242)
    noise = [torch.empty(1, dims.block_size, v).exponential_(1) for v in dims.target_vocab_sizes]
    y = P.non_causal_sample(logits, 1.0, 200, noise)
    assert torch.equal(y[0].int(), torch.from_numpy(g[f"{tag}_tokens"]).int())


@pytest.mark.parametrize("tag,dims", [("tiny", synth.S2_TINY), ("full", synth.S2_FULL)])
def test_stage2_arch_oracle_at_production_equals_stage2_oracle(golden_dir, tag, dims):
    """With rmsnorm / swiglu / no bias the architecture oracle computes exactly what oracle/stage2_port.py computes."""
    g = np.load(f"{golden_dir}/stage2.npz")
    sd = synth.stage2_state_dict(dims, 1)
    idx, spk = torch.from_numpy(g[f"{tag}_idx"]).long(), torch.from_numpy(g[f"{tag}_spk"])
    a = _oracle(dims, sd).forward(idx, spk)
    b = P.Stage2Oracle(sd, dims.n_head, dims.rmsnorm_eps).forward(idx, spk)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.skipif(not ref_harness.available(), reason="reference tree not mounted")
@pytest.mark.parametrize("tag,dims,frames,drop", [v for v in VARIANTS if v[0].startswith("tiny")],
                         ids=[v[0] for v in VARIANTS if v[0].startswith("tiny")])
def test_stage2_arch_oracle_matches_live_reference(tag, dims, frames, drop):
    sd = synth.stage2_state_dict(dims, 1)
    m = G.reference_gpt(dims, sd, drop)
    text, cb0, cb1 = synth.synthetic_stage2_input(dims, frames)
    idx = P.build_input(text, cb0, cb1, dims.block_size)[None]
    spk = synth.synthetic_speaker(seed=5)[None]
    with torch.no_grad():
        ref, _ = m(idx, speaker_embs=spk)
    got = _oracle(dims, sd).forward(idx, spk)
    for a, b in zip(got, ref):
        assert float((a - b).abs().max() / b.abs().max()) < 1e-5


def test_missing_arch_keys_mean_gptconfig_defaults():
    args = synth.stage2_model_args(synth.S2_FULL)
    assert stage2_arch(args) == ("rmsnorm", "swiglu", False)
    for k in G.ARCH_KEYS:
        args.pop(k)
    assert stage2_arch(args) == ("layernorm", "gelu", True)          # model.py:36-43
    assert stage2_arch({"norm_type": "rmsnorm"}) == ("rmsnorm", "gelu", True)
    assert stage2_arch({"bias": False, "nonlinearity_type": "swiglu"}) == ("layernorm", "swiglu", False)


@pytest.mark.parametrize("key,value", [("norm_type", "batchnorm"), ("nonlinearity_type", "relu"), ("norm_type", None)])
def test_unknown_arch_values_raise(key, value):
    with pytest.raises(NotImplementedError, match=key):
        stage2_arch({**synth.stage2_model_args(synth.S2_TINY), key: value})


ARCHS = [(n, m, b) for n in ("rmsnorm", "layernorm") for m in ("swiglu", "gelu") for b in (False, True)]


def _cfg(d, max_batch=1):
    cfg = _lib.S2Config()
    cfg.n_layer, cfg.n_head, cfg.n_embd, cfg.hidden = d.n_layer, d.n_head, d.n_embd, d.hidden
    cfg.block_size, cfg.n_in, cfg.n_out = d.block_size, len(d.vocab_sizes), len(d.target_vocab_sizes)
    for i, v in enumerate(d.vocab_sizes):
        cfg.vocab_in[i] = v
    for i, v in enumerate(d.target_vocab_sizes):
        cfg.vocab_out[i] = v
    cfg.spk_dim, cfg.norm_eps, cfg.max_batch = d.speaker_emb_dim, d.rmsnorm_eps, max_batch
    return cfg


def _arch(norm, mlp, bias):
    return _lib.S2Arch({"rmsnorm": 0, "layernorm": 1}[norm], {"swiglu": 0, "gelu": 1}[mlp], int(bias))


@pytest.mark.parametrize("norm,mlp,bias", ARCHS)
def test_offset_count_matches_state_dict(norm, mlp, bias):
    """The key list SecondStage packs holds every tensor of the architecture's state dict once, and mvb_s2_create_ex reads
    exactly that many offsets: an out-of-range entry at the last position is rejected, one past it is never read (the
    call goes on to reject the null workspace, before touching a device)."""
    lib = _lib.load()
    d = dataclasses.replace(synth.S2_TINY, norm_type=norm, nonlinearity_type=mlp, bias=bias)
    sd = synth.stage2_state_dict(d, 1)
    keys = stage2_keys(len(d.vocab_sizes), len(d.target_vocab_sizes), d.n_layer, norm, mlp, bias)
    assert sorted(keys) == sorted(sd) and len(set(keys)) == len(keys)
    n, arena = len(keys), 1 << 20
    arch, cfg, h = _arch(norm, mlp, bias), _cfg(d), C.c_void_p()
    offs = (C.c_uint64 * (n + 1))(*([256 * i for i in range(n)] + [arena]))     # entry n lies outside the arena
    rc = lib.mvb_s2_create_ex(C.byref(cfg), C.byref(arch), C.c_void_p(256), arena, offs, None, C.byref(h))
    assert rc == _lib.MVB_ERR_ARG and b"null pointer" in lib.mvb_last_error(), lib.mvb_last_error()
    offs[n - 1] = arena
    rc = lib.mvb_s2_create_ex(C.byref(cfg), C.byref(arch), C.c_void_p(256), arena, offs, None, C.byref(h))
    assert rc == _lib.MVB_ERR_ARG and b"weight offset" in lib.mvb_last_error(), lib.mvb_last_error()
    assert not h.value


@pytest.mark.parametrize("field,value", [("norm", 2), ("norm", -1), ("mlp", 2), ("mlp", -1), ("bias", 2), ("bias", -1)])
def test_bad_arch_is_rejected_and_named(field, value):
    lib = _lib.load()
    cfg, arch, h = _cfg(synth.S2_TINY), _lib.S2Arch(0, 0, 0), C.c_void_p()
    setattr(arch, field, value)
    offs = (C.c_uint64 * 64)(*([256 * i for i in range(64)]))
    rc = lib.mvb_s2_create_ex(C.byref(cfg), C.byref(arch), C.c_void_p(256), 1 << 20, offs, C.c_void_p(256), C.byref(h))
    assert rc == _lib.MVB_ERR_ARG
    assert f"arch.{field}".encode() in lib.mvb_last_error(), lib.mvb_last_error()
    assert not h.value


def test_workspace_bytes_for_gelu():
    """mvb_s2_workspace_bytes sizes from cfg.hidden and the SwiGLU (two-weight) split-K plan, which covers c_fc's
    one-weight plan at the same width: GELU's hidden = 4 E needs no arch argument."""
    lib = _lib.load()
    gelu = dataclasses.replace(synth.S2_FULL, norm_type="layernorm", nonlinearity_type="gelu", bias=True)
    assert gelu.hidden == 4 * gelu.n_embd == 1536
    got = [lib.mvb_s2_workspace_bytes(C.byref(_cfg(gelu, b))) for b in (1, 2)]
    # vs hidden 1024: + the ffn rows (1024 x 512 x 4 B per utterance), + the B operand (2 x 128 x 512 x 2 B), + the split-K
    # scratch of mlp.c_proj (K = 1536: 3 tiles x 12 splits instead of 3 x 8, x 256 x 128 x 4 B)
    assert got == [44888064, 84269568]
    assert got[0] - 40955904 == 1024 * 512 * 4 + 2 * 128 * 512 * 2 + 3 * 4 * 256 * 128 * 4
    assert all(g > lib.mvb_s2_workspace_bytes(C.byref(_cfg(synth.S2_FULL, b))) for g, b in zip(got, (1, 2)))
