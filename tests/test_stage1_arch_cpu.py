"""CPU: the stage-1 architectures beyond rmsnorm / swiglu / no bias -- the oracle against golden vectors from the
reference's own causal GPT with its KV cache (and the live reference where it is mounted), _load_model's reading of
model_args, and the library's host-side validation of mvb_s1_create_ex (offset count, arch fields, workspace size)."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from mvb200 import _lib, synth
from mvb200 import fast_inference_utils as U
from mvb200.fast_model import ModelArgs, Transformer, stage1_keys
from oracle import make_golden_stage1_arch as G, ref_harness, stage1_arch_port as A, stage1_port as P

VARIANTS = G.variants()
IDS = [v[0] for v in VARIANTS]
ARCHS = [(n, m, b) for n in ("rmsnorm", "layernorm") for m in ("swiglu", "gelu") for b in (False, True)]


def _oracle(d, sd):
    return A.Stage1ArchOracle(sd, d.n_head, d.norm_eps, norm_type=d.norm_type, nonlinearity_type=d.nonlinearity_type,
                              bias=d.bias)


def _sample_ids(logits, noise):
    sk = {k: torch.tensor(v) for k, v in G.SAMPLING.items()}
    return np.asarray([int(P.sample(lg[:, None], q=noise[i], **sk)[0]) for i, lg in enumerate(logits)])


@pytest.mark.parametrize("tag,dims", VARIANTS, ids=IDS)
def test_stage1_arch_oracle_matches_reference_golden(golden_dir, tag, dims):
    g = np.load(f"{golden_dir}/stage1_arch.npz")
    sd = synth.stage1_state_dict(dims, int(g["weight_seed"]), tie_head=True)
    assert synth.state_dict_checksum(sd) == pytest.approx(float(g[f"{tag}_checksum"]), abs=1e-9)
    noise = G.noise(dims.vocab_size)
    assert float(noise.double().sum()) == pytest.approx(float(g["noise_checksum"]), rel=1e-12)
    prompt, forced = torch.from_numpy(g["prompt"]).long(), torch.from_numpy(g["forced"]).long()
    spk = synth.synthetic_speaker(seed=int(g["spk_seed"]))
    every = A.teacher_forced(_oracle(dims, sd), prompt, spk, forced)               # [1 + n_steps, 2, V]
    got = every[[0] + [int(s) for s in g["steps"]]]
    ref = torch.from_numpy(g[f"{tag}_logits"])
    assert float((got - ref).abs().max() / ref.abs().max()) < 1e-5
    ids = _sample_ids(every, noise)
    assert int((ids != g[f"{tag}_ids"]).sum()) == 0


@pytest.mark.parametrize("dims", [synth.TINY, dataclasses.replace(synth.FULL, n_layer=2)], ids=["tiny", "full2"])
def test_stage1_arch_oracle_at_production_equals_stage1_oracle(dims):
    """With rmsnorm / swiglu / no bias the architecture oracle computes bit for bit what oracle/stage1_port.py does."""
    sd = synth.stage1_state_dict(dims, 0)
    a = _oracle(dims, sd)
    b = P.Stage1Oracle(sd, dims.n_head, dims.norm_eps, torch.float32, faithful_full_cache=False)
    a.setup_caches(); b.setup_caches()
    prompt, spk = synth.synthetic_prompt(12), synth.synthetic_speaker()
    idx = prompt.view(1, -1).repeat(2, 1)
    assert torch.equal(a.forward(idx, spk, torch.arange(12)), b.forward(idx, spk, torch.arange(12)))
    for s, tok in enumerate([5, 1700, 2048]):
        t = torch.tensor([[tok], [tok]])
        assert torch.equal(a.forward(t, spk, torch.tensor([12 + s])), b.forward(t, spk, torch.tensor([12 + s])))


@pytest.mark.skipif(not ref_harness.available(), reason="reference tree not mounted")
@pytest.mark.parametrize("tag,dims", [v for v in VARIANTS if v[0].startswith("tiny")],
                         ids=[v[0] for v in VARIANTS if v[0].startswith("tiny")])
def test_stage1_arch_oracle_matches_live_reference(tag, dims):
    sd = synth.stage1_state_dict(dims, 3, tie_head=True)
    m = G.reference_gpt(dims, sd)
    m.enable_kv_cache()
    m.empty_kv_cache(batch_size=2, kv_cache_maxlen=dims.block_size, dtype=torch.float32)
    prompt, spk = synth.synthetic_prompt(9, seed=2), synth.synthetic_speaker(seed=4)
    o = _oracle(dims, sd)
    o.setup_caches()
    with torch.no_grad():
        for s, idx in enumerate([prompt.long(), torch.tensor([33]), torch.tensor([1999])]):
            ref = m(idx.view(1, 1, -1).repeat(2, 1, 1), speaker_embs=[spk, None])[0][0][:, -1]
            pos = torch.arange(9) if s == 0 else torch.tensor([8 + s])
            got = o.forward(idx.view(1, -1).repeat(2, 1), spk, pos)[:, -1]
            assert float((got - ref).abs().max() / ref.abs().max()) < 1e-5


# ---- architecture resolution in _load_model --------------------------------------------------------------------
def _args(**kw):
    a = synth.stage1_model_args(synth.TINY)
    a.update(kw)
    return a


def _keys(norm="rmsnorm", mlp="swiglu", bias=False):
    return {k: None for k in stage1_keys(2, norm, mlp, bias)}


@pytest.mark.parametrize("norm,mlp,bias", ARCHS)
def test_present_keys_are_taken_as_they_are(norm, mlp, bias):
    args = _args(norm_type=norm, nonlinearity_type=mlp, bias=bias)
    assert U.stage1_arch(args, _keys(norm, mlp, bias)) == (norm, mlp, bias)


def test_missing_keys_mean_the_production_architecture():
    args = _args()
    for k in ("norm_type", "nonlinearity_type", "bias"):
        args.pop(k)
    assert U.stage1_arch(args, _keys()) == ("rmsnorm", "swiglu", False)
    assert U.stage1_arch({}, _keys()) == ("rmsnorm", "swiglu", False)
    assert U.stage1_arch({"norm_type": "layernorm"}, _keys()) == ("layernorm", "swiglu", False)


def test_a_contradicting_state_dict_names_the_missing_key():
    with pytest.raises(ValueError, match="nonlinearity_type"):
        U.stage1_arch({"bias": False}, _keys(mlp="gelu"))
    with pytest.raises(ValueError, match="'bias'"):
        U.stage1_arch({"nonlinearity_type": "swiglu"}, _keys(bias=True))
    with pytest.raises(ValueError, match="'bias'"):        # a LayerNorm beta alone is a .bias tensor too
        U.stage1_arch({"norm_type": "layernorm"}, {**_keys(), "transformer.ln_f.bias": None})
    assert U.stage1_arch({"nonlinearity_type": "gelu"}, _keys(mlp="gelu")) == ("rmsnorm", "gelu", False)


@pytest.mark.parametrize("kw,key", [(dict(norm_type="batchnorm"), "norm_type"), (dict(norm_type=None), "norm_type"),
                                    (dict(nonlinearity_type="relu"), "nonlinearity_type"), (dict(bias="yes"), "bias"),
                                    (dict(bias=1), "bias"), (dict(spk_emb_on_text=False), "spk_emb_on_text"),
                                    (dict(vocab_sizes=[2562, 1025]), "vocab_sizes")])
def test_what_the_engine_does_not_build_raises_not_implemented(kw, key):
    with pytest.raises(NotImplementedError, match=key):
        U.stage1_arch(_args(**kw), _keys())


@pytest.mark.parametrize("mode", ["int4", "int8"])
def test_quantisation_of_a_non_production_architecture_raises_before_the_weights_are_read(tmp_path, monkeypatch, mode):
    d = dataclasses.replace(synth.TINY, norm_type="layernorm", nonlinearity_type="gelu", bias=True, intermediate_size=None)
    d.__post_init__()
    path = tmp_path / "first_stage.pt"
    torch.save(synth.stage1_checkpoint(d, 0, tie_head=True), str(path))

    def no_read(*a, **k):
        raise AssertionError("weights read")
    monkeypatch.setattr(Transformer, "from_state_dict", classmethod(no_read))
    with pytest.raises(NotImplementedError, match="production architecture"):
        U._load_model(path, None, "cuda", torch.bfloat16, quantisation_mode=mode)
    with pytest.raises(NotImplementedError, match="production architecture"):
        Transformer.__init__(object.__new__(Transformer), ModelArgs(n_layer=2, n_head=2, dim=256, norm_type="layernorm"),
                             torch.zeros(1, dtype=torch.uint8), [0], "cpu", mode)


def test_load_model_builds_the_config_of_a_gelu_checkpoint(tmp_path, monkeypatch):
    d = dataclasses.replace(synth.TINY, norm_type="layernorm", nonlinearity_type="gelu", bias=True, intermediate_size=None)
    d.__post_init__()
    path = tmp_path / "first_stage.pt"
    torch.save(synth.stage1_checkpoint(d, 0, tie_head=True), str(path))
    seen = {}
    monkeypatch.setattr(Transformer, "from_state_dict",
                        classmethod(lambda cls, sd, config, **kw: seen.update(config=config, keys=set(sd)) or "model"))
    model, _, _ = U._load_model(path, None, "cuda", torch.bfloat16)
    c = seen["config"]
    assert model == "model"
    assert (c.norm_type, c.nonlinearity_type, c.bias, c.intermediate_size) == ("layernorm", "gelu", True, 4 * d.dim)
    assert set(stage1_keys(d.n_layer, "layernorm", "gelu", True)) <= seen["keys"]


# ---- library host checks -----------------------------------------------------------------------------------------
def _cfg(d, max_utts=1):
    return _lib.S1Config(d.n_layer, d.n_head, d.head_dim, d.dim, d.intermediate_size, d.vocab_size, d.block_size,
                         d.speaker_emb_dim, d.norm_eps, max_utts, _lib.MVB_KV_BF16, d.block_size, 0)


def _arch(norm, mlp, bias):
    return _lib.S1Arch({"rmsnorm": 0, "layernorm": 1}[norm], {"swiglu": 0, "gelu": 1}[mlp], int(bias))


def _dims(norm, mlp, bias):
    d = dataclasses.replace(synth.TINY, norm_type=norm, nonlinearity_type=mlp, bias=bias, intermediate_size=None)
    d.__post_init__()
    return d


@pytest.mark.parametrize("norm,mlp,bias", ARCHS)
def test_offset_count_matches_state_dict(norm, mlp, bias):
    """The key list the packer uses holds every tensor of the architecture's state dict once (the head aside, which is
    tied to wtes.0 in the reference), and mvb_s1_create_ex reads exactly that many offsets: an out-of-range entry at the
    last position is rejected, one past it is never read (the call goes on to reject the null workspace, before touching
    a device)."""
    lib = _lib.load()
    d = _dims(norm, mlp, bias)
    sd = synth.stage1_state_dict(d, 0)
    keys = stage1_keys(d.n_layer, norm, mlp, bias)
    assert sorted(keys) == sorted(sd) and len(set(keys)) == len(keys)
    n, arena = len(keys), 1 << 20
    arch, cfg, h = _arch(norm, mlp, bias), _cfg(d), C.c_void_p()
    offs = (C.c_uint64 * (n + 1))(*([256 * i for i in range(n)] + [arena]))     # entry n lies outside the arena
    rc = lib.mvb_s1_create_ex(C.byref(cfg), C.byref(arch), C.c_void_p(256), arena, offs, C.c_void_p(256), None, C.byref(h))
    assert rc == _lib.MVB_ERR_ARG and b"null pointer" in lib.mvb_last_error(), lib.mvb_last_error()
    offs[n - 1] = arena
    rc = lib.mvb_s1_create_ex(C.byref(cfg), C.byref(arch), C.c_void_p(256), arena, offs, C.c_void_p(256), None, C.byref(h))
    assert rc == _lib.MVB_ERR_ARG and b"weight offset" in lib.mvb_last_error(), lib.mvb_last_error()
    assert not h.value


@pytest.mark.parametrize("field,value", [("norm", 2), ("norm", -1), ("mlp", 2), ("mlp", -1), ("bias", 2), ("bias", -1)])
def test_bad_arch_is_rejected_and_named(field, value):
    lib = _lib.load()
    cfg, arch, h = _cfg(synth.TINY), _lib.S1Arch(0, 0, 0), C.c_void_p()
    setattr(arch, field, value)
    offs = (C.c_uint64 * 64)(*([256 * i for i in range(64)]))
    rc = lib.mvb_s1_create_ex(C.byref(cfg), C.byref(arch), C.c_void_p(256), 1 << 20, offs, C.c_void_p(256), C.c_void_p(256),
                              C.byref(h))
    assert rc == _lib.MVB_ERR_ARG
    assert f"arch.{field}".encode() in lib.mvb_last_error(), lib.mvb_last_error()
    assert not h.value


def test_workspace_bytes_for_gelu():
    """A GELU model's intermediate is 4 dim (8192 at production width).  The workspace is sized from cfg.intermediate
    alone, so it needs no arch argument, and the production configuration's size is what it always was."""
    lib = _lib.load()
    prod = synth.FULL
    gelu = _dims("layernorm", "gelu", True)
    gelu_full = dataclasses.replace(synth.FULL, nonlinearity_type="gelu", intermediate_size=None)
    gelu_full.__post_init__()
    assert gelu_full.intermediate_size == 8192 and gelu.intermediate_size == 1024
    size = lambda d, u=1: lib.mvb_s1_workspace_bytes(C.byref(_cfg(d, u)))   # noqa: E731
    assert size(prod) == 66566656                       # the production engine's workspace is unchanged
    assert size(gelu_full) > size(prod) > 0
    # per utterance slot only its 2 ffn rows depend on the width: 2 x (8192 - 5632) x 4 B more
    assert size(gelu_full, 2) - size(gelu_full, 1) - (size(prod, 2) - size(prod, 1)) == 2 * 2560 * 4
    assert size(gelu) > 0
    # the int4 / int8 GEMVs keep the default 48 KB staging buffer: a GELU width there is rejected
    assert lib.mvb_s1_int4_workspace_bytes(C.byref(_cfg(gelu_full))) == 0
    assert lib.mvb_s1_int8_workspace_bytes(C.byref(_cfg(gelu_full))) == 0
