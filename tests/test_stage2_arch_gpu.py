"""GPU: the stage-2 engine in every architecture of the reference's GPTConfig (LayerNorm, GELU MLP, Linear biases) through
mvb_s2_create_ex, against golden vectors from the reference's own GPT; graph replay, batching, the production path's
identity through mvb_s2_create, and a TTS snapshot whose second_stage.pt leaves the architecture to GPTConfig."""
import dataclasses

import numpy as np
import pytest
import torch

from mvb200 import synth
from oracle import make_golden_stage2_arch as G

from test_stage2_gpu import assert_differing_draws_are_ties

pytestmark = pytest.mark.gpu

VARIANTS = G.variants()


def _checkpoint(d, drop_arch_keys=False):
    ck = synth.stage2_checkpoint(d, 1)
    ck["model_args"] = G.model_args(d, drop_arch_keys)
    return ck


@pytest.mark.parametrize("tag,dims,frames,drop", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_stage2_arch_vs_reference_golden(golden_dir, tag, dims, frames, drop):
    from mvb200.second_stage import SecondStage
    g = np.load(f"{golden_dir}/stage2_arch.npz")
    ck = _checkpoint(dims, drop)
    assert synth.state_dict_checksum(ck["model"]) == pytest.approx(float(g[f"{tag}_checksum"]), abs=1e-9)
    m = SecondStage(ck, device="cuda:0")
    assert (m.arch.norm, m.arch.mlp, m.arch.bias) == (int(dims.norm_type == "layernorm"), int(dims.nonlinearity_type == "gelu"),
                                                      int(dims.bias))
    torch.manual_seed(4242)
    noise = torch.stack([torch.empty(dims.block_size, v).exponential_(1) for v in dims.target_vocab_sizes])
    toks, lg = m.forward_tokens(torch.from_numpy(g[f"{tag}_idx"]), torch.from_numpy(g[f"{tag}_spk"]), 1.0, 200, noise=noise,
                                return_logits=True)
    got = lg.cpu()[list(G.HEADS)][:, g[f"{tag}_keep"]]
    ref = torch.from_numpy(g[f"{tag}_logits"])
    err = float((got - ref).abs().max() / ref.abs().max())
    ref_t = torch.from_numpy(g[f"{tag}_tokens"]).int()
    n_diff = assert_differing_draws_are_ties(lg.cpu(), noise, toks[0].cpu(), ref_t)
    print(f"stage-2 {tag}: logits rel err {err:.2e}, {ref_t.numel() - n_diff}/{ref_t.numel()} ids identical to the reference")
    assert err < 1e-3
    m.close()


ARCH_TINY = [v for v in VARIANTS if v[0].startswith("tiny")]


def _inputs(m, d, B, seed=0):
    idx, spk = [], []
    for j in range(B):
        text, cb0, cb1 = synth.synthetic_stage2_input(d, 30 + 17 * j, n_text=5 + 3 * j, seed=seed + j)
        idx.append(m.build_input(text, [cb0, cb1]))
        spk.append(synth.synthetic_speaker(seed=seed + 50 + j))
    return torch.stack(idx), torch.cat(spk)[:, None]


@pytest.mark.parametrize("tag,dims,frames,drop", ARCH_TINY, ids=[v[0] for v in ARCH_TINY])
def test_stage2_arch_graph_equals_eager_and_batch_equals_solo(tag, dims, frames, drop):
    """Graph replay == eager launches bit for bit (tokens and logits); a batch of three == three batches of one (t = 256:
    every 128-row pass holds one utterance, so the logits are bit-identical)."""
    from mvb200.second_stage import SecondStage
    ck = _checkpoint(dims)
    graph = SecondStage(ck, device="cuda:0", max_batch=3)
    eager = SecondStage(ck, device="cuda:0", max_batch=3, cuda_graph=False)
    idx, spk = _inputs(graph, dims, 3)
    tg, lg = graph.forward_tokens(idx, spk, 1.0, 200, seed=5, return_logits=True)
    te, le = eager.forward_tokens(idx, spk, 1.0, 200, seed=5, return_logits=True)
    assert torch.equal(tg, te) and torch.equal(lg, le), "graph != eager"
    lg = lg.view(len(dims.target_vocab_sizes), 3, dims.block_size, -1)
    for j in range(3):
        tj, lj = graph.forward_tokens(idx[j:j + 1], spk[j:j + 1], 1.0, 200, seed=5, return_logits=True)
        assert torch.equal(lg[:, j], lj.view_as(lg[:, j])), f"utterance {j}: batched logits != solo run"
    graph.close(); eager.close()


def test_create_ex_with_zero_arch_equals_create_on_production():
    """mvb_s2_create_ex with an all-zero arch and mvb_s2_create build the same engine: tokens and logits bit for bit."""
    from mvb200 import _lib
    from mvb200.second_stage import SecondStage
    d = synth.S2_FULL
    ck = synth.stage2_checkpoint(d, 1)
    ex = SecondStage(ck, device="cuda:0", max_batch=2)
    assert (ex.arch.norm, ex.arch.mlp, ex.arch.bias) == (0, 0, 0)
    plain = SecondStage(ck, device="cuda:0", max_batch=2)
    plain.close()
    plain._create(plain._lib.mvb_s2_create, plain._lib.mvb_s2_destroy, plain.cfg, plain._lib.mvb_s2_workspace_bytes)
    idx, spk = _inputs(ex, d, 2, seed=9)
    for s in (1, 2):
        a = ex.forward_tokens(idx, spk, 1.0, 200, seed=s, return_logits=True)
        b = plain.forward_tokens(idx, spk, 1.0, 200, seed=s, return_logits=True)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    ex.close(); plain.close()
    assert _lib.MVB_S2_NORM_RMS == 0 and _lib.MVB_S2_MLP_SWIGLU == 0


def test_tts_with_gptconfig_default_second_stage(tmp_path):
    """A snapshot whose second_stage.pt has model_args without norm_type, nonlinearity_type and bias (the reference reads
    them as GPTConfig's defaults: layernorm, gelu, bias) loads in TTS and synthesises a wav."""
    import os
    import wave
    from mvb200.fast_inference import TTS
    snap = tmp_path / "snapshot"
    snap.mkdir()
    torch.save(synth.stage1_checkpoint(synth.TINY, 0), str(snap / "first_stage.pt"))
    d = dataclasses.replace(synth.S2_TINY, norm_type="layernorm", nonlinearity_type="gelu", bias=True)
    torch.save(_checkpoint(d, drop_arch_keys=True), str(snap / "second_stage.pt"))
    _, enc_sd = synth.encodec_model_and_state_dict(0)
    spk = snap / "spk.pt"
    torch.save(synth.synthetic_speaker(), str(spk))
    tts = TTS(str(snap), output_dir=str(tmp_path / "out"), encodec_state_dict=enc_sd, device="cuda:0")
    a = tts.llm_second_stage.arch
    assert (a.norm, a.mlp, a.bias) == (1, 1, 1)
    tts.model._cfg.max_new = 256           # the tiny random stage 1 does not emit end-of-audio: bound the run
    path = tts.synthesise("Hello, what's up?", str(spk), top_p=0.95, guidance_scale=3.0, temperature=1.0)
    assert os.path.isfile(path) and path.endswith(".wav")
    with wave.open(path) as w:
        assert w.getframerate() == 24000 and w.getnframes() >= 9600
