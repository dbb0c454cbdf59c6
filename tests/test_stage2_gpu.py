"""GPU: stage-2 engine (tensor-core GEMMs + bidirectional attention + sampler) through the C ABI vs golden vectors from
the reference's own GPT and vs the CPU oracle."""
import numpy as np
import pytest
import torch

from mvb200 import synth

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tag,dims", [("tiny", synth.S2_TINY), ("full", synth.S2_FULL)])
def test_stage2_logits_and_tokens_vs_reference_golden(golden_dir, tag, dims):
    from mvb200.second_stage import SecondStage
    g = np.load(f"{golden_dir}/stage2.npz")
    ck = synth.stage2_checkpoint(dims, 1)
    assert synth.state_dict_checksum(ck["model"]) == pytest.approx(float(g[f"{tag}_checksum"]), abs=1e-9)
    m = SecondStage(ck, device="cuda:0")
    idx = torch.from_numpy(g[f"{tag}_idx"])
    spk = torch.from_numpy(g[f"{tag}_spk"])
    torch.manual_seed(4242)
    noise = torch.stack([torch.empty(dims.block_size, v).exponential_(1) for v in dims.target_vocab_sizes])   # [6, t, V]
    toks, lg = m.forward_tokens(idx, spk, 1.0, 200, noise=noise, return_logits=True)
    keep = g[f"{tag}_keep"]
    got = lg.cpu()[:, keep]
    ref = torch.from_numpy(g[f"{tag}_logits"])
    err = float((got - ref).abs().max() / ref.abs().max())
    print(f"stage-2 {tag}: logits rel err {err:.2e}")
    assert err < 1e-3
    ref_t = torch.from_numpy(g[f"{tag}_tokens"])
    ours = toks[0].cpu()
    diff = (ours != ref_t).nonzero().tolist()
    print(f"stage-2 {tag}: {ref_t.numel() - len(diff)}/{ref_t.numel()} sampled ids identical to the reference")
    # a15 gate: identical ids, or -- for every differing draw -- an explicit audit that it is a tie the two
    # implementations may legitimately break differently given logits that agree to ~3e-6: either the exp-race scores
    # p/q of the two candidates are within 1e-3 of each other, or one candidate sits on the top-k(200) boundary
    # (its logit within 1e-4 * max|logit| of the 200th largest).
    lgc = lg.cpu()
    for h, pos in diff:
        row = lgc[h, pos].double()
        a, b = int(ours[h, pos]), int(ref_t[h, pos])
        kth = torch.topk(row, 200).values[-1]
        on_boundary = min(abs(float(row[a] - kth)), abs(float(row[b] - kth))) < 1e-4 * float(row.abs().max())
        masked = torch.where(row < kth, torch.full_like(row, -float("inf")), row)
        sc = torch.softmax(masked, -1) / noise[h, pos].double()
        near_tie = float(min(sc[a], sc[b]) / max(sc[a], sc[b])) > 1 - 1e-3
        assert on_boundary or near_tie, f"draw ({h},{pos}): ours {a} vs reference {b} is not a tie"
    assert len(diff) <= max(1, ref_t.numel() // 1000)


def test_stage2_batch_and_pipeline_shapes():
    from mvb200.second_stage import SecondStage
    from mvb200.tokenise import TrainedBPETokeniser
    d = synth.S2_TINY
    ck = synth.stage2_checkpoint(d, 1)
    m = SecondStage(ck, device="cuda:0", max_batch=2, tokenizer=TrainedBPETokeniser(**ck["meta"]["tokenizer"]))
    g = torch.Generator().manual_seed(1)
    codes = [torch.randint(0, 1024, (1, 2, n), generator=g) for n in (40, 55, 30)]
    spk = torch.cat([synth.synthetic_speaker(seed=i) for i in range(3)])[:, None]
    out = m.non_causal_sample(texts=["hello there", "what is up", "ok"], encodec_tokens=codes, speaker_embs=spk, seed=3)
    assert len(out) == 3 and all(o.shape[0] == 8 for o in out)
    assert [o.shape[1] for o in out] <= [40, 55, 30] and all(int(o.max()) < 1024 for o in out)
    # rows of a batch are independent: utterance 0 alone gives the same first two (input) codebooks and same length rule
    assert torch.equal(out[0][:2], codes[0][0][:, :out[0].shape[1]])


def test_stage2_graph_replay_equals_eager_launches():
    """The forward pass is replayed as one CUDA graph (sampling parameters live in device memory): same seed -> the same
    tokens as the eager launch sequence, for two different seeds / temperatures through the same captured graph."""
    from mvb200.second_stage import SecondStage
    d = synth.S2_TINY
    ck = synth.stage2_checkpoint(d, 1)
    text, cb0, cb1 = synth.synthetic_stage2_input(d, 50)
    graph = SecondStage(ck, device="cuda:0")
    eager = SecondStage(ck, device="cuda:0", cuda_graph=False)
    idx = graph.build_input(text, [cb0, cb1])[None]
    spk = synth.synthetic_speaker(seed=2)[None]
    for seed, temp in ((7, 1.0), (8, 0.7), (7, 1.0)):
        a = graph.forward_tokens(idx, spk, temp, 200, seed=seed).cpu()
        b = eager.forward_tokens(idx, spk, temp, 200, seed=seed).cpu()
        assert torch.equal(a, b)
    assert not torch.equal(graph.forward_tokens(idx, spk, 1.0, 200, seed=7).cpu(), graph.forward_tokens(idx, spk, 1.0, 200, seed=9).cpu())


@pytest.mark.parametrize("tag,dims", [("tiny", synth.S2_TINY),
                                      ("head128", synth.Stage2Dims(n_layer=2, n_head=2, n_embd=256, block_size=256))])
def test_stage2_logits_vs_oracle_port(tag, dims):
    """Head size 64 (k_s2_attn<64>) and 128 (k_s2_attn<128>) through the captured graph of mvb_s2_forward, against the
    float64 oracle port on the same checkpoint, input and speaker."""
    from mvb200.second_stage import SecondStage
    from oracle import stage2_port as P
    ck = synth.stage2_checkpoint(dims, 1)
    m = SecondStage(ck, device="cuda:0")
    text, cb0, cb1 = synth.synthetic_stage2_input(dims, 50)
    idx = m.build_input(text, [cb0, cb1])[None]
    spk = synth.synthetic_speaker(seed=2)[None]
    _, lg = m.forward_tokens(idx, spk, 1.0, 200, seed=3, return_logits=True)
    o = P.Stage2Oracle(ck["model"], dims.n_head, dims.rmsnorm_eps, dtype=torch.float64)
    ref = torch.stack([l[0] for l in o.forward(idx.long(), spk.double())])
    err = float((lg.cpu().double() - ref).abs().max() / ref.abs().max())
    print(f"stage-2 {tag} (head size {dims.n_embd // dims.n_head}): logits rel err vs float64 oracle {err:.2e}")
    assert err < 1e-4
