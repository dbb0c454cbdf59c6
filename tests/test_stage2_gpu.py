"""GPU: stage-2 engine (tensor-core GEMMs + bidirectional attention + sampler) through the C ABI vs golden vectors from
the reference's own GPT and vs the CPU oracle."""
import numpy as np
import pytest
import torch

from mvb200 import synth

pytestmark = pytest.mark.gpu


def assert_differing_draws_are_ties(lg, noise, ours, ref, top_k=200):
    """lg, noise [n_out, rows, V] (the engine's logits and the Exp(1) draws); ours, ref int [n_out, rows].  Identical ids,
    or -- for every differing draw -- an explicit audit that it is a tie the two implementations may legitimately break
    differently given logits that agree to ~3e-6: either the exp-race scores p/q of the two candidates are within 1e-3
    of each other, or one candidate sits on the top-k boundary (its logit within 1e-4 * max|logit| of the k-th largest).
    At most one draw in 1000 may differ.  Returns the number of differing draws."""
    diff = (ours != ref).nonzero().tolist()
    for h, pos in diff:
        row = lg[h, pos].double()
        a, b = int(ours[h, pos]), int(ref[h, pos])
        kth = torch.topk(row, top_k).values[-1]
        on_boundary = min(abs(float(row[a] - kth)), abs(float(row[b] - kth))) < 1e-4 * float(row.abs().max())
        masked = torch.where(row < kth, torch.full_like(row, -float("inf")), row)
        sc = torch.softmax(masked, -1) / noise[h, pos].double()
        near_tie = float(min(sc[a], sc[b]) / max(sc[a], sc[b])) > 1 - 1e-3
        assert on_boundary or near_tie, f"draw ({h},{pos}): ours {a} vs reference {b} is not a tie"
    assert len(diff) <= max(1, ref.numel() // 1000), f"{len(diff)} of {ref.numel()} draws differ"
    return len(diff)


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
    n_diff = assert_differing_draws_are_ties(lg.cpu(), noise, toks[0].cpu(), ref_t)
    print(f"stage-2 {tag}: {ref_t.numel() - n_diff}/{ref_t.numel()} sampled ids identical to the reference")


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


HEAD128 = synth.Stage2Dims(n_layer=2, n_head=2, n_embd=256, block_size=256)
RAGGED = synth.Stage2Dims(block_size=200)     # 128-row GEMM passes straddle utterances; the last attention CTA is partly filled
TOL = 1e-4                                    # logits: max |err| / max |ref| per utterance and hierarchy
SPK_SCALE = 4.0                               # speaker_cond_pos.weight x 4 (exact in bf16): the speaker visibly moves the logits
MAX_BATCH = 8


def _checkpoint(dims):
    ck = synth.stage2_checkpoint(dims, 1)
    ck["model"]["speaker_cond_pos.weight"] = ck["model"]["speaker_cond_pos.weight"] * SPK_SCALE
    return ck


def _oracle(ck, dims):
    from oracle import stage2_port as P
    return P.Stage2Oracle(ck["model"], dims.n_head, dims.rmsnorm_eps, dtype=torch.float64, device="cuda")


def _utterances(m, dims, B, seed=0):
    """idx int32 [B, 2, t] and speakers [B, 1, 256]: utterance j has its own text, code length and speaker."""
    t = dims.block_size
    idx, spk = [], []
    for j in range(B):
        text, cb0, cb1 = synth.synthetic_stage2_input(dims, max(1, t * (3 + 2 * j) // 20), n_text=5 + 3 * j, seed=seed + 100 + j)
        idx.append(m.build_input(text, [cb0, cb1]))
        spk.append(synth.synthetic_speaker(seed=seed + 200 + j))
    return torch.stack(idx), torch.cat(spk)[:, None]


def _rel_err(lg, ref, B):
    """lg fp32 [n_out, B*t, V] from the engine, ref list of n_out float64 [B, t, V] -> [B, n_out] max |err| / max |ref|
    and [B] worst normwise error over the hierarchies."""
    r = torch.stack(ref, 1)                                                   # [B, n_out, t, V]
    d = (lg.double().view(len(ref), B, -1, r.shape[-1]).transpose(0, 1) - r.to(lg.device))
    rel = d.abs().amax((2, 3)) / r.abs().amax((2, 3))
    nw = (d.pow(2).sum((2, 3)).sqrt() / r.pow(2).sum((2, 3)).sqrt()).amax(1)
    return rel.cpu(), nw.cpu()


@pytest.mark.parametrize("tag,dims", [("tiny", synth.S2_TINY), ("head128", HEAD128), ("full", synth.S2_FULL),
                                      ("ragged200", RAGGED)])
def test_stage2_logits_vs_oracle_port(tag, dims):
    """Head size 64 (k_s2_attn<64>) and 128 (k_s2_attn<128>), t = 256, the full t = 1024 and a ragged t = 200, through the
    captured graph of mvb_s2_forward at B = 1, 3 and 8 (one handle, max_batch = 8), against the float64 oracle port (on
    the device) on the same checkpoint, inputs and speakers.  Every utterance and hierarchy must meet the tolerance, and
    an oracle given the speakers rotated by one utterance must not: each utterance's own speaker reaches its rows."""
    from mvb200.second_stage import SecondStage
    ck = _checkpoint(dims)
    m = SecondStage(ck, device="cuda:0", max_batch=MAX_BATCH)
    o = _oracle(ck, dims)
    for B in (1, 3, 8):
        idx, spk = _utterances(m, dims, B)
        _, lg = m.forward_tokens(idx, spk, 1.0, 200, seed=3, return_logits=True)
        rel, nw = _rel_err(lg, o.forward(idx.long(), spk.double()), B)
        print(f"stage-2 {tag} (head size {dims.n_embd // dims.n_head}, t = {dims.block_size}) B={B}: logits rel err vs float64 "
              f"oracle {float(rel.max()):.2e}; per-utterance normwise {[f'{float(v):.1e}' for v in nw]}")
        assert float(rel.max()) < TOL, f"B={B}: (utterance, hierarchy) {divmod(int(rel.argmax()), rel.shape[1])} off"
        if B > 1:
            rot, _ = _rel_err(lg, o.forward(idx.long(), spk.double().roll(1, 0)), B)
            print(f"stage-2 {tag} B={B}: vs the speaker-rotated oracle, per-utterance rel err {[f'{float(v):.1e}' for v in rot.amax(1)]}")
            assert float(rot.max()) > TOL, "an oracle with the speakers rotated also meets the tolerance"
        del lg
        torch.cuda.empty_cache()


@pytest.mark.parametrize("tag,dims", [("head128", HEAD128), ("full", synth.S2_FULL), ("ragged200", RAGGED)])
def test_stage2_batch_rows_equal_solo_runs(tag, dims):
    """Utterance j of a batch of 3 or 8 gives the logits of its solo run.  With t % 128 == 0 every 128-row GEMM pass holds
    rows of one utterance, the GEMM plan does not depend on the row count and split-K is bit-reproducible, so the logits
    are bit-identical; at t = 200 passes straddle utterances and the tolerance applies."""
    from mvb200.second_stage import SecondStage
    ck = _checkpoint(dims)
    m = SecondStage(ck, device="cuda:0", max_batch=MAX_BATCH)
    t = dims.block_size
    idx, spk = _utterances(m, dims, MAX_BATCH, seed=50)
    solo = [m.forward_tokens(idx[j:j + 1], spk[j:j + 1], 1.0, 200, seed=3, return_logits=True)[1] for j in range(MAX_BATCH)]
    for B in (3, 8):
        _, lg = m.forward_tokens(idx[:B], spk[:B], 1.0, 200, seed=3, return_logits=True)
        lg = lg.view(len(dims.target_vocab_sizes), B, t, -1)
        worst, n_equal = 0.0, 0
        for j in range(B):
            a, b = lg[:, j], solo[j]
            n_equal += int(torch.equal(a, b.view_as(a)))
            worst = max(worst, float((a - b.view_as(a)).abs().max() / b.abs().max()))
        print(f"stage-2 {tag} (t = {t}) B={B}: {n_equal}/{B} utterances bit-identical to their solo run, worst rel diff {worst:.2e}")
        if t % 128 == 0:
            assert n_equal == B, f"B={B}: batched logits differ from the solo runs (rel {worst:.2e})"
        assert worst < TOL


@pytest.mark.parametrize("eager", [False, True], ids=["graph", "eager"])
def test_stage2_without_speaker_vs_oracle_port(eager):
    """forward_tokens(idx, None) (k_s2_embed without the speaker term, graphs[0][batch]) at B = 1 and 3 vs the float64
    oracle without a speaker; the oracle with the speakers must not meet the tolerance."""
    from mvb200.second_stage import SecondStage
    dims = synth.S2_TINY
    ck = _checkpoint(dims)
    m = SecondStage(ck, device="cuda:0", max_batch=MAX_BATCH, cuda_graph=not eager)
    o = _oracle(ck, dims)
    for B in (1, 3):
        idx, spk = _utterances(m, dims, B, seed=20)
        _, lg = m.forward_tokens(idx, None, 1.0, 200, seed=3, return_logits=True)
        rel, nw = _rel_err(lg, o.forward(idx.long(), None), B)
        with_spk, _ = _rel_err(lg, o.forward(idx.long(), spk.double()), B)
        print(f"stage-2 no speaker ({'eager' if eager else 'graph'}) B={B}: logits rel err {float(rel.max()):.2e}, per-utterance "
              f"normwise {[f'{float(v):.1e}' for v in nw]}; vs the oracle with speakers {float(with_spk.min()):.1e} or more")
        assert float(rel.max()) < TOL
        assert float(with_spk.min()) > TOL, "the oracle with a speaker term also meets the tolerance"


def test_stage2_graph_signatures():
    """One graph handle and one eager handle (max_batch = 8) driven through (speaker, 3) -> (none, 3) -> (speaker, 1) ->
    (speaker, 8) -> (none, 3) -> (speaker, 3) with new inputs and seeds at every call: the graph cache keyed on
    (speaker, batch) must replay the graph of that signature, so graph and eager agree bit for bit on tokens and logits,
    and the logits meet the tolerance against the oracle for that signature."""
    from mvb200.second_stage import SecondStage
    dims = synth.S2_TINY
    ck = _checkpoint(dims)
    graph = SecondStage(ck, device="cuda:0", max_batch=MAX_BATCH)
    eager = SecondStage(ck, device="cuda:0", max_batch=MAX_BATCH, cuda_graph=False)
    o = _oracle(ck, dims)
    for call, (with_spk, B) in enumerate([(True, 3), (False, 3), (True, 1), (True, 8), (False, 3), (True, 3)]):
        idx, spk = _utterances(graph, dims, B, seed=1000 * call)
        spk = spk if with_spk else None
        tg, lg = graph.forward_tokens(idx, spk, 1.0, 200, seed=call, return_logits=True)
        te, le = eager.forward_tokens(idx, spk, 1.0, 200, seed=call, return_logits=True)
        assert torch.equal(tg, te) and torch.equal(lg, le), f"call {call} (speaker {with_spk}, B={B}): graph != eager"
        rel, _ = _rel_err(lg, o.forward(idx.long(), None if spk is None else spk.double()), B)
        print(f"stage-2 call {call} (speaker {with_spk}, B={B}): graph == eager, logits rel err {float(rel.max()):.2e}")
        assert float(rel.max()) < TOL, f"call {call} (speaker {with_spk}, B={B})"


def test_stage2_token_layout_vs_oracle_sampler():
    """Supplied noise [n_out, B*t, V] (the eager launch sequence) at B = 3: the returned tokens [B, n_out, t] equal
    non_causal_sample of the oracle port on the float64 logits with the same noise, up to audited ties."""
    from mvb200.second_stage import SecondStage
    from oracle import stage2_port as P
    dims = synth.S2_TINY
    ck = _checkpoint(dims)
    m = SecondStage(ck, device="cuda:0", max_batch=MAX_BATCH)
    o = _oracle(ck, dims)
    B, t, n_out, V = 3, dims.block_size, len(dims.target_vocab_sizes), dims.target_vocab_sizes[0]
    idx, spk = _utterances(m, dims, B, seed=7)
    noise = torch.empty(n_out, B * t, V).exponential_(1, generator=torch.Generator().manual_seed(99))
    toks, lg = m.forward_tokens(idx, spk, 1.0, 200, noise=noise, return_logits=True)
    ref = P.non_causal_sample([l.cpu() for l in o.forward(idx.long(), spk.double())], 1.0, 200,
                              noise=[noise[h].view(B, t, V).double() for h in range(n_out)])      # [B, n_out, t]
    assert toks.shape == (B, n_out, t)
    flat = lambda z: z.cpu().long().transpose(0, 1).reshape(n_out, B * t)   # noqa: E731   [B, n_out, t] -> [n_out, B*t]
    n_diff = assert_differing_draws_are_ties(lg.cpu(), noise, flat(toks), flat(ref))
    print(f"stage-2 token layout B={B}: {ref.numel() - n_diff}/{ref.numel()} sampled ids equal to the oracle sampler's")
