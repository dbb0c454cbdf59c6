"""GPU parity tests proper: the CUDA path, called through the C ABI (ctypes), against
  (1) the committed golden vectors produced by the reference's own code, and
  (2) the CPU oracle restatement on the same seeded inputs,
plus size-independent properties (batched == single, cache-dtype bound, termination).
Tolerance: north_star's 1e-3 relative (max-norm) on pre-sampling logits in validation mode (fp32 KV);
token ids identical under identical noise."""
import numpy as np
import pytest
import torch

from mvb200 import synth

pytestmark = pytest.mark.gpu

TOL = 1e-3


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def _mk(dims, sd, kv="fp32", utts=1, max_new=None, tc=None):
    from mvb200.fast_model import ModelArgs, Transformer
    cfg = ModelArgs(block_size=dims.block_size, vocab_size=dims.vocab_size, n_layer=dims.n_layer, n_head=dims.n_head,
                    dim=dims.dim)
    m = Transformer.from_state_dict(sd, cfg, device="cuda:0")
    m.setup_caches(2 * utts, dims.block_size, kv_dtype=kv, max_new=max_new, tensor_core_path=tc)
    return m


@pytest.fixture(scope="module")
def tiny_sd():
    return synth.stage1_state_dict(synth.TINY, 0)


@pytest.fixture(scope="module")
def full_sd():
    return synth.stage1_state_dict(synth.FULL, 0)


@pytest.fixture(scope="module")
def full_arena(full_sd):
    """The 1.2 B weight arena, packed once and kept on the device for every engine the full-size tests create."""
    from mvb200.fast_model import pack_arena
    arena, offsets = pack_arena(full_sd, synth.FULL.n_layer)
    return arena.cuda(), offsets


def _mk_full(full_arena, kv="bf16", utts=1, max_new=None, tc=None):
    from mvb200.fast_model import ModelArgs, Transformer
    m = Transformer(ModelArgs.from_name("metavoice-1B"), full_arena[0], full_arena[1], device="cuda:0")
    m.setup_caches(2 * utts, synth.FULL.block_size, kv_dtype=kv, max_new=max_new, tensor_core_path=tc)
    return m


def _golden(golden_dir, name):
    return np.load(f"{golden_dir}/{name}.npz")


def _teacher_forced(model, g, last):
    prompt = torch.from_numpy(g["prompt"]).cuda(); spk = torch.from_numpy(g["spk"]).cuda()
    toks = torch.from_numpy(g["tokens"])
    T = prompt.numel()
    out = [model(prompt.view(1, -1).repeat(2, 1), spk, torch.arange(T))[:, -1].cpu()]
    for s in range(1, last + 1):
        t = toks[s - 1].view(1, 1).repeat(2, 1).cuda()
        out.append(model(t, spk, torch.tensor([T + s - 1]))[:, -1].cpu())
    return out


def test_tiny_logits_vs_reference_golden(golden_dir, tiny_sd):
    g = _golden(golden_dir, "stage1_tiny")
    assert synth.state_dict_checksum(tiny_sd) == pytest.approx(float(g["weight_checksum"]), abs=1e-9)
    m = _mk(synth.TINY, tiny_sd, "fp32")
    steps = [int(s) for s in g["steps"]]
    lg = _teacher_forced(m, g, max(steps))
    errs = [_rel(lg[s], torch.from_numpy(g["logits"][i])) for i, s in enumerate(steps)]
    print("tiny fp32-KV rel err per step", errs)
    assert max(errs) < TOL


def test_tiny_all_prefill_positions_vs_oracle(tiny_sd):
    from oracle import stage1_port as P
    d = synth.TINY
    m = _mk(d, tiny_sd, "fp32")
    o = P.Stage1Oracle(tiny_sd, d.n_head, d.norm_eps, torch.float32, faithful_full_cache=False); o.setup_caches()
    prompt, spk = synth.synthetic_prompt(33, seed=3), synth.synthetic_speaker(seed=4)
    idx = prompt.view(1, -1).repeat(2, 1)
    idx[1, 5] = 2100  # rows may carry different tokens through the forward seam
    got = m(idx.cuda(), spk.cuda(), torch.arange(33)).cpu()
    want = o.forward(idx, spk, torch.arange(33))
    assert got.shape == want.shape == (2, 33, d.vocab_size)
    assert _rel(got, want) < TOL
    # cond / uncond rows must differ (speaker conditioning active only on row 0)
    assert (got[0] - got[1]).abs().max() > 1e-3


def test_tiny_bf16_kv_bounded_by_reference_own_gap(golden_dir, tiny_sd):
    g = _golden(golden_dir, "stage1_tiny")
    m = _mk(synth.TINY, tiny_sd, "bf16")
    steps = [int(s) for s in g["steps"]]
    lg = _teacher_forced(m, g, max(steps))
    for i, s in enumerate(steps):
        ref32 = torch.from_numpy(g["logits"][i]); ref16 = torch.from_numpy(g["logits_ref_bf16"][i])
        ours, theirs = _rel(lg[s], ref32), _rel(ref16, ref32)
        print(f"step {s}: engine(bf16 KV) vs fp32 ref {ours:.2e}; reference bf16 vs fp32 ref {theirs:.2e}")
        assert ours <= theirs


def test_sampler_known_answers(golden_dir, tiny_sd):
    from mvb200 import fast_inference_utils as U
    g = _golden(golden_dir, "sampler")
    m = _mk(synth.TINY, tiny_sd, "bf16")
    for c in range(g["idx"].shape[0]):
        gs, temp, tp, tk = [float(v) for v in g["params"][c]]
        logits = torch.from_numpy(g["logits"][c])[:, None, :].cuda()
        tok, probs = U.sample(logits, gs, temp, None if tp < 0 else tp, None if tk == 0 else int(tk), model=m,
                              q=torch.from_numpy(g["noise"][c]))
        assert int(tok) == int(g["idx"][c]), f"case {c}"
        ref = torch.from_numpy(g["probs"][c])
        assert torch.equal(probs.cpu() > 0, ref > 0), f"kept set differs in case {c}"
        np.testing.assert_allclose(probs.cpu().numpy(), ref.numpy(), rtol=2e-5, atol=1e-9)


def test_generate_reproduces_reference_tokens_with_reference_noise(golden_dir, tiny_sd):
    """Feed the engine the Exp(1) draws the reference consumed (recomputed here with the same seed and call
    order): token ids must be identical to the reference's (tests/golden/stage1_tiny.npz)."""
    from mvb200 import fast_inference_utils as U
    g = _golden(golden_dir, "stage1_tiny")
    n = len(g["tokens"]); V = synth.TINY.vocab_size
    torch.manual_seed(1337)
    noise = torch.stack([torch.empty(V).exponential_(1) for _ in range(n)])
    for i, s in enumerate(g["steps"]):
        assert torch.equal(noise[int(s)], torch.from_numpy(g["noise"][i]))  # same generator stream as the reference
    m = _mk(synth.TINY, tiny_sd, "fp32")
    y = U.generate(m, torch.from_numpy(g["prompt"]), torch.from_numpy(g["spk"]), max_new_tokens=n,
                   end_of_audio_token=9999, noise=noise, guidance_scale=float(g["guidance"]),
                   temperature=float(g["temperature"]), top_p=float(g["top_p"]))
    assert y[len(g["prompt"]):].tolist() == g["tokens"].tolist()


def test_batched_mixed_lengths_equal_single_runs(tiny_sd):
    """N utterances x 2 CFG rows with per-utterance positions == each utterance alone (SURVEY.md D3).
    Bit-exact token ids on the deterministic CUDA-core path; the persistent kernel accumulates split-K partials with
    red.add (order varies run to run), so there the sampled ids are compared under teacher forcing and must agree
    except for at most one near-tie."""
    from mvb200 import fast_inference_utils as U
    d = synth.TINY
    lens = [5, 17, 9]
    prompts = [synth.synthetic_prompt(T, seed=20 + i) for i, T in enumerate(lens)]
    spk = torch.cat([synth.synthetic_speaker(seed=30 + i) for i in range(3)])
    n_new = 12
    noise = torch.empty(3, n_new, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(5))
    kw = dict(max_new_tokens=n_new, end_of_audio_token=9999, guidance_scale=2.0, temperature=1.0, top_p=0.9)
    # (a) deterministic path: exact
    mb = _mk(d, tiny_sd, "bf16", utts=3, tc="")
    yb = U.generate_batch(mb, prompts, spk, noise=noise, **kw)
    ms = _mk(d, tiny_sd, "bf16", utts=1, tc="")
    for i in range(3):
        ys = U.generate_batch(ms, [prompts[i]], spk[i:i + 1], noise=noise[i:i + 1], **kw)[0]
        assert ys.tolist() == yb[i].tolist() and len(ys) == n_new
    # (b) persistent fused kernel: teacher-forced with (a)'s tokens, sampler draws compared
    forced = torch.stack([y.to(torch.int32) for y in yb])
    mb = _mk(d, tiny_sd, "bf16", utts=3, tc="BC")
    _, sb = U.generate_batch(mb, prompts, spk, noise=noise, forced=forced, return_sampled=True, **kw)
    ms = _mk(d, tiny_sd, "bf16", utts=1, tc="BC")
    mismatches = 0
    for i in range(3):
        _, ss = U.generate_batch(ms, [prompts[i]], spk[i:i + 1], noise=noise[i:i + 1], forced=forced[i:i + 1],
                                 return_sampled=True, **kw)
        mismatches += sum(int(a != b) for a, b in zip(ss[0].tolist(), sb[i].tolist()))
        mismatches += sum(int(a != b) for a, b in zip(sb[i].tolist(), yb[i].tolist()))
    print("persistent-kernel batched/single/CUDA-core sampled-token mismatches:", mismatches, "of", 6 * n_new)
    assert mismatches <= 2


@pytest.mark.parametrize("lens", [[5, 17, 9], [5, 17, 9, 12, 3, 20, 8]], ids=["batch3_n16", "batch7_n32"])
def test_persistent_kernel_batch_logits_match_single(tiny_sd, lens):
    """Same state, batch of 3 (16-row activation operand) / 7 (32-row variant) vs each utterance alone through the
    persistent kernel: logits agree to reduction-order noise (fp32 KV) / bf16 rounding flips of the appended K,V
    (bf16 KV)."""
    import ctypes as C
    from mvb200 import _lib
    d = synth.TINY
    n = len(lens)
    prompts = [synth.synthetic_prompt(T, seed=20 + i) for i, T in enumerate(lens)]
    spks = [synth.synthetic_speaker(seed=30 + i) for i in range(n)]

    def run(kv, n_slots, which):
        m = _mk(d, tiny_sd, kv, utts=n_slots)
        lib, h, st = m._lib, m.handle, m._stream()
        sp = _lib.Sampling(2.0, 1.0, 0.9, 0, 9999, 1)
        for slot, i in enumerate(which):
            m.forward(prompts[i].view(1, -1).repeat(2, 1).cuda(), spks[i].cuda(), torch.arange(lens[i]), utt=slot)
        outs = []
        for step in range(3):
            for slot, i in enumerate(which):
                _lib.check(lib.mvb_s1_begin(h, slot, 100 + 7 * i + step, lens[i] + step, C.byref(sp), None, None, st))
            lg = torch.empty(2 * len(which), d.vocab_size, device="cuda")
            _lib.check(lib.mvb_s1_step_logits(h, len(which), lg.data_ptr(), st))
            outs.append(lg.cpu())
        return outs

    for kv, tol in (("fp32", 3e-5), ("bf16", 3e-4)):
        batch = run(kv, n, list(range(n)))
        for i in range(n):
            single = run(kv, 1, [i])
            for step in range(3):
                assert _rel(batch[step][2 * i:2 * i + 2], single[step]) < tol


def test_end_of_audio_latch_and_errors(tiny_sd):
    from mvb200 import fast_inference_utils as U
    d = synth.TINY
    m = _mk(d, tiny_sd, "bf16", utts=2)
    prompts = [synth.synthetic_prompt(6, seed=1), synth.synthetic_prompt(8, seed=2)]
    spk = torch.cat([synth.synthetic_speaker(seed=1), synth.synthetic_speaker(seed=2)])
    # teacher-force utterance 0 to emit EOA (2048) as its 3rd token: it must stop there, EOA included (utils:226)
    forced = torch.full((2, 10), 100, dtype=torch.int32); forced[0, 2] = 2048
    y = U.generate_batch(m, prompts, spk, max_new_tokens=10, end_of_audio_token=2048, forced=forced,
                         guidance_scale=3.0, temperature=1.0, top_p=0.95)
    assert y[0].tolist() == [100, 100, 2048] and len(y[1]) == 10
    with pytest.raises(ValueError, match="Prompt is too long"):
        U.generate_batch(m, [synth.synthetic_prompt(2048)], spk[:1], guidance_scale=3.0, temperature=1.0)
    with pytest.raises(ValueError):
        m(torch.zeros(2, 4, dtype=torch.int32).cuda(), spk[:1].cuda(), torch.tensor([0, 2, 3, 4]))
    # last cache slot is usable: a single-token forward at position 2047
    out = m(torch.full((2, 1), 7, dtype=torch.int32).cuda(), spk[:1].cuda(), torch.tensor([2047]))
    assert torch.isfinite(out).all()


def test_fetch_sampled_rejects_a_slice_outside_the_slot(tiny_sd):
    """mvb_s1_fetch_sampled copies `cap` tokens of slot `utt`: a slot past max_utts or a cap past max_new would read
    outside that slot's slice of the sampled-token buffer, so both are argument errors."""
    import ctypes as C
    from mvb200 import _lib
    m = _mk(synth.TINY, tiny_sd, "fp32", utts=2, max_new=16)
    lib, h, st = m._lib, m.handle, m._stream()
    out = np.zeros(17, dtype=np.int32)
    dst = out.ctypes.data_as(C.c_void_p)
    _lib.check(lib.mvb_s1_fetch_sampled(h, 1, dst, 16, st))
    with pytest.raises(ValueError, match="utterance slot 2"):
        _lib.check(lib.mvb_s1_fetch_sampled(h, 2, dst, 16, st))
    with pytest.raises(ValueError, match="cap 17"):
        _lib.check(lib.mvb_s1_fetch_sampled(h, 0, dst, 17, st))


def test_full_size_logits_vs_reference_golden(golden_dir, full_sd):
    """The 1.2 B configuration BASELINE.json quotes, against logits the reference's own Transformer produced in
    fp32 (prefill T=32 and teacher-forced decode steps 1, 8, 64)."""
    g = _golden(golden_dir, "stage1_full")
    assert synth.state_dict_checksum(full_sd) == pytest.approx(float(g["weight_checksum"]), abs=1e-9)
    m = _mk(synth.FULL, full_sd, "fp32")
    steps = [int(s) for s in g["steps"]]
    lg = _teacher_forced(m, g, max(steps))
    errs = [_rel(lg[s], torch.from_numpy(g["logits"][i])) for i, s in enumerate(steps)]
    print("full fp32-KV rel err per step", errs)
    assert max(errs) < TOL
    m.close(); del m
    torch.cuda.empty_cache()
    mb = _mk(synth.FULL, full_sd, "bf16")
    lg = _teacher_forced(mb, g, max(steps))
    for i, s in enumerate(steps):
        ref32 = torch.from_numpy(g["logits"][i]); ref16 = torch.from_numpy(g["logits_ref_bf16"][i])
        ours, theirs = _rel(lg[s], ref32), _rel(ref16, ref32)
        print(f"full step {s}: engine(bf16 KV) {ours:.2e} vs reference-bf16 {theirs:.2e}")
        assert ours <= theirs


@pytest.mark.parametrize("tc", [False, True])
def test_prefill_paths_vs_oracle_chunked(tiny_sd, tc):
    """Prefill through the CUDA-core path (one position at a time) and through the tensor-core rows path (64-token
    chunks; T=70 crosses a chunk boundary), all positions, against the oracle; then a decode step on top of the
    cache each path wrote."""
    from oracle import stage1_port as P
    d = synth.TINY
    m = _mk(d, tiny_sd, "fp32", tc=tc)
    o = P.Stage1Oracle(tiny_sd, d.n_head, d.norm_eps, torch.float32, faithful_full_cache=False); o.setup_caches()
    T = 70
    prompt, spk = synth.synthetic_prompt(T, seed=13), synth.synthetic_speaker(seed=14)
    idx = prompt.view(1, -1).repeat(2, 1)
    got = m(idx.cuda(), spk.cuda(), torch.arange(T)).cpu()
    want = o.forward(idx, spk, torch.arange(T))
    assert _rel(got, want) < TOL
    t = torch.tensor([[1234], [1234]], dtype=torch.int32)
    got = m(t.cuda(), spk.cuda(), torch.tensor([T])).cpu()
    want = o.forward(t, spk, torch.tensor([T]))
    assert _rel(got, want) < TOL


def test_batched_decode_tensor_core_path_equals_cuda_core_path(tiny_sd):
    """CUDA-core kernels only / tensor-core rows path / + persistent fused decode kernel: free-running token ids of the
    first two are identical (both deterministic); the persistent kernel is compared under teacher forcing."""
    from mvb200 import fast_inference_utils as U
    d = synth.TINY
    lens = [7, 21, 12, 30]
    prompts = [synth.synthetic_prompt(T, seed=40 + i) for i, T in enumerate(lens)]
    spk = torch.cat([synth.synthetic_speaker(seed=50 + i) for i in range(4)])
    n_new = 16
    noise = torch.empty(4, n_new, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(6))
    kw = dict(max_new_tokens=n_new, end_of_audio_token=9999, noise=noise, guidance_scale=3.0, temperature=1.0, top_p=0.95)
    ya = U.generate_batch(_mk(d, tiny_sd, "fp32", utts=4, tc=""), prompts, spk, **kw)
    ybb = U.generate_batch(_mk(d, tiny_sd, "fp32", utts=4, tc="B"), prompts, spk, **kw)
    mism_b = sum(int(a.tolist() != b.tolist()) for a, b in zip(ya, ybb))
    forced = torch.stack([y.to(torch.int32) for y in ya])
    _, sc = U.generate_batch(_mk(d, tiny_sd, "fp32", utts=4, tc="BC"), prompts, spk, forced=forced, return_sampled=True, **kw)
    mism_c = sum(int(a != b) for y, s_ in zip(ya, sc) for a, b in zip(y.tolist(), s_.tolist()))
    print(f"sequences differing CUDA-core vs tensor-core rows path: {mism_b}/4; sampled ids differing vs persistent kernel: {mism_c}/{4 * n_new}")
    assert mism_b <= 1 and mism_c <= 2 and all(len(y) == n_new for y in ya)


def _persistent_steps(model, spk, prompt, tokens, n_steps):
    """Prefill, then teacher-forced decode positions through the persistent fused kernel; returns logits per step."""
    import ctypes as C
    from mvb200 import _lib
    T = prompt.numel()
    idx = prompt.view(1, -1).repeat(2, 1).cuda()
    out = [model(idx, spk.cuda(), torch.arange(T))[:, -1].cpu()]
    lib, h, st = model._lib, model.handle, model._stream()
    sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 9999, 1)
    for s in range(1, n_steps + 1):
        _lib.check(lib.mvb_s1_begin(h, 0, int(tokens[s - 1]), T + s - 1, C.byref(sp), None, None, st))
        lg = torch.empty(2, model.config.vocab_size, device="cuda")
        _lib.check(lib.mvb_s1_step_logits(h, 1, lg.data_ptr(), st))
        out.append(lg.cpu())
    return out


def test_persistent_kernel_logits_tiny_vs_reference_golden(golden_dir, tiny_sd):
    g = _golden(golden_dir, "stage1_tiny")
    for kv, tol in (("fp32", TOL), ("bf16", None)):
        m = _mk(synth.TINY, tiny_sd, kv)
        steps = [int(s) for s in g["steps"]]
        lg = _persistent_steps(m, torch.from_numpy(g["spk"]), torch.from_numpy(g["prompt"]), g["tokens"], max(steps))
        for i, s in enumerate(steps):
            ref32 = torch.from_numpy(g["logits"][i])
            err = _rel(lg[s], ref32)
            print(f"persistent kernel tiny kv={kv} step {s}: rel err {err:.2e}")
            bound = tol if tol else _rel(torch.from_numpy(g["logits_ref_bf16"][i]), ref32)
            assert err < bound


def test_persistent_kernel_logits_full_vs_reference_golden(golden_dir, full_sd):
    g = _golden(golden_dir, "stage1_full")
    m = _mk(synth.FULL, full_sd, "fp32")
    steps = [int(s) for s in g["steps"]]
    lg = _persistent_steps(m, torch.from_numpy(g["spk"]), torch.from_numpy(g["prompt"]), g["tokens"], max(steps))
    errs = [_rel(lg[s], torch.from_numpy(g["logits"][i])) for i, s in enumerate(steps)]
    print("persistent kernel, 1.2B, fp32 KV, rel err per step", errs)
    assert max(errs) < TOL


def test_full_generate_reproduces_reference_tokens(golden_dir, full_sd):
    """End to end on the 1.2 B configuration: tensor-core prefill + persistent decode kernel + sampler, fed the
    Exp(1) stream the reference consumed (same seed, same call order) -> the reference's own 65 token ids."""
    from mvb200 import fast_inference_utils as U
    g = _golden(golden_dir, "stage1_full")
    n = len(g["tokens"]); V = synth.FULL.vocab_size
    torch.manual_seed(1337)
    noise = torch.stack([torch.empty(V).exponential_(1) for _ in range(n)])
    for i, s in enumerate(g["steps"]):
        assert torch.equal(noise[int(s)], torch.from_numpy(g["noise"][i]))
    m = _mk(synth.FULL, full_sd, "fp32")
    y = U.generate(m, torch.from_numpy(g["prompt"]), torch.from_numpy(g["spk"]), max_new_tokens=n,
                   end_of_audio_token=9999, noise=noise, guidance_scale=float(g["guidance"]),
                   temperature=float(g["temperature"]), top_p=float(g["top_p"]))
    got = y[len(g["prompt"]):].tolist()
    same = sum(int(a == b) for a, b in zip(got, g["tokens"].tolist()))
    print(f"1.2B generate: {same}/{n} token ids identical to the reference")
    assert got == g["tokens"].tolist()


# ---- the configuration bench.py times: 1.2 B model, bf16 KV cache, persistent fused kernel ------------------------------
@pytest.mark.parametrize("attention", ["mma"])
def test_persistent_kernel_logits_full_bf16_kv_vs_reference_golden(golden_dir, full_arena, attention):
    """k_decode_persistent<bf16 KV, 16 columns> -- the exact kernel instance BENCH times -- at full size, prefill T=48
    then teacher-forced positions through mvb_s1_step_logits, against the reference's fp32 logits.  A bf16 cache
    cannot meet 1e-3 (SURVEY.md D8): the bound is the reference's OWN bf16-vs-fp32 gap at the same step.
    The bf16 cache's attention runs on mma.sync over TMA-swizzled tiles."""
    full_bf16_kv_golden(golden_dir, full_arena, attention)


def full_bf16_kv_golden(golden_dir, full_arena, attention="mma"):
    """test_persistent_kernel_logits_full_bf16_kv_vs_reference_golden; the engine plans for the SM count in effect when
    it is created."""
    g = _golden(golden_dir, "stage1_full")
    m = _mk_full(full_arena, "bf16")
    steps = [int(s) for s in g["steps"]]
    assert int(g["prompt"].shape[0]) == 48 and max(steps) >= 255
    lg = _persistent_steps(m, torch.from_numpy(g["spk"]), torch.from_numpy(g["prompt"]), g["tokens"], max(steps))
    for i, s in enumerate(steps):
        ref32 = torch.from_numpy(g["logits"][i]); ref16 = torch.from_numpy(g["logits_ref_bf16"][i])
        ours, theirs = _rel(lg[s], ref32), _rel(ref16, ref32)
        print(f"persistent kernel 1.2B bf16-KV ({attention} attention) step {s}: engine {ours:.2e} vs reference-bf16 {theirs:.2e}")
        assert ours <= theirs and ours < 1.5e-2


def test_full_size_batch8_mixed_lengths_match_single_runs(full_arena):
    """BASELINE configs[2]: 8 utterances with prompt lengths {24..120} decoded together on the 1.2 B model
    (k_decode_persistent<bf16 KV, 32 columns>) vs each utterance alone (<bf16 KV, 16 columns>): logits agree to
    reduction-order noise + bf16 rounding flips of the appended K/V, for three consecutive positions."""
    import ctypes as C
    from mvb200 import _lib
    d = synth.FULL
    lens = [24, 32, 48, 64, 80, 96, 112, 120]
    n = len(lens)
    prompts = [synth.synthetic_prompt(T, seed=60 + i) for i, T in enumerate(lens)]
    spks = [synth.synthetic_speaker(seed=70 + i) for i in range(n)]

    def run(n_slots, which):
        m = _mk_full(full_arena, "bf16", utts=n_slots)
        lib, h, st = m._lib, m.handle, m._stream()
        sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 9999, 1)
        for slot, i in enumerate(which):
            m.forward(prompts[i].view(1, -1).repeat(2, 1).cuda(), spks[i].cuda(), torch.arange(lens[i]), utt=slot)
        outs = []
        for step in range(3):
            for slot, i in enumerate(which):
                _lib.check(lib.mvb_s1_begin(h, slot, 100 + 7 * i + step, lens[i] + step, C.byref(sp), None, None, st))
            lg = torch.empty(2 * len(which), d.vocab_size, device="cuda")
            _lib.check(lib.mvb_s1_step_logits(h, len(which), lg.data_ptr(), st))
            outs.append(lg.cpu())
        m.close()
        return outs

    batch = run(n, list(range(n)))
    worst = 0.0
    for i in range(n):
        single = run(1, [i])
        for step in range(3):
            worst = max(worst, _rel(batch[step][2 * i:2 * i + 2], single[step]))
    print(f"1.2B batch-8 mixed-length vs single runs: worst logits rel diff {worst:.2e}")
    assert worst < 1e-3


def test_full_size_batch8_generate_matches_single_runs(full_arena):
    """Same configuration end to end through the plugin call: 8 mixed-length prompts, top-p sampling under supplied
    noise, teacher-forced with the single-run tokens; the sampler's own draws must agree (<= 2 near-tie flips)."""
    from mvb200 import fast_inference_utils as U
    d = synth.FULL
    lens = [24, 32, 48, 64, 80, 96, 112, 120]
    n, n_new = len(lens), 20
    prompts = [synth.synthetic_prompt(T, seed=60 + i) for i, T in enumerate(lens)]
    spk = torch.cat([synth.synthetic_speaker(seed=70 + i) for i in range(n)])
    noise = torch.empty(n, n_new, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(9))
    kw = dict(max_new_tokens=n_new, end_of_audio_token=9999, guidance_scale=3.0, temperature=1.0, top_p=0.95)
    ms = _mk_full(full_arena, "bf16", utts=1)
    singles = [U.generate_batch(ms, [prompts[i]], spk[i:i + 1], noise=noise[i:i + 1], **kw)[0] for i in range(n)]
    ms.close()
    forced = torch.stack([y.to(torch.int32) for y in singles])
    mb = _mk_full(full_arena, "bf16", utts=n)
    fed, sampled = U.generate_batch(mb, prompts, spk, noise=noise, forced=forced, return_sampled=True, **kw)
    mism = sum(int(a != b) for y, s_ in zip(singles, sampled) for a, b in zip(y.tolist(), s_.tolist()))
    print(f"1.2B batch-8 generate: {mism}/{n * n_new} sampled ids differ from the single runs")
    assert all(len(y) == n_new for y in fed) and mism <= 2


def test_default_rng_reproduces_reference_tokens_from_torch_seed(golden_dir, tiny_sd):
    """No `noise` argument: the Exp(1) draws are taken from torch's generator in the reference's call order
    (utils:61-65, :347), so torch.manual_seed(s) + generate() returns the reference's ids.  The golden run used the CPU
    generator (the reference executed on CPU), hence rng="torch-cpu"; rng="torch" (the default) draws from the CUDA
    generator exactly as the reference does on a GPU and must be reproducible from the seed."""
    from mvb200 import fast_inference_utils as U
    g = _golden(golden_dir, "stage1_tiny")
    n = len(g["tokens"])
    m = _mk(synth.TINY, tiny_sd, "fp32")
    kw = dict(max_new_tokens=n, end_of_audio_token=9999, guidance_scale=float(g["guidance"]),
              temperature=float(g["temperature"]), top_p=float(g["top_p"]))
    torch.manual_seed(1337)
    y = U.generate(m, torch.from_numpy(g["prompt"]), torch.from_numpy(g["spk"]), rng="torch-cpu", **kw)
    assert y[len(g["prompt"]):].tolist() == g["tokens"].tolist()
    torch.manual_seed(1337)
    a = U.generate(m, torch.from_numpy(g["prompt"]), torch.from_numpy(g["spk"]), **kw)
    torch.manual_seed(1337)
    b = U.generate(m, torch.from_numpy(g["prompt"]), torch.from_numpy(g["spk"]), **kw)
    assert a.tolist() == b.tolist() and len(a) == len(g["prompt"]) + n


def test_batch_runs_to_the_context_end_without_leaving_the_cache(tiny_sd):
    """Two prompts of different lengths, max_new_tokens=None (run to the end of the 2048-slot context): the shorter
    budget latches `done` on the device and its position stays inside the cache while the other utterance keeps
    decoding; both equal their single runs (deterministic CUDA-core path: exact; persistent kernel: teacher-forced)."""
    from mvb200 import fast_inference_utils as U
    d = synth.TINY
    lens = [2040, 2030]
    prompts = [synth.synthetic_prompt(T, seed=80 + i) for i, T in enumerate(lens)]
    spk = torch.cat([synth.synthetic_speaker(seed=90 + i) for i in range(2)])
    max_new = 2048 - min(lens)
    noise = torch.empty(2, max_new, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(3))
    kw = dict(max_new_tokens=None, end_of_audio_token=9999, guidance_scale=3.0, temperature=1.0, top_p=0.95)
    ms = _mk(d, tiny_sd, "bf16", utts=1, tc="")
    singles = []
    for i in range(2):
        room = 2048 - lens[i]
        singles.append(U.generate_batch(ms, [prompts[i]], spk[i:i + 1], noise=noise[i:i + 1, :room], **kw)[0])
        assert len(singles[i]) == room
    mb = _mk(d, tiny_sd, "bf16", utts=2, tc="")
    yb = U.generate_batch(mb, prompts, spk, noise=noise, **kw)
    assert [y.tolist() for y in yb] == [y.tolist() for y in singles]
    forced = torch.zeros(2, max_new, dtype=torch.int32)
    for i in range(2):
        forced[i, :len(singles[i])] = singles[i].to(torch.int32)
    mc = _mk(d, tiny_sd, "bf16", utts=2, tc="BC")
    fed, sampled = U.generate_batch(mc, prompts, spk, noise=noise, forced=forced, return_sampled=True, **kw)
    assert [len(y) for y in fed] == [2048 - T for T in lens]
    mism = sum(int(a != b) for y, s_ in zip(singles, sampled) for a, b in zip(y.tolist(), s_.tolist()))
    assert mism <= 1
    # the cache rows of utterance 1 must not have been touched by utterance 0 running past its budget: rerun 1 alone
    y1 = U.generate_batch(_mk(d, tiny_sd, "bf16", utts=1, tc=""), [prompts[1]], spk[1:2], noise=noise[1:2], **kw)[0]
    assert y1.tolist() == singles[1].tolist()


def test_resident_forward_then_decode_equals_generate(tiny_sd):
    """set_speaker + forward (prefill) followed directly by mvb_s1_decode -- the documented resident flow and what
    bench.py's `value` times -- samples the same tokens as the plugin call mvb_s1_generate (the prefill leaves its
    last-position logits in the buffer the persistent kernel accumulates into; decode must start from zero)."""
    import ctypes as C
    import numpy as np
    from mvb200 import _lib, fast_inference_utils as U
    d = synth.TINY
    T, n_new = 14, 12
    prompt, spk = synth.synthetic_prompt(T, seed=5), synth.synthetic_speaker(seed=6)
    noise = torch.empty(1, n_new, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(8))
    kw = dict(max_new_tokens=n_new, end_of_audio_token=9999, guidance_scale=3.0, temperature=1.0, top_p=0.95)
    ref = U.generate_batch(_mk(d, tiny_sd, "bf16", tc=""), [prompt], spk, noise=noise, **kw)[0]
    m = _mk(d, tiny_sd, "bf16")
    lib, h, st = m._lib, m.handle, m._stream()
    d_noise = noise[0].cuda().contiguous()
    d_forced = ref.to(torch.int32).cuda().contiguous()
    sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 9999, 1)
    m.set_speaker(0, spk)
    _lib.check(lib.mvb_s1_begin(h, 0, -1, 0, C.byref(sp), d_noise.data_ptr(), d_forced.data_ptr(), st))
    idx = prompt.view(1, -1).repeat(2, 1).to(torch.int32).cuda().contiguous()
    _lib.check(lib.mvb_s1_forward(h, 0, idx.data_ptr(), T, 0, None, 0, st))
    _lib.check(lib.mvb_s1_decode(h, 1, n_new, st))
    got = np.zeros(n_new, dtype=np.int32)
    _lib.check(lib.mvb_s1_fetch_sampled(h, 0, got.ctypes.data_as(C.c_void_p), n_new, st))
    mism = sum(int(a != b) for a, b in zip(got.tolist(), ref.tolist()))
    print("resident forward+decode vs generate: sampled-id mismatches", mism, "of", n_new)
    assert mism <= 1


@pytest.mark.parametrize("n", [12, 40])
def test_path_b_decode_above_8_utterances_vs_oracle(tiny_sd, n):
    """Decode bodies for 9..64 utterances run on the tensor-core rows path (k_tc_gemm at 2n = 24 / 80 rows: NC = 4 / 16,
    k_attn_rows at mixed per-row positions).  Three teacher-forced positions through mvb_s1_step_logits for n
    mixed-length utterances (fp32 KV): every utterance's logits against the CPU oracle, and against the same utterance
    decoded alone."""
    import ctypes as C
    from mvb200 import _lib
    from oracle import stage1_port as P
    d = synth.TINY
    lens = [3 + (7 * i) % 29 for i in range(n)]
    prompts = [synth.synthetic_prompt(T, seed=200 + i) for i, T in enumerate(lens)]
    spks = [synth.synthetic_speaker(seed=300 + i) for i in range(n)]
    feed = lambda i, step: 100 + 37 * i + 11 * step      # noqa: E731  teacher-forced token of utterance i at `step`

    def run(n_slots, which):
        m = _mk(d, tiny_sd, "fp32", utts=n_slots)
        lib, h, st = m._lib, m.handle, m._stream()
        sp = _lib.Sampling(2.0, 1.0, 0.9, 0, 9999, 1)
        for slot, i in enumerate(which):
            m.forward(prompts[i].view(1, -1).repeat(2, 1).cuda(), spks[i].cuda(), torch.arange(lens[i]), utt=slot)
        outs = []
        for step in range(3):
            for slot, i in enumerate(which):
                _lib.check(lib.mvb_s1_begin(h, slot, feed(i, step), lens[i] + step, C.byref(sp), None, None, st))
            lg = torch.empty(2 * len(which), d.vocab_size, device="cuda")
            _lib.check(lib.mvb_s1_step_logits(h, len(which), lg.data_ptr(), st))
            outs.append(lg.cpu())
        m.close()
        return outs

    batch = run(n, list(range(n)))
    worst_o = worst_s = 0.0
    for i in range(n):
        o = P.Stage1Oracle(tiny_sd, d.n_head, d.norm_eps, torch.float32, faithful_full_cache=False); o.setup_caches()
        o.forward(prompts[i].view(1, -1).repeat(2, 1), spks[i], torch.arange(lens[i]))
        single = run(1, [i])
        for step in range(3):
            t = torch.full((2, 1), feed(i, step), dtype=torch.int32)
            want = o.forward(t, spks[i], torch.tensor([lens[i] + step]))[:, -1]
            got = batch[step][2 * i:2 * i + 2]
            worst_o = max(worst_o, _rel(got, want))
            worst_s = max(worst_s, _rel(got, single[step]))
    print(f"{n} utterances (R = {2 * n}) on the tensor-core rows path: worst logits rel err vs oracle {worst_o:.2e}, "
          f"vs single runs {worst_s:.2e}")
    assert worst_o < TOL and worst_s < TOL
