"""GPU: the int4 stage-1 engine (quantisation_mode="int4") on the tiny and the 1.2 B synthetic checkpoints.

An int4 engine computes the same function as a bf16 engine whose arena holds W_deq (mvb200/quantize.py), so that engine and
the CPU oracle on W_deq are the references: prefill runs the same tensor-core kernels on the same bf16 weights (bit-identical
logits and KV cache); decode runs k_gemv_w4 instead of k_gemv / the persistent kernel (within 1e-3)."""
import os
import wave

import pytest
import torch

from mvb200 import quantize as Q
from mvb200 import synth

pytestmark = pytest.mark.gpu

TOL = 1e-3


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def _cfg(d):
    from mvb200.fast_model import ModelArgs
    return ModelArgs(block_size=d.block_size, vocab_size=d.vocab_size, n_layer=d.n_layer, n_head=d.n_head, dim=d.dim)


def _mk(d, sd, mode, kv="fp32", utts=1, max_new=None, tc=None):
    from mvb200.fast_model import Transformer
    m = Transformer.from_state_dict(sd, _cfg(d), device="cuda:0", quantisation_mode=mode)
    m.setup_caches(2 * utts, d.block_size, kv_dtype=kv, max_new=max_new, tensor_core_path=tc)
    return m


@pytest.fixture(scope="module", params=["tiny", "full"])
def dims_sd(request):
    d = synth.TINY if request.param == "tiny" else synth.FULL
    sd = synth.stage1_state_dict(d, 0)
    return d, sd, Q.dequantized_state_dict(sd, d.n_layer)


@pytest.mark.parametrize("kv", ["fp32", "bf16"])
def test_prefill_bit_identical_to_wdeq_engine(dims_sd, kv):
    d, sd, sdq = dims_sd
    prompt, spk = synth.synthetic_prompt(70), synth.synthetic_speaker()     # two prefill chunks
    idx = prompt.view(1, -1).repeat(2, 1).cuda()
    m4 = _mk(d, sd, "int4", kv)
    a = m4(idx, spk.cuda(), torch.arange(70))
    kv4 = m4._kv.clone()
    m4.close()
    mq = _mk(d, sdq, None, kv)
    b = mq(idx, spk.cuda(), torch.arange(70))
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "prefill logits differ from the W_deq bf16 engine"
    assert torch.equal(kv4, mq._kv), "KV cache after prefill differs from the W_deq bf16 engine"
    mq.close()
    # quantisation took effect: the unquantised bf16 engine gives different logits on the same inputs
    mb = _mk(d, sd, None, kv)
    c = mb(idx, spk.cuda(), torch.arange(70))
    print(f"{d.dim}: int4 vs unquantised bf16 prefill logits rel diff {_rel(a.cpu(), c.cpu()):.2e}")
    assert _rel(a.cpu(), c.cpu()) > 1e-3


def test_teacher_forced_decode_vs_oracle_and_wdeq_engine(dims_sd):
    """Decode steps 1, 8, 64 and 255 (fp32 KV) within 1e-3 of the CPU oracle on W_deq and of the W_deq bf16 engine."""
    from oracle import stage1_port as P
    d, sd, sdq = dims_sd
    T, last, check = 12, 255, {1, 8, 64, 255}
    prompt, spk = synth.synthetic_prompt(T), synth.synthetic_speaker()
    toks = torch.randint(0, 2048, (last,), generator=torch.Generator().manual_seed(9))
    o = P.Stage1Oracle(sdq, d.n_head, d.norm_eps, torch.float32, faithful_full_cache=False)
    o.setup_caches()
    m4, mq = _mk(d, sd, "int4"), _mk(d, sdq, None)
    idx = prompt.view(1, -1).repeat(2, 1)
    for m in (m4, mq):
        m(idx.cuda(), spk.cuda(), torch.arange(T))
    o.forward(idx, spk, torch.arange(T))
    worst = 0.0
    for s in range(1, last + 1):
        t = toks[s - 1].view(1, 1).repeat(2, 1)
        pos = torch.tensor([T + s - 1])
        a = m4(t.cuda(), spk.cuda(), pos)[:, -1].cpu()
        b = mq(t.cuda(), spk.cuda(), pos)[:, -1].cpu()
        if s in check:
            want = o.forward(t, spk, pos)[:, -1]
            e1, e2 = _rel(a, want), _rel(a, b)
            worst = max(worst, e1, e2)
            assert e1 < TOL and e2 < TOL, (s, e1, e2)
        else:
            o.forward(t, spk, pos)
    print(f"dim {d.dim}: worst rel err vs oracle / W_deq engine {worst:.2e}")


def test_sampled_ids_under_reference_noise(dims_sd):
    """256 tokens with the reference's Exp(1) noise: the int4 engine's sampler draws, teacher-forced with the W_deq bf16
    engine's tokens, differ in at most 2 steps."""
    from mvb200 import fast_inference_utils as U
    d, sd, sdq = dims_sd
    n = 256
    prompt, spk = synth.synthetic_prompt(10), synth.synthetic_speaker().view(1, -1)
    noise = torch.empty(1, n, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(4))
    kw = dict(max_new_tokens=n, end_of_audio_token=9999, guidance_scale=3.0, temperature=1.0, top_p=0.95)
    mq = _mk(d, sdq, None, "bf16", max_new=n)
    want = U.generate_batch(mq, [prompt], spk, noise=noise, **kw)[0]
    mq.close()
    m4 = _mk(d, sd, "int4", "bf16", max_new=n)
    _, got = U.generate_batch(m4, [prompt], spk, noise=noise, forced=want.to(torch.int32)[None], return_sampled=True, **kw)
    diff = sum(int(a != b) for a, b in zip(got[0].tolist(), want.tolist()))
    print(f"dim {d.dim}: {diff} of {n} sampled ids differ from the W_deq bf16 engine")
    assert len(got[0]) == n and diff <= 2


def test_batch_of_8_mixed_lengths_equals_solo_runs():
    from mvb200 import fast_inference_utils as U
    d = synth.TINY
    sd = synth.stage1_state_dict(d, 0)
    lens = [5, 17, 9, 12, 3, 20, 8, 30]
    prompts = [synth.synthetic_prompt(T, seed=20 + i) for i, T in enumerate(lens)]
    spk = torch.cat([synth.synthetic_speaker(seed=30 + i) for i in range(8)])
    n_new = 24
    noise = torch.empty(8, n_new, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(5))
    kw = dict(max_new_tokens=n_new, end_of_audio_token=9999, guidance_scale=2.0, temperature=1.0, top_p=0.9)
    mb = _mk(d, sd, "int4", "bf16", utts=8)
    before = mb._lib.mvb_s1_launch_count(mb.handle)
    yb = U.generate_batch(mb, prompts, spk, noise=noise, **kw)
    launches = mb._lib.mvb_s1_launch_count(mb.handle) - before
    ms = _mk(d, sd, "int4", "bf16", utts=1)
    for i in range(8):
        ys = U.generate_batch(ms, [prompts[i]], spk[i:i + 1], noise=noise[i:i + 1], **kw)[0]
        assert ys.tolist() == yb[i].tolist() and len(ys) == n_new
    # every decode step is the per-layer path: identity slots + embed + 5 kernels per layer + head + sampler
    m = mb._lib.mvb_s1_launch_count
    b0 = m(mb.handle)
    from mvb200 import _lib as L
    L.check(mb._lib.mvb_s1_decode(mb.handle, 8, 3, mb._stream()))
    torch.cuda.synchronize()
    per_burst = m(mb.handle) - b0
    print(f"generate_batch launches {launches}; a 3-step burst: {per_burst}")
    assert per_burst == 1 + 3 * (5 * d.n_layer + 3), per_burst


def test_continuous_batcher_on_int4_engine():
    from mvb200 import fast_inference_utils as U
    from mvb200.serving import ContinuousBatcher
    d = synth.TINY
    sd = synth.stage1_state_dict(d, 0)
    lens, news = [5, 17, 9, 30, 12], [40, 7, 70, 33, 20]
    prompts = [synth.synthetic_prompt(T, seed=100 + i) for i, T in enumerate(lens)]
    spks = [synth.synthetic_speaker(seed=200 + i) for i in range(5)]
    noise = [torch.empty(n, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(300 + i)) for i, n in enumerate(news)]
    kw = dict(guidance_scale=2.5, temperature=1.0, top_p=0.9, end_of_audio_token=9999)
    solo = _mk(d, sd, "int4", "bf16")
    want = [U.generate_batch(solo, [prompts[i]], spks[i], max_new_tokens=news[i], noise=noise[i][None], **kw)[0] for i in range(5)]
    solo.close()
    cb = ContinuousBatcher(_mk(d, sd, "int4", "bf16", utts=2), burst=16)
    ids = [cb.submit(prompts[i], spks[i], max_new_tokens=news[i], noise=noise[i], **kw) for i in range(5)]
    got = cb.run_until_done()
    assert sorted(got) == sorted(ids) and cb.idle
    for i in range(5):
        assert got[ids[i]].tolist() == want[i].tolist(), i


def test_tts_int4_writes_a_wav(tmp_path):
    from mvb200.fast_inference import TTS
    snap = tmp_path / "snapshot"
    snap.mkdir()
    torch.save(synth.stage1_checkpoint(synth.TINY, 0), str(snap / "first_stage.pt"))
    torch.save(synth.stage2_checkpoint(synth.S2_TINY, 1), str(snap / "second_stage.pt"))
    _, enc_sd = synth.encodec_model_and_state_dict(0)
    spk = snap / "spk.pt"
    torch.save(synth.synthetic_speaker(), str(spk))
    with pytest.warns(UserWarning, match="quantisation will degrade"):
        tts = TTS(str(snap), output_dir=str(tmp_path / "out"), encodec_state_dict=enc_sd, device="cuda:0",
                  quantisation_mode="int4")
    assert tts.model.quantisation_mode == "int4"
    assert tts.model_size == tts.model.int4_model_size_bytes(tts.model.config)
    tts.model._cfg.max_new = 256
    path = tts.synthesise("Hello, what's up?", str(spk), top_p=0.95, guidance_scale=3.0, temperature=1.0)
    assert os.path.isfile(path) and path.endswith(".wav")
    with wave.open(path) as w:
        assert w.getframerate() == 24000 and w.getnframes() >= 9600
