"""GPU: the int8 stage-1 engine (quantisation_mode="int8") on the tiny and the 1.2 B synthetic checkpoints.

An int8 engine computes y_j = s_j sum_k x_k q_jk.  When every scale is a power of two, s q is exact in bf16 and that is the
function of a bf16 engine whose arena holds W' = s q; on a path where both engines sum in the same order the results are
bit-identical.  So the checkpoint is rebuilt to have power-of-two scales (each Linear row rescaled so that its largest
magnitude is 127.5 2^e, see pow2_scales), and:
  * prefill runs the same tensor-core kernels on the same operands (q widened to bf16 and scaled in the epilogue, against
    s q): logits and KV-cache bytes are bit-identical;
  * decode runs k_gemv_w8 instead of k_gemv / the persistent kernel: within 1e-3.
The tiny engine is also held against the reference's own int8 model (tests/golden/int8_stage1_tiny.npz)."""
import os
import wave

import numpy as np
import pytest
import torch

from mvb200 import quantize as Q
from mvb200 import synth

pytestmark = pytest.mark.gpu

TOL = 1e-3
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "int8_stage1_tiny.npz")


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


def pow2_scales(sd, n_layer):
    """Every Linear row rescaled so that its largest magnitude is exactly 127.5 2^e (representable in bf16): its int8
    quantisation then has s32 = 2^e exactly, so the stored bf16 scale is the power of two 2^e."""
    out = dict(sd)
    for k, linear, _ in Q._keys(n_layer):
        if linear:
            w = sd[k].to(torch.bfloat16).double()
            amax, i = w.abs().max(1)
            target = 127.5 * torch.exp2(torch.round(torch.log2(amax / 127.5)))
            w2 = (w * (target / amax)[:, None]).float().to(torch.bfloat16)   # |.| <= target, which bf16 holds exactly
            rows = torch.arange(w.shape[0])
            w2[rows, i] = (torch.sign(w[rows, i]) * target).float().to(torch.bfloat16)
            out[k] = w2
    return out


@pytest.fixture(scope="module", params=["tiny", "full"])
def dims_sd(request):
    d = synth.TINY if request.param == "tiny" else synth.FULL
    sd = pow2_scales(synth.stage1_state_dict(d, 0), d.n_layer)
    sdq = Q.int8_dequantized_state_dict(sd, d.n_layer)
    for k, linear, _ in Q._keys(d.n_layer):
        if linear:
            s = Q.quantize_per_channel(sd[k])[1].float()
            assert torch.equal(s, torch.exp2(torch.round(torch.log2(s)))), f"{k}: scales are not powers of two"
    return d, sd, sdq


@pytest.mark.parametrize("kv", ["fp32", "bf16"])
def test_prefill_bit_identical_to_sq_engine(dims_sd, kv):
    d, sd, sdq = dims_sd
    prompt, spk = synth.synthetic_prompt(70), synth.synthetic_speaker()     # two prefill chunks
    idx = prompt.view(1, -1).repeat(2, 1).cuda()
    m8 = _mk(d, sd, "int8", kv)
    a = m8(idx, spk.cuda(), torch.arange(70))
    kv8 = m8._kv.clone()
    m8.close()
    mq = _mk(d, sdq, None, kv)
    b = mq(idx, spk.cuda(), torch.arange(70))
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "prefill logits differ from the s q bf16 engine"
    assert torch.equal(kv8, mq._kv), "KV cache after prefill differs from the s q bf16 engine"
    mq.close()


def test_teacher_forced_decode_vs_sq_engine(dims_sd):
    """Decode steps 1, 8, 64 and 255 (fp32 KV) within 1e-3 of the s q bf16 engine (its persistent kernel)."""
    d, sd, sdq = dims_sd
    T, last, check = 12, 255, {1, 8, 64, 255}
    prompt, spk = synth.synthetic_prompt(T), synth.synthetic_speaker()
    toks = torch.randint(0, 2048, (last,), generator=torch.Generator().manual_seed(9))
    m8, mq = _mk(d, sd, "int8"), _mk(d, sdq, None)
    idx = prompt.view(1, -1).repeat(2, 1)
    for m in (m8, mq):
        m(idx.cuda(), spk.cuda(), torch.arange(T))
    worst = 0.0
    for s in range(1, last + 1):
        t = toks[s - 1].view(1, 1).repeat(2, 1).cuda()
        pos = torch.tensor([T + s - 1])
        a = m8(t, spk.cuda(), pos)[:, -1].cpu()
        b = mq(t, spk.cuda(), pos)[:, -1].cpu()
        if s in check:
            e = _rel(a, b)
            worst = max(worst, e)
            assert e < TOL, (s, e)
    print(f"dim {d.dim}: worst rel err vs the s q engine {worst:.2e}")


def test_logits_differ_from_unquantised_engine():
    d = synth.TINY
    sd = synth.stage1_state_dict(d, 0)
    prompt, spk = synth.synthetic_prompt(20), synth.synthetic_speaker()
    idx = prompt.view(1, -1).repeat(2, 1).cuda()
    a = _mk(d, sd, "int8")(idx, spk.cuda(), torch.arange(20)).cpu()
    b = _mk(d, sd, None)(idx, spk.cuda(), torch.arange(20)).cpu()
    print(f"int8 vs unquantised bf16 prefill logits rel diff {_rel(a, b):.2e}")
    assert _rel(a, b) > 1e-3


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_tiny_vs_reference_int8_model(golden):
    """Prefill and teacher-forced steps 1 / 8 / 64 / 255 (fp32 KV) within 1e-3 of the reference's own int8 model."""
    d = synth.TINY
    sd = synth.stage1_state_dict(d, 0)
    assert float(golden["weight_checksum"]) == synth.state_dict_checksum(sd)
    prompt, spk = torch.from_numpy(golden["prompt"]), torch.from_numpy(golden["spk"])
    toks = torch.from_numpy(golden["tokens"])
    T = prompt.numel()
    m8 = _mk(d, sd, "int8")
    got = m8(prompt.view(1, -1).repeat(2, 1).cuda(), spk.cuda(), torch.arange(T)).cpu()
    e0 = _rel(got, torch.from_numpy(golden["prefill_logits"]))
    assert e0 < TOL, e0
    steps = golden["steps"].tolist()
    worst = e0
    for s in range(1, max(steps) + 1):
        t = toks[s - 1].view(1, 1).repeat(2, 1).cuda()
        a = m8(t, spk.cuda(), torch.tensor([T + s - 1]))[:, -1].cpu()
        if s in steps:
            e = _rel(a, torch.from_numpy(golden["logits"][steps.index(s)]))
            worst = max(worst, e)
            assert e < TOL, (s, e)
    print(f"tiny: worst rel err vs the reference int8 model {worst:.2e} (its own bf16-vs-fp32 gap "
          f"{float(golden['ref_bf16_gap'].max()):.2e})")


def test_sampled_ids_under_reference_noise(golden):
    """256 tokens with the reference's Exp(1) noise, teacher-forced with the reference int8 model's tokens: the engine's
    sampler draws differ from the reference's in at most 2 steps."""
    from mvb200 import fast_inference_utils as U
    d = synth.TINY
    n = int(golden["tokens"].size)
    prompt, spk = torch.from_numpy(golden["prompt"]), torch.from_numpy(golden["spk"]).view(1, -1)
    noise = torch.empty(1, n, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(int(golden["noise_seed"])))
    want = torch.from_numpy(golden["tokens"])
    kw = dict(max_new_tokens=n, end_of_audio_token=9999, guidance_scale=3.0, temperature=1.0, top_p=0.95)
    m8 = _mk(d, synth.stage1_state_dict(d, 0), "int8", "fp32", max_new=n)
    _, got = U.generate_batch(m8, [prompt], spk, noise=noise, forced=want.to(torch.int32)[None], return_sampled=True, **kw)
    diff = sum(int(a != b) for a, b in zip(got[0].tolist(), want.tolist()))
    print(f"{diff} of {n} sampled ids differ from the reference int8 model")
    assert len(got[0]) == n and diff <= 2


def test_batch_of_8_mixed_lengths_equals_solo_runs():
    from mvb200 import fast_inference_utils as U
    from mvb200 import _lib as L
    d = synth.TINY
    sd = synth.stage1_state_dict(d, 0)
    lens = [5, 17, 9, 12, 3, 20, 8, 30]
    prompts = [synth.synthetic_prompt(T, seed=20 + i) for i, T in enumerate(lens)]
    spk = torch.cat([synth.synthetic_speaker(seed=30 + i) for i in range(8)])
    n_new = 24
    noise = torch.empty(8, n_new, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(5))
    kw = dict(max_new_tokens=n_new, end_of_audio_token=9999, guidance_scale=2.0, temperature=1.0, top_p=0.9)
    mb = _mk(d, sd, "int8", "bf16", utts=8)
    yb = U.generate_batch(mb, prompts, spk, noise=noise, **kw)
    ms = _mk(d, sd, "int8", "bf16", utts=1)
    for i in range(8):
        ys = U.generate_batch(ms, [prompts[i]], spk[i:i + 1], noise=noise[i:i + 1], **kw)[0]
        assert ys.tolist() == yb[i].tolist() and len(ys) == n_new
    # every decode step is the per-layer path, never the persistent kernel: identity slots + embed + 5 kernels per layer
    # + head + sampler
    m = mb._lib.mvb_s1_launch_count
    b0 = m(mb.handle)
    L.check(mb._lib.mvb_s1_decode(mb.handle, 8, 3, mb._stream()))
    torch.cuda.synchronize()
    per_burst = m(mb.handle) - b0
    assert per_burst == 1 + 3 * (5 * d.n_layer + 3), per_burst
    b0 = m(ms.handle)
    L.check(ms._lib.mvb_s1_decode(ms.handle, 1, 3, ms._stream()))
    torch.cuda.synchronize()
    assert m(ms.handle) - b0 == 1 + 3 * (5 * d.n_layer + 3)


def test_continuous_batcher_on_int8_engine():
    from mvb200 import fast_inference_utils as U
    from mvb200.serving import ContinuousBatcher
    d = synth.TINY
    sd = synth.stage1_state_dict(d, 0)
    lens, news = [5, 17, 9, 30, 12], [40, 7, 70, 33, 20]
    prompts = [synth.synthetic_prompt(T, seed=100 + i) for i, T in enumerate(lens)]
    spks = [synth.synthetic_speaker(seed=200 + i) for i in range(5)]
    noise = [torch.empty(n, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(300 + i)) for i, n in enumerate(news)]
    kw = dict(guidance_scale=2.5, temperature=1.0, top_p=0.9, end_of_audio_token=9999)
    solo = _mk(d, sd, "int8", "bf16")
    want = [U.generate_batch(solo, [prompts[i]], spks[i], max_new_tokens=news[i], noise=noise[i][None], **kw)[0] for i in range(5)]
    solo.close()
    cb = ContinuousBatcher(_mk(d, sd, "int8", "bf16", utts=2), burst=16)
    ids = [cb.submit(prompts[i], spks[i], max_new_tokens=news[i], noise=noise[i], **kw) for i in range(5)]
    got = cb.run_until_done()
    assert sorted(got) == sorted(ids) and cb.idle
    for i in range(5):
        assert got[ids[i]].tolist() == want[i].tolist(), i


def test_tts_int8_writes_a_wav(tmp_path):
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
                  quantisation_mode="int8")
    assert tts.model.quantisation_mode == "int8"
    assert tts.model_size == tts.model.int8_model_size_bytes(tts.model.config)
    tts.model._cfg.max_new = 256
    path = tts.synthesise("Hello, what's up?", str(spk), top_p=0.95, guidance_scale=3.0, temperature=1.0)
    assert os.path.isfile(path) and path.endswith(".wav")
    with wave.open(path) as w:
        assert w.getframerate() == 24000 and w.getnframes() >= 9600
