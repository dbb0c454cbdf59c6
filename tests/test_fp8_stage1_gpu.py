"""GPU: the fp8 stage-1 engine (quantisation_mode="fp8") on the tiny and the 1.2 B synthetic checkpoints.

An fp8 engine computes y_j = s_j sum_k x_k q_jk.  When every scale is a power of two, s q is exact in bf16 and that is the
function of a bf16 engine whose arena holds W' = s q.  So the checkpoint is rebuilt to have power-of-two scales (each
Linear row rescaled so that its largest magnitude is 448 2^e), and:
  * prefill runs the same tensor-core kernels on the same operands (q widened to bf16 and scaled in the epilogue, against
    s q): logits and KV-cache bytes are bit-identical;
  * decode runs k_gemv_f8 instead of k_gemv / the persistent kernel: within 1e-3.
Batches: up to 8 slots decode through k_gemv_f8, whose outputs for a slot do not depend on the batch, so a batched run
equals solo runs token for token; more than 8 slots take the widened tensor-core path."""
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


def pow2_scales(sd, n_layer):
    """Every Linear row rescaled so that its largest magnitude is exactly 448 2^e (representable in bf16): its fp8
    quantisation then has the scale 2^e exactly."""
    out = dict(sd)
    for k, linear, _ in Q._keys(n_layer):
        if linear:
            w = sd[k].to(torch.bfloat16).double()
            amax, i = w.abs().max(1)
            target = 448 * torch.exp2(torch.round(torch.log2(amax / 448)))
            w2 = (w * (target / amax)[:, None]).float().to(torch.bfloat16)
            w2 = torch.maximum(torch.minimum(w2.float(), target.float()[:, None]), -target.float()[:, None]).to(torch.bfloat16)
            rows = torch.arange(w.shape[0])
            w2[rows, i] = (torch.sign(w[rows, i]) * target).float().to(torch.bfloat16)
            out[k] = w2
    return out


@pytest.fixture(scope="module", params=["tiny", "full"])
def dims_sd(request):
    d = synth.TINY if request.param == "tiny" else synth.FULL
    sd = pow2_scales(synth.stage1_state_dict(d, 0), d.n_layer)
    sdq = Q.fp8_dequantized_state_dict(sd, d.n_layer)
    for k, linear, _ in Q._keys(d.n_layer):
        if linear:
            s = Q.quantize_fp8_per_channel(sd[k])[1].float()
            assert torch.equal(s, torch.exp2(torch.round(torch.log2(s)))), f"{k}: scales are not powers of two"
    return d, sd, sdq


@pytest.mark.parametrize("kv", ["fp32", "bf16"])
def test_prefill_bit_identical_to_sq_engine(dims_sd, kv):
    d, sd, sdq = dims_sd
    prompt, spk = synth.synthetic_prompt(70), synth.synthetic_speaker()     # two prefill chunks
    idx = prompt.view(1, -1).repeat(2, 1).cuda()
    m8 = _mk(d, sd, "fp8", kv)
    a = m8(idx, spk.cuda(), torch.arange(70))
    kv8 = m8._kv.clone()
    m8.close()
    mq = _mk(d, sdq, None, kv)
    b = mq(idx, spk.cuda(), torch.arange(70))
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "prefill logits differ from the s q bf16 engine"
    assert torch.equal(kv8, mq._kv), "KV cache after prefill differs from the s q bf16 engine"
    mq.close()


def test_teacher_forced_decode_vs_sq_engine(dims_sd):
    """Decode steps 1, 8, 64 and 255 (fp32 KV) within 1e-3 of the s q bf16 engine."""
    d, sd, sdq = dims_sd
    T, last, check = 12, 255, {1, 8, 64, 255}
    prompt, spk = synth.synthetic_prompt(T), synth.synthetic_speaker()
    toks = torch.randint(0, 2048, (last,), generator=torch.Generator().manual_seed(9))
    m8, mq = _mk(d, sd, "fp8"), _mk(d, sdq, None)
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


def _batch(d, sd, n, n_new=24, seed=20):
    lens = [5, 17, 9, 12, 3, 20, 8, 30, 11, 6, 14, 25][:n]
    prompts = [synth.synthetic_prompt(T, seed=seed + i) for i, T in enumerate(lens)]
    spk = torch.cat([synth.synthetic_speaker(seed=30 + i) for i in range(n)])
    noise = torch.empty(n, n_new, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(5))
    return prompts, spk, noise, dict(max_new_tokens=n_new, end_of_audio_token=9999, guidance_scale=2.0, temperature=1.0, top_p=0.9)


@pytest.mark.parametrize("dims", ["tiny", "full"])
def test_batch_of_8_equals_solo_runs(dims):
    """8 slots decode in one k_gemv_f8 launch per projection (one launch row: the weights are read once per step) and
    produce, token for token, what each utterance produces alone."""
    from mvb200 import fast_inference_utils as U
    from mvb200 import _lib as L
    d = synth.TINY if dims == "tiny" else synth.FULL
    sd = synth.stage1_state_dict(d, 0)
    prompts, spk, noise, kw = _batch(d, sd, 8)
    mb = _mk(d, sd, "fp8", "bf16", utts=8)
    yb = U.generate_batch(mb, prompts, spk, noise=noise, **kw)
    m = mb._lib.mvb_s1_launch_count
    b0 = m(mb.handle)
    L.check(mb._lib.mvb_s1_decode(mb.handle, 8, 3, mb._stream()))
    torch.cuda.synchronize()
    assert m(mb.handle) - b0 == 1 + 3 * (5 * d.n_layer + 3)    # the per-layer path: 5 kernels per layer
    mb.close()
    ms = _mk(d, sd, "fp8", "bf16", utts=1)
    for i in range(8):
        ys = U.generate_batch(ms, [prompts[i]], spk[i:i + 1], noise=noise[i:i + 1], **kw)[0]
        assert ys.tolist() == yb[i].tolist() and len(ys) == kw["max_new_tokens"], i


def _step_logits(m, n, toks, pos):
    """One decode position for slots [0, n) from tokens toks at positions pos: logits [2 n, vocab]."""
    import ctypes as C
    from mvb200 import _lib as L
    sp = L.Sampling(1.0, 1.0, 0.9, 0, 9999, 0)
    for i in range(n):
        L.check(m._lib.mvb_s1_begin(m.handle, i, int(toks[i]), int(pos[i]), C.byref(sp), None, None, m._stream()))
    out = torch.empty(2 * n, m.config.vocab_size, device="cuda")
    L.check(m._lib.mvb_s1_step_logits(m.handle, n, out.data_ptr(), m._stream()))
    torch.cuda.synchronize()
    return out.cpu()


def test_more_than_8_slots_take_the_widened_path():
    """12 slots: one decode step runs the widened tensor-core rows path (launch count) and matches each slot's k_gemv_f8
    logits, computed in batches of 4, within 1e-3."""
    d = synth.TINY
    sd = synth.stage1_state_dict(d, 0)
    n = 12
    prompts, spk, _, _ = _batch(d, sd, n)
    toks = torch.randint(0, 2048, (n,), generator=torch.Generator().manual_seed(3))
    pos = [p.numel() for p in prompts]

    def prefill(m, ids):
        for j, i in enumerate(ids):
            m(prompts[i].view(1, -1).repeat(2, 1).cuda(), spk[i:i + 1].cuda(), torch.arange(pos[i]), utt=j)

    mb = _mk(d, sd, "fp8", "fp32", utts=n)
    prefill(mb, range(n))
    b0 = mb._lib.mvb_s1_launch_count(mb.handle)
    big = _step_logits(mb, n, toks, pos)
    launches = mb._lib.mvb_s1_launch_count(mb.handle) - b0 - n    # minus the n begins
    assert launches > 1 + 5 * d.n_layer + 3, launches             # the rows path: widen + GEMMs, more than path A's
    mb.close()
    ms = _mk(d, sd, "fp8", "fp32", utts=4)
    for g in range(0, n, 4):
        ids = list(range(g, g + 4))
        prefill(ms, ids)
        small = _step_logits(ms, 4, toks[g:g + 4], pos[g:g + 4])
        e = _rel(big[2 * g:2 * g + 8], small)
        assert e < TOL, (g, e)


def test_continuous_batcher_and_prompt_guidance_on_fp8_engine():
    from mvb200 import fast_inference_utils as U
    from mvb200.serving import ContinuousBatcher
    d = synth.TINY
    sd = synth.stage1_state_dict(d, 0)
    lens, news = [5, 17, 9, 30, 12], [40, 7, 70, 33, 20]
    prompts = [synth.synthetic_prompt(T, seed=100 + i) for i, T in enumerate(lens)]
    spks = [synth.synthetic_speaker(seed=200 + i) for i in range(5)]
    noise = [torch.empty(n, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(300 + i)) for i, n in enumerate(news)]
    kw = dict(guidance_scale=2.5, temperature=1.0, top_p=0.9, end_of_audio_token=9999)
    solo = _mk(d, sd, "fp8", "bf16")
    want = [U.generate_batch(solo, [prompts[i]], spks[i], max_new_tokens=news[i], noise=noise[i][None], **kw)[0] for i in range(5)]
    solo.close()
    cb = ContinuousBatcher(_mk(d, sd, "fp8", "bf16", utts=2), burst=16)
    ids = [cb.submit(prompts[i], spks[i], max_new_tokens=news[i], noise=noise[i], **kw) for i in range(5)]
    got = cb.run_until_done()
    assert sorted(got) == sorted(ids) and cb.idle
    for i in range(5):
        assert got[ids[i]].tolist() == want[i].tolist(), i
    # a prompt-guided request decodes on two slots
    m = _mk(d, sd, "fp8", "bf16", utts=2)
    out = U.generate_batch(m, [prompts[0]], spks[0], max_new_tokens=20, guidance_scale=(3.0, 2.0), end_of_text_token=2561,
                           end_of_audio_token=9999, temperature=1.0, top_p=0.9)[0]
    assert len(out) == 20


def test_tts_fp8_writes_a_wav(tmp_path):
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
                  quantisation_mode="fp8")
    assert tts.model.quantisation_mode == "fp8"
    assert tts.model_size == tts.model.int8_model_size_bytes(tts.model.config)
    tts.model._cfg.max_new = 256
    path = tts.synthesise("Hello, what's up?", str(spk), top_p=0.95, guidance_scale=3.0, temperature=1.0)
    assert os.path.isfile(path) and path.endswith(".wav")
    with wave.open(path) as w:
        assert w.getframerate() == 24000 and w.getnframes() >= 9600
