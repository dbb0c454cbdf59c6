"""GPU: stage-1 engines with an fp8 KV cache (kv_dtype="fp8") on the tiny and the 1.2 B synthetic checkpoints.

Oracle rule.  A float64 oracle whose _attend stores dequantize_kv_fp8(quantize_kv_fp8(fp32(k))) (and the same for v) is
the function an fp8-cache engine computes: its logits are gated at the bf16-KV tolerance of DESIGN §2 (1e-2), and ids
sampled under recorded Exp(1) draws may differ in at most 2 of 256 positions.  The engine forms k and v in fp32 (on path
B from hi + lo bf16 activation terms), so an element within ~1e-6 of an e4m3 rounding midpoint can round the other way
than in the oracle and then differs from it by one e4m3 step (2^-3 of the element, against 2^-8 for a bf16 rounding
flip).  On the 24-layer 1.2 B synthetic model those flips compound to up to 3.5e-2 on the prefill logits (the bf16-KV
engine's own flips reach 1.5e-2 against the fp32 reference there, test_stage1_gpu.py), so the full-size gate is
FULL_TOL = 5e-2 and up to FULL_IDS = 8 of the 256 sampled ids may differ (4 measured on an H100: near-ties of
argmax(p / q) under logits 1-2e-2 apart); the tiny model is gated at 1e-2 and 2 ids.  Path A against path B (a batch against solo runs) differs by the same
flips: logits within BATCH_TOL = 2e-3 rather than the bf16 batch test's 1e-3, and the sampled-id criterion is unchanged.
The error against the unquantised oracle is printed, not gated: it is the quality cost of the format."""
import dataclasses
import os
import wave

import pytest
import torch

from mvb200 import quantize as Q
from mvb200 import synth
from oracle import stage1_arch_port as AP
from oracle import stage1_port as P

pytestmark = pytest.mark.gpu

TOL = 1e-2
FULL_TOL = 5e-2
FULL_IDS = 8
BATCH_TOL = 2e-3


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


def _kvq(t):
    c, s = Q.quantize_kv_fp8(t.float())
    return Q.dequantize_kv_fp8(c, s).to(t.dtype)


class _F8KV:
    """k and v enter the oracle's cache as the fp8 cache stores them"""

    def _attend(self, li, q, k, v, *rest):
        return super()._attend(li, q, _kvq(k), _kvq(v), *rest)


class F8Oracle(_F8KV, P.Stage1Oracle):
    pass


class F8ArchOracle(_F8KV, AP.Stage1ArchOracle):
    pass


def _cfg(d):
    from mvb200.fast_model import ModelArgs
    return ModelArgs(block_size=d.block_size, vocab_size=d.vocab_size, n_layer=d.n_layer, n_head=d.n_head, dim=d.dim,
                     intermediate_size=d.intermediate_size, norm_eps=d.norm_eps,
                     norm_type=getattr(d, "norm_type", "rmsnorm"), nonlinearity_type=getattr(d, "nonlinearity_type", "swiglu"),
                     bias=getattr(d, "bias", False))


def _mk(d, sd, kv="fp8", utts=1, mode=None, tc=None, max_new=None):
    from mvb200.fast_model import Transformer
    m = Transformer.from_state_dict(sd, _cfg(d), device="cuda:0", quantisation_mode=mode)
    m.setup_caches(2 * utts, d.block_size, kv_dtype=kv, tensor_core_path=tc, max_new=max_new)
    return m


def _dims(name):
    return synth.TINY if name == "tiny" else synth.FULL


@pytest.fixture(scope="module", params=["tiny", "full"])
def dims_sd(request):
    d = _dims(request.param)
    return d, synth.stage1_state_dict(d, 0)


def _layer0(m, d, utts=1):
    """fp8 cache views of layer 0: codes [K|V][row][head][pos][128] uint8, scales [K|V][row][head][pos] int16"""
    rows = 2 * utts
    n_vec = d.n_layer * 2 * rows * d.n_head * d.block_size
    raw = m._kv
    codes = raw[:128 * n_vec].view(d.n_layer, 2, rows, d.n_head, d.block_size, 128)[0]
    scales = raw[128 * n_vec:130 * n_vec].view(torch.int16).view(d.n_layer, 2, rows, d.n_head, d.block_size)[0]
    return codes, scales


def test_layer0_bytes_equal_quantised_fp32_cache(dims_sd):
    """After a 70-token prefill (two chunks), layer 0's codes and scales are bit-identical to quantize_kv_fp8 of the layer-0
    K / V an fp32-cache engine stored: both run the same qkv projection of layer 0."""
    d, sd = dims_sd
    prompt, spk = synth.synthetic_prompt(70), synth.synthetic_speaker()
    idx = prompt.view(1, -1).repeat(2, 1).cuda()
    m32 = _mk(d, sd, "fp32")
    m32(idx, spk.cuda(), torch.arange(70))
    k32 = m32._kv.view(torch.float32).view(d.n_layer, 2, 2, d.n_head, d.block_size, 128)[0, :, :, :, :70].cpu()
    m32.close()
    m8 = _mk(d, sd, "fp8")
    m8(idx, spk.cuda(), torch.arange(70))
    codes, scales = _layer0(m8, d)
    c, s = Q.quantize_kv_fp8(k32)
    assert torch.equal(codes[:, :, :, :70].cpu(), c.view(torch.uint8)), "layer-0 codes differ"
    assert torch.equal(scales[:, :, :, :70].cpu(), s.view(torch.int16)), "layer-0 scales differ"
    m8.close()


def test_logits_and_ids_vs_quantised_oracle(dims_sd):
    """Prefill (48 tokens, every position) and teacher-forced decode steps 1, 8, 64 and 255 against the float64 oracle over
    the quantised cache; ids sampled by the engine's sampler under recorded Exp(1) draws at 256 positions against the
    oracle's draws on its own logits."""
    from mvb200 import fast_inference_utils as U
    d, sd = dims_sd
    T, last, check = 48, 255, {1, 8, 64, 255}
    prompt, spk = synth.synthetic_prompt(T, seed=5), synth.synthetic_speaker(seed=6)
    toks = torch.randint(0, 1024, (last,), generator=torch.Generator().manual_seed(7))
    noise = torch.empty(last + 1, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(8))
    m = _mk(d, sd, "fp8")
    o = F8Oracle(sd, d.n_head, d.norm_eps, torch.float64, faithful_full_cache=False)
    o.setup_caches()
    o32 = P.Stage1Oracle(sd, d.n_head, d.norm_eps, torch.float32, faithful_full_cache=False)   # unquantised, printed only
    o32.setup_caches()
    idx = prompt.view(1, -1).repeat(2, 1)
    got = m(idx.cuda(), spk.cuda(), torch.arange(T)).cpu()
    want = o.forward(idx, spk, torch.arange(T))
    e_pre = _rel(got, want)
    e_pre_unq = _rel(got, o32.forward(idx, spk, torch.arange(T)))
    tol = TOL if d is synth.TINY else FULL_TOL
    errs, errs_unq, mism = {}, {}, 0
    lg, lw = got[:, -1:], want[:, -1:]
    for s in range(last + 1):
        tok, _ = U.sample(lg.cuda(), 3.0, 1.0, 0.95, model=m, q=noise[s])
        wtok, _ = P.sample(lw, torch.tensor(3.0), torch.tensor(1.0), torch.tensor(0.95), q=noise[s].double())
        mism += int(int(tok) != int(wtok))
        if s == last:
            break
        t = toks[s].view(1, 1).repeat(2, 1)
        pos = torch.tensor([T + s])
        lg = m(t.cuda(), spk.cuda(), pos).cpu()
        lw = o.forward(t, spk, pos)
        lu = o32.forward(t, spk, pos)
        if s + 1 in check:
            errs[s + 1], errs_unq[s + 1] = _rel(lg, lw), _rel(lg, lu)
    m.close()
    print(f"dim {d.dim} fp8 KV: prefill rel err {e_pre:.2e} vs the quantised oracle, {e_pre_unq:.2e} vs the unquantised "
          f"(fp32) oracle; decode steps {errs} vs quantised, {errs_unq} vs unquantised; sampled ids differing: {mism}/256")
    assert e_pre < tol and max(errs.values()) < tol, (e_pre, errs)
    assert mism <= (2 if d is synth.TINY else FULL_IDS), mism


def _pow2_rows(sd, n_layer, top):
    """Every Linear row rescaled so that its largest magnitude is exactly top 2^e (top = 448: fp8's scale is then 2^e;
    127.5: int8's): the dequantised s q is then exact in bf16 and the oracle computes the engine's function."""
    out = dict(sd)
    for k, linear, _ in Q._keys(n_layer):
        if linear:
            w = sd[k].to(torch.bfloat16).double()
            amax, i = w.abs().max(1)
            target = top * torch.exp2(torch.round(torch.log2(amax / top)))
            w2 = (w * (target / amax)[:, None]).clamp(-target[:, None], target[:, None])
            w2[torch.arange(w.shape[0]), i] = torch.sign(w[torch.arange(w.shape[0]), i]) * target
            out[k] = w2.float().to(torch.bfloat16)
    return out


def _tf(m, prompt, spk, toks):
    T = prompt.numel()
    out = [m(prompt.view(1, -1).repeat(2, 1).cuda(), spk.cuda(), torch.arange(T))[:, -1].cpu()]
    for i, t in enumerate(toks):
        out.append(m(t.view(1, 1).repeat(2, 1).cuda(), spk.cuda(), torch.tensor([T + i]))[:, -1].cpu())
    return torch.stack(out)


def _tf_oracle(o, prompt, spk, toks):
    T = prompt.numel()
    out = [o.forward(prompt.view(1, -1).repeat(2, 1), spk, torch.arange(T))[:, -1]]
    for i, t in enumerate(toks):
        out.append(o.forward(t.view(1, 1).repeat(2, 1), spk, torch.tensor([T + i]))[:, -1])
    return torch.stack(out)


@pytest.mark.parametrize("mode", [None, "int4", "int8", "fp8", "arch"])
def test_weight_formats_and_architectures(mode):
    """bf16, int4, int8 and fp8 weights, and a LayerNorm + GELU + bias architecture: the fp8-cache engine (prefill on path
    B, decode on path A) against the quantised-cache oracle of the weights the engine computes with (for int8 / fp8 the
    s q of the dequantised state dict on power-of-two scales, exact), 20-token prompt and 32 teacher-forced steps."""
    d = synth.TINY
    if mode == "arch":
        d = dataclasses.replace(d, norm_type="layernorm", nonlinearity_type="gelu", bias=True, intermediate_size=None)
        d.__post_init__()
        sd = synth.stage1_state_dict(d, 6, tie_head=True)
        o = F8ArchOracle(sd, d.n_head, d.norm_eps, torch.float64, norm_type="layernorm", nonlinearity_type="gelu", bias=True)
    else:
        sd = synth.stage1_state_dict(d, 0)
        if mode in ("int8", "fp8"):
            sd = _pow2_rows(sd, d.n_layer, 448.0 if mode == "fp8" else 127.5)
        ref = {None: lambda s: s, "int4": lambda s: Q.dequantized_state_dict(s, d.n_layer),
               "int8": lambda s: Q.int8_dequantized_state_dict(s, d.n_layer),
               "fp8": lambda s: Q.fp8_dequantized_state_dict(s, d.n_layer)}[mode](sd)
        o = F8Oracle(ref, d.n_head, d.norm_eps, torch.float64, faithful_full_cache=False)
    o.setup_caches()
    prompt, spk = synth.synthetic_prompt(20, seed=11), synth.synthetic_speaker(seed=12)
    toks = torch.randint(0, 1024, (32,), generator=torch.Generator().manual_seed(13))
    m = _mk(d, sd, "fp8", mode=None if mode == "arch" else mode)
    got = _tf(m, prompt, spk, toks)
    m.close()
    want = _tf_oracle(o, prompt, spk, toks)
    e = max(_rel(got[i], want[i]) for i in range(got.shape[0]))
    print(f"fp8 KV, weights {mode or 'bf16'}: worst rel err vs the quantised oracle over prefill + 32 steps {e:.2e}")
    assert e < TOL, e


def test_batch_of_8_mixed_lengths_vs_solo_runs():
    """1.2 B: 8 mixed-length utterances decoded as one batch (path B) against each alone (path A), three teacher-forced
    positions: logits within BATCH_TOL.  Then end to end under recorded noise, teacher-forced with the solo tokens: at most 2
    of the 160 sampled ids differ."""
    import ctypes as C
    from mvb200 import _lib
    from mvb200 import fast_inference_utils as U
    d = synth.FULL
    sd = synth.stage1_state_dict(d, 0)
    from mvb200.fast_model import ModelArgs, Transformer, pack_arena
    arena, offsets = pack_arena(sd, d.n_layer)
    arena = arena.cuda()

    def mk(utts):
        m = Transformer(ModelArgs.from_name("metavoice-1B"), arena, offsets, device="cuda:0")
        m.setup_caches(2 * utts, d.block_size, kv_dtype="fp8")
        return m

    lens = [24, 32, 48, 64, 80, 96, 112, 120]
    n = len(lens)
    prompts = [synth.synthetic_prompt(T, seed=60 + i) for i, T in enumerate(lens)]
    spks = [synth.synthetic_speaker(seed=70 + i) for i in range(n)]

    def run(which):
        m = mk(len(which))
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

    batch = run(list(range(n)))
    worst = 0.0
    for i in range(n):
        single = run([i])
        for step in range(3):
            worst = max(worst, _rel(batch[step][2 * i:2 * i + 2], single[step]))
    n_new = 20
    spk = torch.cat(spks)
    noise = torch.empty(n, n_new, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(9))
    kw = dict(max_new_tokens=n_new, end_of_audio_token=9999, guidance_scale=3.0, temperature=1.0, top_p=0.95)
    ms = mk(1)
    singles = [U.generate_batch(ms, [prompts[i]], spk[i:i + 1], noise=noise[i:i + 1], **kw)[0] for i in range(n)]
    ms.close()
    mb = mk(n)
    fed, sampled = U.generate_batch(mb, prompts, spk, noise=noise, forced=torch.stack([y.to(torch.int32) for y in singles]),
                                    return_sampled=True, **kw)
    mb.close()
    mism = sum(int(a != b) for y, s_ in zip(singles, sampled) for a, b in zip(y.tolist(), s_.tolist()))
    print(f"1.2B fp8 KV batch of 8 vs solo runs: worst logits rel diff {worst:.2e}; {mism}/{n * n_new} sampled ids differ")
    assert worst < BATCH_TOL
    assert all(len(y) == n_new for y in fed) and mism <= 2


def test_continuous_batcher_and_prompt_guidance():
    """Tiny, engine without the rows path (per-utterance kernels, so a slot's arithmetic does not depend on the batch): 5
    requests through 2 ContinuousBatcher slots equal the solo runs token for token; a prompt-guided request (two slots)
    against the three-row oracle over quantised caches, a first divergence only at an oracle near-tie."""
    from mvb200 import fast_inference_utils as U
    from mvb200.serving import ContinuousBatcher
    from oracle import prompt_guidance_port as PG
    d = synth.TINY
    sd = synth.stage1_state_dict(d, 0)
    lens, news = [5, 17, 9, 30, 12], [40, 7, 70, 33, 20]
    prompts = [synth.synthetic_prompt(T, seed=100 + i) for i, T in enumerate(lens)]
    spks = [synth.synthetic_speaker(seed=200 + i) for i in range(5)]
    noise = [torch.empty(n, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(300 + i)) for i, n in enumerate(news)]
    kw = dict(guidance_scale=2.5, temperature=1.0, top_p=0.9, end_of_audio_token=9999)
    solo = _mk(d, sd, "fp8", tc="")
    want = [U.generate_batch(solo, [prompts[i]], spks[i], max_new_tokens=news[i], noise=noise[i][None], **kw)[0] for i in range(5)]
    solo.close()
    cb = ContinuousBatcher(_mk(d, sd, "fp8", utts=2, tc=""), burst=16)
    ids = [cb.submit(prompts[i], spks[i], max_new_tokens=news[i], noise=noise[i], **kw) for i in range(5)]
    got = cb.run_until_done()
    assert sorted(got) == sorted(ids) and cb.idle
    for i in range(5):
        assert got[ids[i]].tolist() == want[i].tolist(), i
    cb.model.close()
    EOA, EOT, gs, n_new = 9999, 2561, (3.0, 2.0), 20
    prompt, spk = synth.synthetic_prompt(11, seed=130), synth.synthetic_speaker(seed=131)
    nz = torch.empty(n_new, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(132))
    m = _mk(d, sd, "fp8", utts=2)
    out = U.generate_batch(m, [prompt], spk, max_new_tokens=n_new, end_of_audio_token=EOA, noise=nz[None], guidance_scale=gs,
                           end_of_text_token=EOT, temperature=1.0, top_p=None)[0].tolist()
    m.close()
    mk = lambda: F8ArchOracle(sd, d.n_head, d.norm_eps, torch.float64)   # noqa: E731
    o, oc = mk(), mk()
    o.setup_caches()
    oc.setup_caches()
    sink = []
    ref = PG.generate3(o, oc, prompt, spk, guidance_scale=gs, end_of_text_token=EOT, max_new_tokens=n_new,
                       end_of_audio_token=EOA, noise=nz.double(), temperature=1.0, top_p=None, logit_sink=sink)[11:].tolist()
    assert len(out) == n_new
    k = next((i for i, (a, b) in enumerate(zip(out, ref)) if a != b), None)
    print(f"prompt-guided request on fp8 KV: first divergence from the quantised-cache oracle at {k}")
    if k is not None:
        _, pr = PG.sample3(sink[k][0][:, None], gs, 1.0, None)
        score = (pr / nz[k].double()).sort(descending=True).values
        assert float(score[0] / score[1] - 1) < 1e-2, (k, out, ref)


def test_tts_fp8_kv_writes_wavs(tmp_path):
    from mvb200.fast_inference import TTS
    snap = tmp_path / "snapshot"
    snap.mkdir()
    torch.save(synth.stage1_checkpoint(synth.TINY, 0), str(snap / "first_stage.pt"))
    torch.save(synth.stage2_checkpoint(synth.S2_TINY, 1), str(snap / "second_stage.pt"))
    _, enc_sd = synth.encodec_model_and_state_dict(0)
    spk = snap / "spk.pt"
    torch.save(synth.synthetic_speaker(), str(spk))
    tts = TTS(str(snap), output_dir=str(tmp_path / "out"), encodec_state_dict=enc_sd, device="cuda:0", kv_dtype="fp8",
              max_utts=4)
    assert tts.model.kv_dtype == "fp8" and tts.model._cfg.kv_dtype == 2
    tts.model._cfg.max_new = 256
    path = tts.synthesise("Hello, what's up?", str(spk), top_p=0.95, guidance_scale=3.0, temperature=1.0)
    paths = tts.synthesise_batch(["One two.", "Three four five."], [str(spk)] * 2, top_p=0.95, guidance_scale=3.0, temperature=1.0)
    for p in [path] + list(paths):
        assert os.path.isfile(p) and p.endswith(".wav")
        with wave.open(p) as w:
            assert w.getframerate() == 24000 and w.getnframes() > 0
