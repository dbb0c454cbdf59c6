"""GPU: one stage-1 engine serving last-N-block finetunes (voices) and batching utterances across them.

Voice 0 is the base checkpoint; voices 1 and 2 overlay its last block and its last two blocks plus ln_f (the synthetic
finetunes of tests/test_voices_cpu.py).  A batch on voice 0 alone is unchanged; on the CUDA-core path a mixed batch
gives every utterance exactly what a single-voice engine built from its voice's full checkpoint gives; on the
tensor-core rows path (one grouped launch per projection) it agrees with the float64 oracle of that checkpoint, logits
and sampled ids; the serving layers route voices through.  The engine tests run in every architecture
mvb_s1_create_ex builds (TINY width) and at production width."""
import ctypes as C
import dataclasses
import os
import wave

import pytest
import torch

from mvb200 import _lib, synth
from mvb200 import fast_inference_utils as U
from mvb200.fast_model import ModelArgs, Transformer
from oracle import stage1_arch_port as A
from test_voices_cpu import finetune

pytestmark = pytest.mark.gpu

D = synth.TINY
N_NEW = 12
LENS = [5, 17, 9, 12, 3, 20, 8, 14]
VOICES = [0, 1, 2, 2, 1, 0, 1, 2]
ARCHS = [("rmsnorm", "swiglu", False), ("layernorm", "gelu", True), ("rmsnorm", "swiglu", True),
         ("layernorm", "swiglu", False)]
ARCH_IDS = ["-".join(str(x) for x in a) for a in ARCHS]


def _dims(arch=ARCHS[0], base=synth.TINY):
    d = dataclasses.replace(base, norm_type=arch[0], nonlinearity_type=arch[1], bias=arch[2], intermediate_size=None)
    d.__post_init__()
    return d


def _config(d):
    return ModelArgs(block_size=d.block_size, vocab_size=d.vocab_size, n_layer=d.n_layer, n_head=d.n_head, dim=d.dim,
                     intermediate_size=d.intermediate_size, norm_eps=d.norm_eps, norm_type=d.norm_type,
                     nonlinearity_type=d.nonlinearity_type, bias=d.bias)


_SDS = {}


def _sds(d=D):
    """Base, N = 1 and N = 2 finetunes (kept: the production-width ones take a while to draw)."""
    key = repr(d)
    if key not in _SDS:
        base = synth.stage1_state_dict(d, 0)
        _SDS[key] = [base, finetune(d, 0, 1, seed=41), finetune(d, 0, 2, seed=42)]
    return _SDS[key]


def _mk(sd, kv="bf16", utts=8, tc=None, voices=(), d=D):
    m = Transformer.from_state_dict(sd, _config(d), device="cuda")
    m.setup_caches(2 * utts, d.block_size, kv_dtype=kv, tensor_core_path=tc, max_new=64)
    for v in voices:
        m.add_voice(v)
    return m


def _inputs(n=8, d=D, n_new=N_NEW):
    prompts = [synth.synthetic_prompt(T, seed=200 + i) for i, T in enumerate(LENS[:n])]
    spk = torch.cat([synth.synthetic_speaker(seed=210 + i) for i in range(n)])
    noise = torch.empty(n, n_new, d.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(9))
    return prompts, spk, noise


KW = dict(end_of_audio_token=9999, guidance_scale=3.0, temperature=1.0, top_p=0.95)


def _step_logits(m, n, toks, n_new=N_NEW, d=D):
    """One decode position of slots [0, n) after generate_batch: token toks[i] at the first position its decode has not
    written (prompt + n_new - 1), so that the attention reads only this utterance's own cache; logits [2n, V]."""
    lib, h, st = m._lib, m.handle, m._stream()
    sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 9999, 1)
    for i in range(n):
        _lib.check(lib.mvb_s1_begin(h, i, int(toks[i]), LENS[i] + n_new - 1, C.byref(sp), None, None, st))
    lg = torch.empty(2 * n, d.vocab_size, device="cuda")
    _lib.check(lib.mvb_s1_step_logits(h, n, lg.data_ptr(), st))
    torch.cuda.synchronize()
    return lg.cpu()


@pytest.mark.parametrize("n", [1, 8])
def test_voice_0_is_unchanged_by_registered_voices(n):
    """Deterministic paths (no resident kernel, whose red.add order varies from run to run): tokens, logits and KV bytes
    of an engine with two voices registered and every slot on voice 0 equal those of an engine without voices."""
    sds = _sds()
    prompts, spk, noise = _inputs(n)
    out = []
    for voices in ((), sds[1:]):
        m = _mk(sds[0], utts=n, tc="B", voices=voices)
        toks = U.generate_batch(m, prompts, spk, noise=noise, max_new_tokens=N_NEW, **KW)
        lg = _step_logits(m, n, [t[-1] for t in toks])
        out.append(([t.tolist() for t in toks], lg, m._kv.cpu().clone()))
        m.close()
    assert out[0][0] == out[1][0]
    assert torch.equal(out[0][1], out[1][1])
    assert torch.equal(out[0][2], out[1][2])


@pytest.mark.parametrize("n", [1, 8])
def test_voice_0_keeps_the_resident_kernel_on_default_paths(n):
    """Default paths: a burst of voice-0 slots launches exactly what an engine without voices launches (one resident
    kernel per burst), also after a slot on a finetuned voice has been released; a finetuned slot in the batch moves it
    to the per-layer path."""
    sds = _sds()
    counts = {}
    for tag, voices, sel in (("plain", (), [0] * n), ("voices", sds[1:], [0] * n), ("released", sds[1:], [1] + [0] * (n - 1)),
                             ("finetuned", sds[1:], [1] + [0] * (n - 1))):
        m = _mk(sds[0], utts=n, voices=voices)
        lib, h, st = m._lib, m.handle, m._stream()
        sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 9999, 1)
        for u in range(n):
            if voices:
                m.set_voice(u, sel[u])
            _lib.check(lib.mvb_s1_begin(h, u, 17 + u, 6, C.byref(sp), None, None, st))
        if tag == "released":      # a finished request's slot, parked: it must not hold its voice
            _lib.check(lib.mvb_s1_release(h, 0, st))
        _lib.check(lib.mvb_s1_decode(h, n, 1, st))
        before = lib.mvb_s1_launch_count(h)
        _lib.check(lib.mvb_s1_decode(h, n, 8, st))
        torch.cuda.synchronize()
        counts[tag] = lib.mvb_s1_launch_count(h) - before
        m.close()
    print(counts)
    assert counts["plain"] == counts["voices"] == counts["released"] < 8 * 5 * D.n_layer
    assert counts["finetuned"] >= 8 * 5 * D.n_layer


def _path_a_exact(d, kv, n, n_new):
    sds = _sds(d)
    prompts, spk, noise = _inputs(n, d, n_new)
    m = _mk(sds[0], kv, utts=n, tc="", voices=sds[1:], d=d)
    toks = U.generate_batch(m, prompts, spk, noise=noise, voices=VOICES[:n], max_new_tokens=n_new, **KW)
    lg = _step_logits(m, n, [t[-1] for t in toks], n_new, d)
    m.close()
    for v in range(3):
        ms = _mk(sds[v], kv, utts=1, tc="", d=d)
        for i in [i for i in range(n) if VOICES[i] == v]:
            solo = U.generate_batch(ms, [prompts[i]], spk[i:i + 1], noise=noise[i:i + 1], max_new_tokens=n_new, **KW)[0]
            assert solo.tolist() == toks[i].tolist(), (kv, v, i)
            sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 9999, 1)
            lib, h, st = ms._lib, ms.handle, ms._stream()
            _lib.check(lib.mvb_s1_begin(h, 0, int(toks[i][-1]), LENS[i] + n_new - 1, C.byref(sp), None, None, st))
            one = torch.empty(2, d.vocab_size, device="cuda")
            _lib.check(lib.mvb_s1_step_logits(h, 1, one.data_ptr(), st))
            torch.cuda.synchronize()
            assert torch.equal(one.cpu(), lg[2 * i:2 * i + 2]), (kv, v, i)
        ms.close()


@pytest.mark.parametrize("arch", ARCHS, ids=ARCH_IDS)
@pytest.mark.parametrize("kv", ["bf16", "fp8"])
def test_path_a_mixed_batch_equals_single_voice_engines(kv, arch):
    """CUDA-core path (tensor_core_path=False): 8 utterances over 3 voices decode together exactly as each alone on an
    engine built from its voice's full checkpoint: tokens, then one more position's logits, bit for bit."""
    _path_a_exact(_dims(arch), kv, 8, N_NEW)


def test_path_a_mixed_batch_at_production_width():
    _path_a_exact(synth.FULL, "bf16", 3, 4)


def _oracle(sd, d):
    o = A.Stage1ArchOracle(sd, d.n_head, d.norm_eps, torch.float64, norm_type=d.norm_type,
                           nonlinearity_type=d.nonlinearity_type, bias=d.bias)
    o.setup_caches()
    return o


@pytest.mark.parametrize("arch", ARCHS, ids=ARCH_IDS)
def test_path_b_mixed_batch_against_the_float64_oracle(arch):
    """Default paths (tensor-core rows path from 2 utterances, one grouped launch per projection): prefill each slot on
    its voice, then one decode position of the mixed batch; every utterance's logits within 1e-3 of the float64 oracle of
    its voice's full checkpoint (fp32 cache).  Then 8 teacher-forced steps under supplied noise: at most 2 of the 64
    sampled ids differ from those the oracle's sampler draws from its own logits."""
    d = _dims(arch)
    sds = _sds(d)
    prompts, spk, noise = _inputs(8, d, 9)
    m = _mk(sds[0], "fp32", voices=sds[1:], d=d)
    lib, h, st = m._lib, m.handle, m._stream()
    sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 9999, 1)
    for i in range(8):
        m.set_voice(i, VOICES[i])
        _lib.check(lib.mvb_s1_begin(h, i, -1, 0, C.byref(sp), None, None, st))   # latches the voice
        m(prompts[i].view(1, -1).repeat(2, 1).cuda(), spk[i:i + 1].cuda(), torch.arange(LENS[i]), utt=i)
    toks = [100 + 13 * i for i in range(8)]
    for i in range(8):
        _lib.check(lib.mvb_s1_begin(h, i, toks[i], LENS[i], C.byref(sp), None, None, st))
    lg = torch.empty(16, d.vocab_size, device="cuda")
    _lib.check(lib.mvb_s1_step_logits(h, 8, lg.data_ptr(), st))
    lg = lg.cpu().double()
    forced = torch.randint(0, 2048, (8, 9), generator=torch.Generator().manual_seed(5), dtype=torch.int32)
    _, sampled = U.generate_batch(m, [p.to(torch.int32) for p in prompts], spk, noise=noise, forced=forced,
                                  max_new_tokens=9, voices=VOICES, return_sampled=True, **KW)
    m.close()
    diff = 0
    for i in range(8):
        o = _oracle(sds[VOICES[i]], d)
        o.forward(prompts[i].view(1, -1).repeat(2, 1), spk[i:i + 1], torch.arange(LENS[i]))
        want = o.forward(torch.tensor([[toks[i]], [toks[i]]]), spk[i:i + 1], torch.tensor([LENS[i]]))[:, -1]
        err = float((lg[2 * i:2 * i + 2] - want).abs().max() / want.abs().max())
        print(f"utterance {i} voice {VOICES[i]}: rel err {err:.2e}")
        assert err < 1e-3, (i, err)
        # the sampler's draws: prefill sample, then 8 steps fed the forced tokens
        o = _oracle(sds[VOICES[i]], d)
        T = LENS[i]
        lgo = o.forward(prompts[i].view(1, -1).repeat(2, 1), spk[i:i + 1], torch.arange(T))
        ids = []
        for s_ in range(9):
            w, _ = _sample(lgo, noise[i, s_])
            ids.append(int(w))
            if s_ < 8:
                t = int(forced[i, s_])
                lgo = o.forward(torch.tensor([[t], [t]]), spk[i:i + 1], torch.tensor([T + s_]))
        diff += sum(int(a != b) for a, b in zip(sampled[i].tolist(), ids))
    print("sampled-id mismatches:", diff, "of 72")
    assert diff <= 2


def _sample(lg, q):
    from oracle import stage1_port as P
    return P.sample(lg, torch.tensor(3.0), torch.tensor(1.0), torch.tensor(0.95), q=q.double())


def test_path_b_mixed_batch_at_production_width():
    """Production width (split-K active): a decode position of 3 slots on 3 voices through the grouped launches agrees
    with engines built from each voice's full checkpoint, decoding that slot alone on the rows path, within 1e-3."""
    d = synth.FULL
    sds = _sds(d)
    prompts, spk, _ = _inputs(3, d)
    sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 9999, 1)

    def run(m, slots, voices):
        lib, h, st = m._lib, m.handle, m._stream()
        for j, i in enumerate(slots):
            if voices is not None:
                m.set_voice(j, voices[j])
            _lib.check(lib.mvb_s1_begin(h, j, -1, 0, C.byref(sp), None, None, st))
            m(prompts[i].view(1, -1).repeat(2, 1).cuda(), spk[i:i + 1].cuda(), torch.arange(LENS[i]), utt=j)
        for j, i in enumerate(slots):
            _lib.check(lib.mvb_s1_begin(h, j, 100 + 13 * i, LENS[i], C.byref(sp), None, None, st))
        n = max(2, len(slots))      # a single slot decodes beside a parked copy, so that it too takes the rows path
        if len(slots) == 1:
            _lib.check(lib.mvb_s1_begin(h, 1, 5, 0, C.byref(sp), None, None, st))
        lg = torch.empty(2 * n, d.vocab_size, device="cuda")
        _lib.check(lib.mvb_s1_step_logits(h, n, lg.data_ptr(), st))
        torch.cuda.synchronize()
        return lg.cpu().double()

    m = _mk(sds[0], "fp32", utts=3, tc="B", voices=sds[1:], d=d)
    got = run(m, [0, 1, 2], [0, 1, 2])
    m.close()
    for v in range(3):
        ms = _mk(sds[v], "fp32", utts=2, tc="B", d=d)
        want = run(ms, [v], None)[:2]
        ms.close()
        err = float((got[2 * v:2 * v + 2] - want).abs().max() / want.abs().max())
        print(f"voice {v}: rel err {err:.2e}")
        assert err < 1e-3, (v, err)


def test_continuous_batcher_refills_slots_across_voices():
    from mvb200.serving import ContinuousBatcher
    sds = _sds()
    lens, news, vs = [6, 13, 4, 9, 11], [10, 5, 12, 7, 9], [1, 2, 0, 2, 1]
    prompts = [synth.synthetic_prompt(T, seed=100 + i) for i, T in enumerate(lens)]
    spks = [synth.synthetic_speaker(seed=110 + i) for i in range(5)]
    noise = [torch.empty(n, D.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(120 + i))
             for i, n in enumerate(news)]
    kw = dict(guidance_scale=3.0, temperature=1.0, top_p=0.95, end_of_audio_token=9999)
    m = _mk(sds[0], utts=2, tc="", voices=sds[1:])
    cb = ContinuousBatcher(m, burst=4)
    ids = [cb.submit(prompts[i], spks[i], max_new_tokens=news[i], noise=noise[i].cuda(), voice=vs[i], **kw) for i in range(5)]
    done = cb.run_until_done()
    for i in range(5):
        solo = U.generate_batch(m, [prompts[i]], spks[i], max_new_tokens=news[i], noise=noise[i][None], voices=[vs[i]], **kw)[0]
        assert done[ids[i]].tolist() == solo.tolist(), i
    with pytest.raises(KeyError):
        cb.submit(prompts[0], spks[0], voice=3)
    m.close()


def test_prompt_guided_request_runs_its_companion_on_its_voice():
    sds = _sds()
    prompt, spk = synth.synthetic_prompt(11, seed=130), synth.synthetic_speaker(seed=131)
    noise = torch.empty(1, 16, D.vocab_size).exponential_(1, generator=torch.Generator().manual_seed(132))
    kw = dict(max_new_tokens=16, end_of_audio_token=2048, noise=noise, guidance_scale=(3.0, 2.0), end_of_text_token=2561,
              temperature=1.0, top_p=None)
    m = _mk(sds[0], utts=2, tc="", voices=sds[1:])
    got = U.generate_batch(m, [prompt], spk, voices=[2], **kw)[0]
    m.close()
    ms = _mk(sds[2], utts=2, tc="")
    want = U.generate_batch(ms, [prompt], spk, **kw)[0]
    ms.close()
    assert got.tolist() == want.tolist()


def test_tts_synthesise_batch_with_voices_writes_one_wav_per_text(tmp_path):
    from mvb200.fast_inference import TTS
    snap = tmp_path / "snapshot"
    snap.mkdir()
    torch.save(synth.stage1_checkpoint(D, 0), str(snap / "first_stage.pt"))
    ck = synth.stage1_checkpoint(D, 0)
    ck["model"] = finetune(D, 0, 1, seed=41)
    torch.save(ck, str(tmp_path / "voice_a.pt"))
    torch.save(synth.stage2_checkpoint(synth.S2_TINY, 1), str(snap / "second_stage.pt"))
    _, enc_sd = synth.encodec_model_and_state_dict(0)
    spk = snap / "spk.pt"
    torch.save(synth.synthetic_speaker(), str(spk))
    tts = TTS(str(snap), output_dir=str(tmp_path / "out"), encodec_state_dict=enc_sd, device="cuda:0", max_utts=2,
              voices={"a": str(tmp_path / "voice_a.pt")})
    tts.model._cfg.max_new = 256
    texts = ["Hello, what's up?", "The quick brown fox.", "A third sentence."]
    with pytest.raises(KeyError):
        tts.synthesise_batch(texts, [str(spk)] * 3, voices=["a", "nobody", None])
    paths = tts.synthesise_batch(texts, [str(spk)] * 3, voices=["a", None, "a"], seed=5)
    assert len(paths) == 3
    for p in paths:
        if p is None:
            continue
        assert os.path.isfile(p) and p.endswith(".wav")
        with wave.open(p) as w:
            assert w.getframerate() == 24000 and w.getnframes() >= 9600
    assert sum(p is not None for p in paths) >= 1
