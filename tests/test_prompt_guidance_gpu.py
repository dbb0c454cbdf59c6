"""GPU: prompt guidance, guidance_scale = (s, p) (fam/llm/mixins/causal.py:89-105, 224-262), through the C ABI.

A guided utterance owns its slot and a companion slot whose speaker-on row is the uncond-prompt row; k_sample mixes the
three rows.  Checked here:
  1. mvb_s1_sample_guided against the probabilities the reference's own _sample_next_token hands to torch.multinomial
     (tests/golden/prompt_guidance.npz) and, with top-k / top-p, against the float64 oracle;
  2. (s, 1.0) is s token for token, on a one-slot engine (no companion exists);
  3. end to end against the float64 three-row oracle (oracle/prompt_guidance_port.py) with supplied noise, on the
     persistent kernel with the unfused sampler, path A and path B, with a text token forced mid-stream;
  4. one guided request decodes identically alone, batched with unguided requests and through ContinuousBatcher in
     other slots, and its neighbours equal their solo runs (bf16, int4, int8);
  5. the lifecycle of a link (end-of-audio latch, release, re-use of the companion slot) and argument errors;
  6. TTS.synthesise_batch with (s, p) and with (s, 1.0).
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from mvb200 import synth

pytestmark = pytest.mark.gpu

EOA, EOT = 2048, 2561
V = synth.TINY.vocab_size


def _mk(sd, utts, kv="fp32", tc=None, unfused=None, mode=None):
    from mvb200.fast_model import ModelArgs, Transformer
    d = synth.TINY
    cfg = ModelArgs(block_size=d.block_size, vocab_size=d.vocab_size, n_layer=d.n_layer, n_head=d.n_head, dim=d.dim)
    m = Transformer.from_state_dict(sd, cfg, device="cuda:0", quantisation_mode=mode)
    m.setup_caches(2 * utts, d.block_size, kv_dtype=kv, tensor_core_path=tc, unfused_sampler=unfused)
    return m


@pytest.fixture(scope="module")
def tiny_sd():
    return synth.stage1_state_dict(synth.TINY, 0)


def _oracles(sd):
    from oracle import stage1_port as P
    d = synth.TINY
    out = []
    for _ in range(2):
        o = P.Stage1Oracle(sd, d.n_head, d.norm_eps, torch.float64, faithful_full_cache=False)
        o.setup_caches()
        out.append(o)
    return out


# ---- 1. the sampler ----------------------------------------------------------------------------------------------------
def test_sample_guided_vs_reference_probabilities(golden_dir, tiny_sd):
    from mvb200 import fast_inference_utils as U
    from oracle import prompt_guidance_port as G
    g = np.load(os.path.join(golden_dir, "prompt_guidance.npz"))
    m = _mk(tiny_sd, 1, "bf16")
    gen = torch.Generator().manual_seed(9)
    for c, (s, p, temp) in enumerate(g["params"]):
        logits = torch.from_numpy(g["logits"][c])[:, None].cuda()
        q = torch.empty(V).exponential_(1, generator=gen)
        tok, probs = U.sample(logits, (float(s), float(p)), float(temp), model=m, q=q)
        probs = probs.cpu().double()
        ref = torch.from_numpy(g["probs"][c]).double()
        np.testing.assert_allclose(probs.numpy(), ref.numpy(), rtol=2e-5, atol=1e-9, err_msg=f"case {c}")
        assert int(tok) == int(torch.argmax(probs / q.double())), f"case {c}"
    # top-k and the fast path's top-p after the mix, against the float64 oracle
    for c, (gs, temp, tp, tk) in enumerate([((3.0, 2.0), 1.0, 0.9, None), ((2.0, 1.5), 0.8, None, 40),
                                            ((1.0, 3.0), 1.2, 0.5, None), ((4.0, 2.5), 1.0, None, 1)]):
        lg = torch.randn(3, 1, V, generator=gen) * 2.5
        q = torch.empty(V).exponential_(1, generator=gen)
        tok, probs = U.sample(lg.cuda(), gs, temp, tp, tk, model=m, q=q)
        _, want, kept = G.sample3(lg.double(), gs, temp, tp, tk, return_kept=True)
        assert torch.equal(probs.cpu() > 0, kept), f"variant {c}: kept set"
        np.testing.assert_allclose(probs.cpu().double().numpy(), want.numpy(), rtol=1e-4, atol=1e-9, err_msg=f"variant {c}")
        assert int(tok) == int(torch.argmax(probs.cpu().double() / q.double())), f"variant {c}"


# ---- 2. p == 1 ---------------------------------------------------------------------------------------------------------
def test_p_equal_one_is_the_scalar_path_without_a_companion(tiny_sd):
    from mvb200 import fast_inference_utils as U
    m = _mk(tiny_sd, 1, "bf16", tc="")        # one slot: a companion could not exist
    prompt, spk = synth.synthetic_prompt(9, seed=3), synth.synthetic_speaker(seed=4)
    noise = torch.empty(1, 20, V).exponential_(1, generator=torch.Generator().manual_seed(5))
    kw = dict(max_new_tokens=20, end_of_audio_token=EOA, temperature=1.0, top_p=0.9, noise=noise)
    a = U.generate_batch(m, [prompt], spk, guidance_scale=3.0, **kw)[0]
    b = U.generate_batch(m, [prompt], spk, guidance_scale=(3.0, 1.0), end_of_text_token=EOT, **kw)[0]
    c = U.generate_batch(m, [prompt], spk, guidance_scale=(3.0, 1.0), **kw)[0]
    assert a.tolist() == b.tolist() == c.tolist()
    with pytest.raises(ValueError, match="2 slots"):
        U.generate_batch(m, [prompt], spk, guidance_scale=(3.0, 2.0), end_of_text_token=EOT, **kw)


# ---- 3. end to end vs the float64 oracle -------------------------------------------------------------------------------
def _first_divergence(got, want, label):
    """Index of the first differing token, or None when the sequences are equal."""
    for k in range(min(len(got), len(want))):
        if got[k] != want[k]:
            return k
    assert len(got) == len(want), (label, len(got), len(want))
    return None


@pytest.mark.parametrize("body", ["persistent_unfused", "path_a", "path_b"])
def test_end_to_end_vs_float64_oracle(tiny_sd, body):
    from mvb200 import fast_inference_utils as U
    from oracle import prompt_guidance_port as G
    tc, unfused = {"persistent_unfused": ("BC", True), "path_a": ("", None), "path_b": ("B", None)}[body]
    lens, n_new = [5, 17, 9], 24
    prompts = [synth.synthetic_prompt(T, seed=40 + i) for i, T in enumerate(lens)]
    spk = torch.cat([synth.synthetic_speaker(seed=50 + i) for i in range(3)])
    noise = torch.empty(3, n_new, V).exponential_(1, generator=torch.Generator().manual_seed(6))
    for i in range(3):                       # a text token drawn mid-stream: the companion must be fed end-of-text
        noise[i, 4 + i, 2300 + i] = 1e-30
    gs, kw = (3.0, 2.0), dict(temperature=1.0, top_p=None)     # the tail after the mix is test 1's
    m = _mk(tiny_sd, 6, "fp32", tc=tc, unfused=unfused)
    got = U.generate_batch(m, prompts, spk, max_new_tokens=n_new, end_of_audio_token=EOA, noise=noise, guidance_scale=gs,
                           end_of_text_token=EOT, **kw)
    flips = 0
    for i in range(3):
        o, oc = _oracles(tiny_sd)
        sink = []
        want = G.generate3(o, oc, prompts[i], spk[i:i + 1], guidance_scale=gs, end_of_text_token=EOT, max_new_tokens=n_new,
                           end_of_audio_token=EOA, noise=noise[i].double(), logit_sink=sink, **kw)[lens[i]:].tolist()
        assert want[4 + i] == 2300 + i and EOA not in want[:4 + i]
        k = _first_divergence(got[i].tolist(), want, body)
        if k is not None:
            # a first divergence must sit on an oracle near-tie of argmax(p / q) (the engine computes in fp32); what
            # follows it is a different sequence and is not compared
            _, pr = G.sample3(sink[k][0][:, None], gs, kw["temperature"], kw["top_p"])
            score = (pr / noise[i, k].double()).sort(descending=True).values
            gap = float(score[0] / score[1] - 1)
            print(f"{body} utterance {i}: diverges at step {k}, oracle best/second - 1 = {gap:.2e}")
            assert gap < 1e-4, f"{body} utterance {i} step {k}: not a near-tie ({gap})"
            flips += 1
    print(f"{body}: {3 - flips} of 3 guided utterances token for token with the float64 oracle")
    assert flips <= 1


# ---- 4. independence ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [None, "int4", "int8"], ids=["bf16", "int4", "int8"])
def test_guided_request_is_independent_of_its_batch(tiny_sd, mode):
    from mvb200 import fast_inference_utils as U
    from mvb200.serving import ContinuousBatcher, seeded_noise
    lens, news = [7, 12, 5], [30, 18, 25]
    prompts = [synth.synthetic_prompt(T, seed=60 + i) for i, T in enumerate(lens)]
    spks = [synth.synthetic_speaker(seed=70 + i) for i in range(3)]
    kw = dict(temperature=1.0, top_p=0.9, end_of_audio_token=EOA)
    m = _mk(tiny_sd, 4, "bf16", tc="", mode=mode)
    noise = [seeded_noise(m, lens[i], 80 + i, news[i]) for i in range(3)]
    gs = [3.0, (3.0, 2.0), 2.5]               # request 1 is guided
    alone = []
    for i in range(3):
        extra = dict(end_of_text_token=EOT) if i == 1 else {}
        alone.append(U.generate_batch(m, [prompts[i]], spks[i], max_new_tokens=news[i], noise=noise[i][None], guidance_scale=gs[i],
                                      **kw, **extra)[0].tolist())
    # batched with unguided utterances, two orders of submission (the guided request lands in different slots)
    for order in ([0, 1, 2], [2, 0, 1]):
        cb = ContinuousBatcher(m, burst=8)
        ids = {i: cb.submit(prompts[i], spks[i], max_new_tokens=news[i], noise=noise[i], guidance_scale=gs[i],
                            end_of_text_token=EOT, **kw) for i in order}
        cb._admit()
        print(f"{mode} order {order}: (request, slot, companion) "
              f"{[(r.rid, r.slot, r.companion) for r in cb._active.values()]}")
        out = cb.run_until_done()
        for i in range(3):
            assert out[ids[i]].tolist() == alone[i], f"{mode} order {order} request {i}"
    assert len(alone[1]) > 5


def test_finished_guided_request_frees_its_companion(tiny_sd):
    """Slot layout primary < active unguided slot < companion, with the guided request finishing first: once the
    batcher has seen it done, the next burst covers only the slots still active (the old companion is beyond them) and
    runs; every request equals its solo run."""
    from mvb200 import fast_inference_utils as U
    from mvb200.serving import ContinuousBatcher, seeded_noise
    lens, news = [6, 9, 7, 8], [60, 5, 60, 10]
    gs = [3.0, 3.0, 3.0, (3.0, 2.0)]                      # A, B, C unguided, G guided
    prompts = [synth.synthetic_prompt(T, seed=110 + i) for i, T in enumerate(lens)]
    spks = [synth.synthetic_speaker(seed=115 + i) for i in range(4)]
    kw = dict(temperature=1.0, top_p=0.9, end_of_audio_token=9999)     # lengths fixed by max_new
    m = _mk(tiny_sd, 4, "bf16", tc="")
    noise = [seeded_noise(m, lens[i], 120 + i, news[i]) for i in range(4)]
    alone = [U.generate_batch(m, [prompts[i]], spks[i], max_new_tokens=news[i], noise=noise[i][None], guidance_scale=gs[i],
                              end_of_text_token=EOT, **kw)[0].tolist() for i in range(4)]
    cb = ContinuousBatcher(m, burst=8)
    sub = lambda i: cb.submit(prompts[i], spks[i], max_new_tokens=news[i], noise=noise[i], guidance_scale=gs[i],  # noqa: E731
                              end_of_text_token=EOT, **kw)
    ids = [sub(i) for i in range(3)]
    assert cb.step() == [ids[1]]                          # A, B, C in slots 0, 1, 2; B finishes in the first burst
    ids.append(sub(3))
    cb._admit()
    g = cb._active[1]
    assert g.rid == ids[3] and g.companion == 3           # G in slot 1, its companion in slot 3
    finished = []
    while ids[3] not in finished:
        finished += cb.step()
    assert ids[0] not in finished and ids[2] not in finished
    assert sorted(cb._active) == [0, 2] and not cb._companions   # the next burst decodes slots 0..2 only
    out = cb.run_until_done()
    for i in range(4):
        assert out[ids[i]].tolist() == alone[i], f"request {i}"

    # the link of a finished guided request is gone: an unguided burst samples in the resident kernel again
    from mvb200 import _lib
    m2 = _mk(tiny_sd, 4, "bf16")                          # every engine path
    lib, h, st = m2._lib, m2.handle, m2._stream()
    for s in range(4):
        _lib.check(lib.mvb_s1_release(h, s, st))
    pr = prompts[3].numpy().astype(np.int32)
    sv = spks[3].numpy().astype(np.float32).reshape(-1)
    sp = _lib.Sampling(3.0, 1.0, 0.9, 0, 9999, 7)
    _lib.check(lib.mvb_s1_admit_guided(h, 0, 3, pr.ctypes.data_as(C.c_void_p), pr.size, sv.ctypes.data_as(C.c_void_p),
                                       C.byref(sp), 2.0, EOT, 3, None, st))
    _lib.check(lib.mvb_s1_decode(h, 4, 4, st))
    assert lib.mvb_s1_decode(h, 1, 8, st) == _lib.MVB_ERR_ARG     # done on the device, but not yet seen by the host
    assert _poll(m2, 4)[0] == [1, 1, 1, 1]
    before = lib.mvb_s1_launch_count(h)
    _lib.check(lib.mvb_s1_decode(h, 1, 8, st))
    launches = lib.mvb_s1_launch_count(h) - before
    print(f"8-step burst after the guided request finished: {launches} launches")
    assert launches < 8, "the burst fell back to the unfused sampler"


# ---- 5. lifecycle and errors -------------------------------------------------------------------------------------------
def _poll(m, n):
    from mvb200 import _lib
    done, n_gen = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
    _lib.check(m._lib.mvb_s1_poll(m.handle, n, done.ctypes.data_as(C.c_void_p), n_gen.ctypes.data_as(C.c_void_p), m._stream()))
    return done.tolist(), n_gen.tolist()


def _fetch(m, slot):
    from mvb200 import _lib
    buf = np.zeros(256, dtype=np.int32)
    n = C.c_int32(0)
    _lib.check(m._lib.mvb_s1_fetch(m.handle, slot, buf.ctypes.data_as(C.c_void_p), 256, C.byref(n), None, m._stream()))
    return buf[:n.value].tolist()


def test_link_lifecycle(tiny_sd):
    from mvb200 import _lib
    from mvb200 import fast_inference_utils as U
    m = _mk(tiny_sd, 3, "bf16", tc="")
    lib, h, st = m._lib, m.handle, m._stream()
    prompt = synth.synthetic_prompt(8, seed=90).numpy().astype(np.int32)
    spk = synth.synthetic_speaker(seed=91).numpy().astype(np.float32).reshape(-1)
    sp = _lib.Sampling(3.0, 1.0, -1.0, 0, EOA, 5)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    for s in range(3):
        _lib.check(lib.mvb_s1_release(h, s, st))
    # end-of-audio drawn at step 3 parks the companion with the primary
    noise = torch.empty(40, V).exponential_(1, generator=torch.Generator().manual_seed(92)).cuda()
    noise[3, EOA] = 1e-30
    _lib.check(lib.mvb_s1_admit_guided(h, 0, 2, vp(prompt), prompt.size, vp(spk), C.byref(sp), 2.0, EOT, 40, noise.data_ptr(), st))
    for _ in range(4):
        _lib.check(lib.mvb_s1_decode(h, 3, 1, st))
    done, n_gen = _poll(m, 3)
    assert done == [1, 1, 1] and n_gen[0] == n_gen[2] == 4 and _fetch(m, 0)[-1] == EOA
    # release parks both slots of a running guided utterance
    _lib.check(lib.mvb_s1_admit_guided(h, 1, 0, vp(prompt), prompt.size, vp(spk), C.byref(sp), 2.0, EOT, 40, None, st))
    _lib.check(lib.mvb_s1_decode(h, 2, 2, st))
    assert _poll(m, 2)[0] == [0, 0]
    _lib.check(lib.mvb_s1_release(h, 1, st))
    assert _poll(m, 2)[0] == [1, 1]
    # an unguided request admitted into the old companion slot decodes exactly as it does alone
    other = synth.synthetic_prompt(11, seed=93)
    on = torch.empty(1, 16, V).exponential_(1, generator=torch.Generator().manual_seed(94))
    solo = U.generate_batch(_mk(tiny_sd, 1, "bf16", tc=""), [other], synth.synthetic_speaker(seed=95), max_new_tokens=16,
                            noise=on, guidance_scale=3.0, temperature=1.0, end_of_audio_token=9999)[0].tolist()
    sp2 = _lib.Sampling(3.0, 1.0, -1.0, 0, 9999, 5)
    o_np, s_np, d_on = other.numpy().astype(np.int32), synth.synthetic_speaker(seed=95).numpy().astype(np.float32).reshape(-1), on[0].cuda()
    _lib.check(lib.mvb_s1_admit(h, 0, vp(o_np), o_np.size, vp(s_np), C.byref(sp2), 16, d_on.data_ptr(), st))
    for _ in range(20):
        _lib.check(lib.mvb_s1_decode(h, 2, 1, st))
    assert _poll(m, 2)[0][0] == 1 and _fetch(m, 0) == solo
    # argument errors launch nothing
    before = lib.mvb_s1_launch_count(h)
    bad_s = _lib.Sampling(0.5, 1.0, -1.0, 0, EOA, 5)
    for args in ((0, 1, sp, 0.5), (0, 1, bad_s, 2.0), (0, 1, sp, float("nan")), (1, 1, sp, 2.0), (0, 3, sp, 2.0), (0, -1, sp, 2.0)):
        u, c, spx, p = args
        assert lib.mvb_s1_admit_guided(h, u, c, vp(prompt), prompt.size, vp(spk), C.byref(spx), p, EOT, 40, None, st) == _lib.MVB_ERR_ARG, args
    assert lib.mvb_s1_admit_guided(h, 0, 1, vp(prompt), prompt.size, vp(spk), C.byref(sp), 2.0, V, 40, None, st) == _lib.MVB_ERR_ARG
    lg = torch.zeros(3, V, device="cuda")
    tok = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert lib.mvb_s1_sample_guided(h, lg.data_ptr(), C.byref(sp), 0.9, None, 0, tok.data_ptr(), None, st) == _lib.MVB_ERR_ARG
    assert lib.mvb_s1_launch_count(h) == before
    # a link whose companion is outside the decoded slots is refused
    _lib.check(lib.mvb_s1_admit_guided(h, 0, 2, vp(prompt), prompt.size, vp(spk), C.byref(sp), 2.0, EOT, 40, None, st))
    assert lib.mvb_s1_decode(h, 2, 1, st) == _lib.MVB_ERR_ARG
    _lib.check(lib.mvb_s1_decode(h, 3, 1, st))


# ---- 6. TTS ------------------------------------------------------------------------------------------------------------
def test_synthesise_batch_with_prompt_guidance(tmp_path):
    from mvb200.fast_inference import TTS
    d = tmp_path / "snapshot"
    d.mkdir()
    torch.save(synth.stage1_checkpoint(synth.TINY, 0), str(d / "first_stage.pt"))
    torch.save(synth.stage2_checkpoint(synth.S2_TINY, 1), str(d / "second_stage.pt"))
    _, enc_sd = synth.encodec_model_and_state_dict(0)
    spk = str(d / "spk.pt")
    torch.save(synth.synthetic_speaker(seed=11), spk)
    tts = TTS(str(d), output_dir=str(tmp_path / "out"), encodec_state_dict=enc_sd, device="cuda:0", max_utts=2)
    tts.model._cfg.max_new = 256
    texts = ["Hello, what's up?", "The quick brown fox."]
    guided = tts.synthesise_batch(texts, [spk, spk], guidance_scale=(3.0, 2.0), seed=1234)
    assert len(guided) == 2 and any(p is not None for p in guided)
    for p in guided:
        assert p is None or (os.path.isfile(p) and p.endswith(".wav"))
    a = tts.synthesise_batch(texts, [spk, spk], guidance_scale=3.0, seed=1234)
    b = tts.synthesise_batch(texts, [spk, spk], guidance_scale=(3.0, 1.0), seed=1234)
    assert [open(p, "rb").read() if p else None for p in a] == [open(p, "rb").read() if p else None for p in b]
    one = TTS(str(d), output_dir=str(tmp_path / "out1"), encodec_state_dict=enc_sd, device="cuda:0")
    with pytest.raises(ValueError, match="max_utts=2"):
        one.synthesise_batch(texts[:1], [spk], guidance_scale=(3.0, 2.0))
