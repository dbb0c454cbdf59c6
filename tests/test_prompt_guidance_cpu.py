"""CPU: prompt guidance (guidance_scale = (s, p), fam/llm/mixins/causal.py:89-105, 224-262) without a GPU.

  * The float64 three-row oracle (oracle/prompt_guidance_port.py) against the probabilities the reference's own
    ``_sample_next_token`` hands to ``torch.multinomial`` (tests/golden/prompt_guidance.npz, fp32).  The reference mixes
    in fp32: three products and two sums of terms up to ~60 in magnitude, then the division by the temperature, each
    rounded once, move a logit by a few 1e-6 and a probability by that much relatively.  Bound: 3e-5 relative.
  * Host-side argument checks that raise before any library call.
"""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import prompt_guidance_port as G


def test_oracle_mix_vs_reference_probabilities(golden_dir):
    g = np.load(os.path.join(golden_dir, "prompt_guidance.npz"))
    assert g["params"].shape == (10, 3)
    assert {tuple(r[:2]) for r in g["params"]} == {(3, 1), (3, 1.5), (1, 2), (2.5, 3), (3.1, 1.7)}
    worst = 0.0
    for c, (s, p, temp) in enumerate(g["params"]):
        logits = torch.from_numpy(g["logits"][c]).double()[:, None]
        _, probs = G.sample3(logits, (float(s), float(p)), float(temp))
        ref = torch.from_numpy(g["probs"][c]).double()
        err = ((probs - ref).abs() / (3e-5 * ref + 1e-12)).max().item()
        worst = max(worst, err)
        assert err <= 1.0, (c, s, p, temp, err)
        # the oracle is not blind to the third row: dropping it moves the probabilities far outside the bound (p > 1)
        if p > 1:
            _, two = G.sample3(torch.cat([logits[:2], torch.zeros_like(logits[:1])]), (float(s), float(p)), float(temp))
            assert ((two - ref).abs() / (3e-5 * ref + 1e-12)).max().item() > 100
    print(f"three-row oracle vs reference: worst |err| / bound = {worst:.3f}")


def test_fp32_rounded_scales_stay_within_the_bound(golden_dir):
    """The C ABI carries s and p as fp32.  For (3.1, 1.7), which fp32 cannot represent, the mix formed from the rounded
    scales (as the engine forms it) still meets the 3e-5 bound against the reference, which used the Python doubles."""
    g = np.load(os.path.join(golden_dir, "prompt_guidance.npz"))
    for c, (s, p, temp) in enumerate(g["params"]):
        if (s, p) != (3.1, 1.7):
            continue
        s32, p32 = float(np.float32(s)), float(np.float32(p))
        assert (s32, p32) != (s, p)
        _, probs = G.sample3(torch.from_numpy(g["logits"][c]).double()[:, None], (s32, p32), float(temp))
        ref = torch.from_numpy(g["probs"][c]).double()
        assert ((probs - ref).abs() / (3e-5 * ref + 1e-12)).max().item() <= 1.0, c


def test_p_equal_one_is_the_two_row_mix():
    """(s, 1.0) mixes exactly like the fast path's scalar s: the third row's coefficient is 0."""
    from oracle import stage1_port as P
    lg = torch.randn(3, 1, 64, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    q = torch.empty(64, dtype=torch.float64).exponential_(1, generator=torch.Generator().manual_seed(2))
    i3, p3 = G.sample3(lg, (2.5, 1.0), 0.8, q=q)
    i2, p2 = P.sample(lg[:2], torch.tensor(2.5, dtype=torch.float64), torch.tensor(0.8, dtype=torch.float64), q=q)
    assert int(i3) == int(i2) and torch.equal(p3, p2)


def test_uncond_prompt_tokens_map_text_to_eot():
    t = torch.tensor([5, 2048, 2049, 2560, 1023, 2561])
    assert G.uncond_prompt_tokens(t, 2048, 2561).tolist() == [5, 2048, 2561, 2561, 1023, 2561]


@pytest.mark.parametrize("gs,msg", [((0.5, 2.0), ">= 1"), ((3.0, 0.9), ">= 1"), ((float("nan"), 2.0), "finite"),
                                    ((3.0, float("inf")), "finite"), ((3.0, 2.0, 1.0), "pair")])
def test_split_guidance_rejects_bad_scales(gs, msg):
    from mvb200.fast_inference_utils import split_guidance
    with pytest.raises(ValueError, match=msg):
        split_guidance(gs, 2561)


def test_split_guidance_forms():
    from mvb200.fast_inference_utils import split_guidance
    assert split_guidance(3.0) == (3.0, None)
    assert split_guidance((3.0, 1.0)) == (3.0, None)            # no end-of-text token needed: no prompt guidance
    assert split_guidance([2.5, 3.0], 2561) == (2.5, 3.0)
    with pytest.raises(ValueError, match="end_of_text_token"):
        split_guidance((3.0, 2.0))
    assert split_guidance((3.0, 2.0), need_eot=False) == (3.0, 2.0)


class _NoLib:
    """A model stand-in whose every library call fails the test: the checks below must raise first."""
    def __getattr__(self, name):
        raise AssertionError(f"library reached: {name}")


def test_generate_batch_checks_slots_and_eot_before_the_library():
    from mvb200 import fast_inference_utils as U
    model = SimpleNamespace(max_utts=3, _lib=_NoLib(), handle=None, config=SimpleNamespace(block_size=2048, vocab_size=2562))
    prompts = [torch.tensor([2050, 2561]), torch.tensor([2051, 2561])]
    spk = torch.zeros(2, 256)
    with pytest.raises(ValueError, match="4 slots"):
        U.generate_batch(model, prompts, spk, guidance_scale=(3.0, 2.0), end_of_text_token=2561, seed=1)
    with pytest.raises(ValueError, match="end_of_text_token"):
        U.generate_batch(model, prompts[:1], spk[:1], guidance_scale=(3.0, 2.0), seed=1)
    with pytest.raises(ValueError, match="teacher forcing"):
        U.generate_batch(model, prompts[:1], spk[:1], guidance_scale=(3.0, 2.0), end_of_text_token=2561, seed=1,
                         forced=torch.zeros(1, 4, dtype=torch.int32))


def test_tts_names_max_utts_for_a_one_slot_engine():
    from mvb200.fast_inference import TTS
    tts = SimpleNamespace(tokenizer=SimpleNamespace(eot_token=2561), model=SimpleNamespace(max_utts=1))
    with pytest.raises(ValueError, match="max_utts=2"):
        TTS._check_guidance(tts, (3.0, 2.0))
    TTS._check_guidance(tts, (3.0, 1.0))
    TTS._check_guidance(tts, 3.0)
    TTS._check_guidance(SimpleNamespace(tokenizer=tts.tokenizer, model=SimpleNamespace(max_utts=2)), (3.0, 2.0))
