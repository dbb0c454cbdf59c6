"""ORACLE (test infrastructure): tests/golden/stage1_arch.npz from the REFERENCE'S OWN causal ``fam.llm.model.GPT`` with
its KV cache (``enable_kv_cache``, mixins/causal.py:426-461; attn.py:84-115), run on CPU in fp32 -- the model the slow
path ``fam.llm.inference`` builds from ``GPTConfig(**model_args)`` (inference.py:102-156) -- for the stage-1 architectures
other than the production one (rmsnorm, swiglu, no bias): the seven other combinations of {rmsnorm, layernorm} x
{swiglu, gelu} x {bias, no bias} at synth.TINY, and GPTConfig's default (layernorm, gelu, bias) at production width
(dim 2048, 16 heads, 2 layers).

Each model runs the reference's CFG batch [cond, uncond] (``speaker_embs=[spk, None]``: the uncond row has no speaker,
model.py:249-262): a prefill of a synthetic prompt, then N_STEPS teacher-forced decode steps.  Kept per model: the cond
and uncond logits of the last position at the prefill and at steps STEPS, and the token the reference's own
``fast_inference_utils.sample`` (utils:107-120; guidance 3, temperature 1, top_p 0.95) draws at the prefill and at every
step, with its Exp(1) draw ``q`` (utils:61-65) taken from the seeded CPU generator ``NOISE_SEED`` ([1 + N_STEPS, vocab]
in order; the tests regenerate it and check its checksum).  Build container only."""
import dataclasses
import itertools
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "metavoice-src_b200"))
from mvb200 import synth  # noqa: E402
from oracle import ref_harness as R  # noqa: E402

T_PROMPT, N_STEPS, STEPS = 24, 255, (1, 8, 64, 255)
NOISE_SEED, FORCED_SEED, WEIGHT_SEED, SPK_SEED = 77, 78, 5, 11
SAMPLING = dict(guidance_scale=3.0, temperature=1.0, top_p=0.95)


def variants():
    """(tag, dims) of every golden entry."""
    out = []
    for norm, mlp, bias in itertools.product(("rmsnorm", "layernorm"), ("swiglu", "gelu"), (False, True)):
        if (norm, mlp, bias) != ("rmsnorm", "swiglu", False):
            d = dataclasses.replace(synth.TINY, norm_type=norm, nonlinearity_type=mlp, bias=bias, intermediate_size=None)
            d.__post_init__()
            out.append((f"tiny_{norm}_{mlp}_{'bias' if bias else 'nobias'}", d))
    full = dataclasses.replace(synth.FULL, n_layer=2, norm_type="layernorm", nonlinearity_type="gelu", bias=True,
                               intermediate_size=None)
    full.__post_init__()
    out.append(("full_gptconfig_default", full))
    return out


def noise(vocab: int) -> torch.Tensor:
    return torch.empty(1 + N_STEPS, vocab).exponential_(1, generator=torch.Generator().manual_seed(NOISE_SEED))


def forced_tokens() -> torch.Tensor:
    return torch.randint(0, 2048, (N_STEPS,), generator=torch.Generator().manual_seed(FORCED_SEED), dtype=torch.int64)


def reference_gpt(d, sd):
    R._import_reference()
    from fam.llm.model import GPT, GPTConfig
    m = GPT(GPTConfig(**synth.stage1_model_args(d)), speaker_emb_dim=d.speaker_emb_dim).eval()
    m.load_state_dict({k: v.float() for k, v in sd.items()})      # strict: every tensor of the architecture, no other
    return m


def run_reference(d, sd):
    """(logits [1 + len(STEPS), 2, V] float32, sampled ids [1 + N_STEPS] int)."""
    m = reference_gpt(d, sd)
    assert (m.config.norm_type, m.config.nonlinearity_type, m.config.bias) == (d.norm_type, d.nonlinearity_type, d.bias)
    fiu = R.reference_functions()
    q = noise(d.vocab_size)
    draw = {"i": 0}

    def sample_one(probs):             # utils:61-65 with the recorded Exp(1) draw of this position
        qi = q[draw["i"]].to(probs.dtype)
        draw["i"] += 1
        return torch.argmax(probs / qi, dim=-1, keepdim=True).to(dtype=torch.int)

    orig = fiu.multinomial_sample_one_no_sync
    fiu.multinomial_sample_one_no_sync = sample_one
    try:
        prompt = synth.synthetic_prompt(T_PROMPT).long()
        spk = synth.synthetic_speaker(seed=SPK_SEED)                  # [1, 256]
        forced = forced_tokens()
        sk = {k: torch.tensor(v) for k, v in SAMPLING.items()}
        m.enable_kv_cache()
        m.empty_kv_cache(batch_size=2, kv_cache_maxlen=d.block_size, dtype=torch.float32)
        kept, ids = [], []
        with torch.no_grad():
            idx = prompt.view(1, 1, -1).repeat(2, 1, 1)               # [b = {cond, uncond}, hierarchies, t]
            for step in range(N_STEPS + 1):
                lg, _ = m(idx, speaker_embs=[spk, None])
                lg = lg[0]                                            # [2, 1, V]: the last position (model.py:303-307)
                if step == 0 or step in STEPS:
                    kept.append(lg[:, -1].clone())
                tok, _ = fiu.sample(lg, **sk)
                ids.append(int(tok))
                if step < N_STEPS:
                    idx = forced[step].view(1, 1, 1).repeat(2, 1, 1)
        assert draw["i"] == N_STEPS + 1
    finally:
        fiu.multinomial_sample_one_no_sync = orig
    return torch.stack(kept), np.asarray(ids, np.int16)


def main():
    out = {"steps": np.asarray(STEPS, np.int32), "t_prompt": np.int32(T_PROMPT), "n_steps": np.int32(N_STEPS),
           "noise_seed": np.int64(NOISE_SEED), "forced_seed": np.int64(FORCED_SEED), "weight_seed": np.int64(WEIGHT_SEED),
           "spk_seed": np.int64(SPK_SEED), "prompt": synth.synthetic_prompt(T_PROMPT).numpy(),
           "forced": forced_tokens().numpy().astype(np.int16)}
    out["noise_checksum"] = np.float64(noise(synth.TINY.vocab_size).double().sum())
    for tag, d in variants():
        sd = synth.stage1_state_dict(d, WEIGHT_SEED, tie_head=True)
        logits, ids = run_reference(d, sd)
        out[f"{tag}_logits"] = logits.numpy().astype(np.float32)      # [1 + len(STEPS), 2, V]
        out[f"{tag}_ids"] = ids                                       # [1 + N_STEPS]
        out[f"{tag}_checksum"] = np.float64(synth.state_dict_checksum(sd))
        print(tag, "ok", logits.shape, ids[:8])
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "stage1_arch.npz"), **out)


if __name__ == "__main__":
    main()
