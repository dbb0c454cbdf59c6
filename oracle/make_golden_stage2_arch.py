"""ORACLE (test infrastructure): tests/golden/stage2_arch.npz from the REFERENCE'S OWN ``fam.llm.model.GPT`` (causal=False)
run on CPU in fp32, for the stage-2 architectures other than the synthetic production one (rmsnorm, swiglu, no bias):
every other combination of {rmsnorm, layernorm} x {swiglu, gelu} x {bias, no bias} at S2_TINY, and GPTConfig's own
default (layernorm, gelu, bias: model_args without the three keys) and (rmsnorm, swiglu, bias) at S2_FULL.  Each entry
holds the logits of the first and last hierarchy at three kept positions (the last text token, mid-audio, the last
padding position), all tokens sampled under manual_seed(4242) (int16) and the state-dict checksum, as
oracle/make_golden_stage2.py does for the production architecture; the subset keeps the file small, the tokens pin every
hierarchy and position.  Build container only."""
import dataclasses
import itertools
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "metavoice-src_b200"))
from mvb200 import synth  # noqa: E402
from oracle import ref_harness as R, stage2_port as P  # noqa: E402

ARCH_KEYS = ("norm_type", "nonlinearity_type", "bias")
HEADS = (0, 5)                  # hierarchies whose logits are kept


def variants():
    """(tag, dims, frames, drop_arch_keys) for every golden entry."""
    out = []
    for norm, mlp, bias in itertools.product(("rmsnorm", "layernorm"), ("swiglu", "gelu"), (False, True)):
        if (norm, mlp, bias) != ("rmsnorm", "swiglu", False):
            d = dataclasses.replace(synth.S2_TINY, norm_type=norm, nonlinearity_type=mlp, bias=bias)
            out.append((f"tiny_{norm}_{mlp}_{'bias' if bias else 'nobias'}", d, 60, False))
    out.append(("full_gptconfig_default", dataclasses.replace(synth.S2_FULL, norm_type="layernorm", nonlinearity_type="gelu",
                                                              bias=True), 375, True))
    out.append(("full_rmsnorm_swiglu_bias", dataclasses.replace(synth.S2_FULL, bias=True), 375, False))
    return out


def model_args(d, drop_arch_keys):
    a = synth.stage2_model_args(d)
    if drop_arch_keys:              # GPTConfig(**model_args) fills them with its defaults
        for k in ARCH_KEYS:
            a.pop(k)
    return a


def reference_gpt(d, sd, drop_arch_keys):
    R._import_reference()
    from fam.llm.model import GPT, GPTConfig
    m = GPT(GPTConfig(**model_args(d, drop_arch_keys)), speaker_emb_dim=d.speaker_emb_dim).eval()
    m.load_state_dict({k: v.float() for k, v in sd.items()})      # strict: every tensor of the architecture, no other
    return m


def main():
    out = {}
    for tag, d, frames, drop in variants():
        sd = synth.stage2_state_dict(d, 1)
        m = reference_gpt(d, sd, drop)
        assert (m.config.norm_type, m.config.nonlinearity_type, m.config.bias) == (d.norm_type, d.nonlinearity_type, d.bias)
        text, cb0, cb1 = synth.synthetic_stage2_input(d, frames)
        idx = P.build_input(text, cb0, cb1, d.block_size)[None]
        spk = synth.synthetic_speaker(seed=21)[None]
        with torch.no_grad():
            logits, _ = m(idx, speaker_embs=spk)
        torch.manual_seed(4242)
        y = m.generate(idx, None, temperature=1.0, top_k=200, top_p=None, speaker_embs=spk, batch_size=1, guidance_scale=None)
        torch.manual_seed(4242)
        noise = [torch.empty(1, d.block_size, v).exponential_(1) for v in d.target_vocab_sizes]
        y2 = P.non_causal_sample([l.clone() for l in logits], 1.0, 200, noise)
        assert torch.equal(y, y2), "multinomial != exp-race with the same generator stream"
        keep = [len(text) - 1, len(text) + frames // 2, d.block_size - 1]
        out[f"{tag}_idx"] = idx.numpy().astype(np.int32)
        out[f"{tag}_spk"] = spk.numpy()
        out[f"{tag}_keep"] = np.asarray(keep, np.int32)
        out[f"{tag}_logits"] = torch.stack([logits[h][0, keep] for h in HEADS]).numpy()   # [len(HEADS), n_keep, V]
        out[f"{tag}_tokens"] = y[0].numpy().astype(np.int16)                              # [6, t]
        out[f"{tag}_checksum"] = np.float64(synth.state_dict_checksum(sd))
        print(tag, "ok", y.shape)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "stage2_arch.npz"), **out)


if __name__ == "__main__":
    main()
