"""ORACLE (test infrastructure): tests/golden/prompt_guidance.npz -- the probabilities the REFERENCE'S OWN
``CausalInferenceMixin._sample_next_token`` (fam/llm/mixins/causal.py:56-137) hands to ``torch.multinomial`` for
three-row prompt guidance, captured by calling that very method (unbound) on a stand-in ``self`` whose ``__call__``
returns seeded fp32 logits [3, 1, V] (V = 2562) and by recording the argument of ``torch.multinomial``.

Sweep: (s, p) in {(3, 1), (3, 1.5), (1, 2), (2.5, 3), (3.1, 1.7)} x temperature in {1.0, 0.7}, top_k = top_p = None (the GPT path's
top-p, causal.py:9-20, is not the fast path's; the engine keeps the fast path's tail after the mix).  With p == 1 the
reference reads two rows; the third row of the stored logits is then unused.
Build container only (fam.llm.mixins.causal imports on the CPU):  python oracle/make_golden_prompt_guidance.py
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness as R  # noqa: E402

V = 2562
# the last pair is not representable in fp32: the engine forms its coefficients from the fp32-rounded scales
SCALES = [(3.0, 1.0), (3.0, 1.5), (1.0, 2.0), (2.5, 3.0), (3.1, 1.7)]
TEMPERATURES = [1.0, 0.7]


def main() -> None:
    R._import_reference()
    from fam.llm.mixins.causal import CausalInferenceMixin

    g = torch.Generator().manual_seed(4242)
    logits, probs, params = [], [], []
    for s, p in SCALES:
        for temp in TEMPERATURES:
            # three rows that differ enough for each term of the mix to matter, on the scale of real stage-1 logits
            lg = torch.randn(3, 1, V, generator=g) * torch.tensor([3.0, 2.5, 2.0]).view(3, 1, 1)
            rows = lg if p > 1 else lg[:2]
            stand_in = type("StandIn", (), {"config": SimpleNamespace(block_size=2048),
                                            "__call__": lambda self, idx, speaker_embs=None, _r=rows: ([_r.clone()], None)})()
            seen = []
            real = torch.multinomial

            def capture(prob, num_samples=1, **kw):
                seen.append(prob.detach().clone())
                return real(prob, num_samples, **kw)

            torch.multinomial = capture
            try:
                idx = torch.zeros(rows.shape[0], 1, 4, dtype=torch.long)
                CausalInferenceMixin._sample_next_token(stand_in, idx=idx, speaker_embs=None, temperature=temp, top_k=None,
                                                        top_p=None, guidance_scale=(s, p))
            finally:
                torch.multinomial = real
            assert len(seen) == 1 and seen[0].shape == (1, V), [t.shape for t in seen]
            logits.append(lg[:, 0].numpy())
            probs.append(seen[0][0].numpy())
            params.append((s, p, temp))
    out = os.path.join(ROOT, "tests", "golden", "prompt_guidance.npz")
    np.savez_compressed(out, logits=np.stack(logits).astype(np.float32), probs=np.stack(probs).astype(np.float32),
                        params=np.asarray(params, dtype=np.float64))
    print(f"wrote {out}: {len(params)} cases")


if __name__ == "__main__":
    main()
