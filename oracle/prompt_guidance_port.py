"""ORACLE (test infrastructure, never the product path): the reference's prompt guidance, three CFG rows per utterance.

``fam/llm/mixins/causal.py:89-105`` mixes the rows {cond, uncond speaker, uncond prompt} of ``_sample_next_token`` as
``(s + p - 1) cond + (1 - s) uncond_spk + (1 - p) uncond_prompt``, and ``:224-262`` builds the uncond-prompt row from the
same tokens with every token ``> end_of_audio`` replaced by end-of-text, under the speaker.  After the mix this module
keeps the fast path's tail (``oracle/stage1_port.py``: temperature, top-k, the fast path's top-p, softmax, exp-race),
which is what the engine does.  ``generate3`` restates the loop on two ``Stage1Oracle`` instances: one holds the
primary's {cond, uncond speaker} pair, the other (the companion) the uncond-prompt row, whose second row is ignored.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import stage1_port as P


def mix3(logits: torch.Tensor, s: float, p: float) -> torch.Tensor:
    """logits [3, ..., V] -> [..., V], in the logits' dtype with Python-float coefficients, in causal.py:100-104's order."""
    cond, uncond_spk, uncond_prompt = logits[0], logits[1], logits[2]
    return (s + p - 1) * cond + (1 - s) * uncond_spk + (1 - p) * uncond_prompt


def sample3(logits: torch.Tensor, guidance_scale: Tuple[float, float], temperature, top_p=None, top_k=None,
            q: Optional[torch.Tensor] = None, return_kept: bool = False):
    """logits [3, S, V] -> (idx int32 [1], probs [V]); q = optional Exp(1) noise [V]."""
    s, p = (float(v) for v in guidance_scale)
    mixed = mix3(logits[:, -1], s, p)
    t = torch.as_tensor(temperature, dtype=mixed.dtype)
    tp = None if top_p is None else torch.as_tensor(top_p, dtype=mixed.dtype)
    probs, kept = P.logits_to_probs(mixed, temperature=t, top_p=tp, top_k=top_k)
    idx = P.exp_race_argmax(probs, q)
    return (idx, probs, kept) if return_kept else (idx, probs)


def uncond_prompt_tokens(tokens: torch.Tensor, end_of_audio_token: int, end_of_text_token: int) -> torch.Tensor:
    """causal.py:259-262: every token > end_of_audio becomes end-of-text."""
    return torch.where(tokens > end_of_audio_token, torch.full_like(tokens, end_of_text_token), tokens)


@torch.no_grad()
def generate3(model: P.Stage1Oracle, companion: P.Stage1Oracle, prompt: torch.Tensor, spk_emb: torch.Tensor, *,
              guidance_scale: Tuple[float, float], end_of_text_token: int, max_new_tokens: Optional[int] = None,
              end_of_audio_token: int = 2048, noise: Optional[torch.Tensor] = None, temperature=1.0, top_p=None,
              top_k=None, logit_sink: Optional[list] = None) -> torch.Tensor:
    """``stage1_port.generate`` with three rows: returns prompt ++ generated tokens (EOA included).  ``model`` and
    ``companion`` are two oracles over the same weights with caches of their own; ``noise`` [n_steps, V] replaces the
    generator draws; ``logit_sink`` collects (mixed-row logits [3, V], sampled token) per step."""
    T = prompt.size(0)
    max_seq = model.block_size if max_new_tokens is None else min(T + max_new_tokens, model.block_size)
    max_new = max_seq - T
    if max_new <= 0:
        raise ValueError("Prompt is too long to generate more tokens")
    step = 0

    def one(tok: torch.Tensor, pos: torch.Tensor):
        nonlocal step
        cu = uncond_prompt_tokens(tok, end_of_audio_token, end_of_text_token)
        lg = model.forward(tok.view(1, -1).repeat(2, 1), spk_emb, pos)
        lp = companion.forward(cu.view(1, -1).repeat(2, 1), spk_emb, pos)
        rows = torch.stack([lg[0], lg[1], lp[0]])
        q = None if noise is None else noise[step].to(rows.dtype)
        idx, _ = sample3(rows, guidance_scale, temperature, top_p, top_k, q=q)
        if logit_sink is not None:
            logit_sink.append((rows[:, -1].clone(), int(idx)))
        step += 1
        return idx

    seq = [prompt.to(torch.int)]
    cur = one(prompt.to(torch.int), torch.arange(0, T))
    seq.append(cur.view(1))
    pos = T
    for _ in range(max_new - 1):
        if bool((cur == end_of_audio_token).any()):
            break
        cur = one(cur.view(1), torch.tensor([pos]))
        pos += 1
        seq.append(cur.view(1))
    return torch.cat(seq)
