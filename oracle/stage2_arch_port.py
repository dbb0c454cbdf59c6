"""ORACLE (test infrastructure, never the product path): CPU restatement of the reference's stage-2 ``GPT.forward``
(causal=False, fam/llm/model.py:195-314) in every architecture ``GPTConfig`` builds (model.py:26-46):

  * ``norm_type``          "rmsnorm" (``RMSNorm``, layers.py:20-30) or "layernorm" (``LayerNorm``, layers.py:8-17: eps 1e-5,
                           a bias when ``bias``)
  * ``nonlinearity_type``  "swiglu" (``SwiGLU``, layers.py:33-42) or "gelu" (``c_fc`` -> exact ``nn.GELU()`` -> ``c_proj``,
                           layers.py:45-48)
  * ``bias``               biases on ``c_attn``, ``attn.c_proj``, ``c_fc`` / ``swiglu.w1`` / ``swiglu.w3``, ``mlp.c_proj``
                           (attn.py:61-64, layers.py:37-53); ``speaker_cond_pos`` and ``lm_heads`` never have one
                           (model.py:128, 136)

The input builder and the sampler are oracle/stage2_port.py's; with the production architecture (rmsnorm, swiglu, no bias)
this class computes what ``stage2_port.Stage2Oracle`` computes.  Pinned by tests/test_stage2_arch_cpu.py against
tests/golden/stage2_arch.npz (oracle/make_golden_stage2_arch.py, the reference's own ``GPT``) and against the live
reference when /root/reference is mounted.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from oracle.stage2_port import PAD, build_input, non_causal_sample  # noqa: F401  (re-exported for callers)


class Stage2ArchOracle:
    def __init__(self, sd: Dict[str, torch.Tensor], n_head: int, eps: float, dtype=torch.float32, device="cpu", *,
                 norm_type: str = "rmsnorm", nonlinearity_type: str = "swiglu", bias: bool = False):
        """``eps`` is RMSNorm's; LayerNorm uses 1e-5 (layers.py:17).  With ``bias`` the Linear (and LayerNorm) biases are
        read from ``sd``."""
        assert norm_type in ("rmsnorm", "layernorm") and nonlinearity_type in ("swiglu", "gelu")
        cv = lambda t: t.to(device=device, dtype=dtype).contiguous()   # noqa: E731
        opt = lambda k: cv(sd[k]) if bias else None                     # noqa: E731
        self.n_head, self.eps = n_head, eps
        self.layernorm, self.gelu = norm_type == "layernorm", nonlinearity_type == "gelu"
        self.wtes = []
        while f"transformer.wtes.{len(self.wtes)}.weight" in sd:
            self.wtes.append(cv(sd[f"transformer.wtes.{len(self.wtes)}.weight"]))
        self.wpe = cv(sd["transformer.wpe.weight"])
        self.w_spk = cv(sd["speaker_cond_pos.weight"])
        self.ln_f = cv(sd["transformer.ln_f.weight"])
        self.ln_f_b = opt("transformer.ln_f.bias") if self.layernorm else None
        self.heads = []
        while f"lm_heads.{len(self.heads)}.weight" in sd:
            self.heads.append(cv(sd[f"lm_heads.{len(self.heads)}.weight"]))
        self.layers = []
        while f"transformer.h.{len(self.layers)}.ln_1.weight" in sd:
            p = f"transformer.h.{len(self.layers)}."
            ffn = dict(w1="mlp.c_fc") if self.gelu else dict(w1="mlp.swiglu.w1", w3="mlp.swiglu.w3")
            names = dict(qkv="attn.c_attn", o="attn.c_proj", **ffn, w2="mlp.c_proj")
            L = {k: cv(sd[p + n + ".weight"]) for k, n in names.items()}
            L.update({k + "_b": opt(p + n + ".bias") for k, n in names.items()})
            L.update(g1=cv(sd[p + "ln_1.weight"]), g2=cv(sd[p + "ln_2.weight"]))
            L.update(b1=opt(p + "ln_1.bias") if self.layernorm else None, b2=opt(p + "ln_2.bias") if self.layernorm else None)
            self.layers.append(L)
        self.block_size = self.wpe.shape[0]

    def _norm(self, x, g, b=None):
        if self.layernorm:      # layers.py:8-17: F.layer_norm with eps 1e-5
            return F.layer_norm(x, g.shape, g, b, 1e-5)
        return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + self.eps) * g   # layers.py:20-30 (no fp32 upcast)

    @staticmethod
    def _lin(x, w, b):
        return x @ w.t() if b is None else x @ w.t() + b

    def _mlp(self, n, L):       # layers.py:36-72
        if self.gelu:
            h = F.gelu(self._lin(n, L["w1"], L["w1_b"]))                 # nn.GELU(): approximate='none'
        else:
            h = F.silu(self._lin(n, L["w1"], L["w1_b"])) * self._lin(n, L["w3"], L["w3_b"])
        return self._lin(h, L["w2"], L["w2_b"])

    @torch.no_grad()
    def forward(self, idx: torch.Tensor, spk: Optional[torch.Tensor]) -> List[torch.Tensor]:
        """idx int64 [b, 2, t]; spk [b, 1, spk_dim] -> list of 6 logits [b, t, V_target] (model.py:232-311)."""
        b, nh_in, t = idx.shape
        idx = idx.to(self.wpe.device)
        x = sum(w[idx[:, i]] for i, w in enumerate(self.wtes)) + self.wpe[:t]
        if spk is not None:
            x = x + spk.to(x) @ self.w_spk.t()                         # spk_emb_on_text=True: all positions
        E = x.shape[-1]
        hs = E // self.n_head
        for L in self.layers:
            n = self._norm(x, L["g1"], L["b1"])
            q, k, v = self._lin(n, L["qkv"], L["qkv_b"]).view(b, t, 3, self.n_head, hs).unbind(2)   # attn.py:175,136-140
            q, k, v = (z.transpose(1, 2) for z in (q, k, v))
            att = torch.softmax((q @ k.transpose(-1, -2)) / math.sqrt(hs), dim=-1) @ v   # non-causal, no padding mask
            x = x + self._lin(att.transpose(1, 2).reshape(b, t, E), L["o"], L["o_b"])
            x = x + self._mlp(self._norm(x, L["g2"], L["b2"]), L)
        x = self._norm(x, self.ln_f, self.ln_f_b)
        return [x @ h.t() for h in self.heads]
