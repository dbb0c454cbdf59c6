"""ORACLE (test infrastructure, never the product path): CPU restatement of the reference's causal ``GPT`` with a KV
cache -- the slow path ``fam.llm.inference`` builds from ``GPTConfig(**model_args)`` (inference.py:102-156) -- for the
{cond, uncond} row pair of one utterance, in every architecture ``GPTConfig`` builds (model.py:26-46):

  * ``norm_type``          "rmsnorm" (``RMSNorm``, layers/layers.py:20-30) or "layernorm" (``LayerNorm``,
                           layers/layers.py:8-17: F.layer_norm with eps 1e-5 and a bias when ``bias``)
  * ``nonlinearity_type``  "swiglu" (``SwiGLU``, layers/layers.py:33-42, 53-60) or "gelu" (``c_fc`` -> exact
                           ``nn.GELU()`` -> ``c_proj``, layers/layers.py:45-48, 63-72)
  * ``bias``               biases on ``attn.c_attn`` (layers/attn.py:61), ``attn.c_proj`` (attn.py:64) and every MLP
                           Linear (layers.py:37-38, 47-49, 59-60); ``speaker_cond_pos`` (model.py:128) and the head,
                           tied to ``wtes.0`` (model.py:130-143), never have one

The row pair is the reference's CFG batch: row 0 with the speaker, row 1 built with the speaker left out
(``speaker_embs=[spk, None]``, model.py:249-262 gives that row a zero speaker embedding).  With the production
architecture (rmsnorm, swiglu, no bias) it computes bit for bit what ``oracle/stage1_port.Stage1Oracle`` computes with
``faithful_full_cache=False``.  Pinned by tests/test_stage1_arch_cpu.py against tests/golden/stage1_arch.npz
(oracle/make_golden_stage1_arch.py, the reference's own ``GPT``) and against the live reference when it is mounted.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F


class Stage1ArchOracle:
    def __init__(self, sd: Dict[str, torch.Tensor], n_head: int, eps: float = 1e-5, dtype=torch.float32, *,
                 norm_type: str = "rmsnorm", nonlinearity_type: str = "swiglu", bias: bool = False):
        """``eps`` is RMSNorm's (``rmsnorm_eps``); LayerNorm uses 1e-5 (layers.py:17).  With ``bias`` the Linear (and
        LayerNorm) biases are read from ``sd``."""
        assert norm_type in ("rmsnorm", "layernorm") and nonlinearity_type in ("swiglu", "gelu")
        sd = {(k[len("_orig_mod."):] if k.startswith("_orig_mod.") else k): v for k, v in sd.items()}
        cv = lambda t: t.to(dtype).contiguous()          # noqa: E731
        opt = lambda k: cv(sd[k]) if bias else None      # noqa: E731
        self.dtype, self.n_head, self.eps = dtype, n_head, eps
        self.layernorm, self.gelu = norm_type == "layernorm", nonlinearity_type == "gelu"
        self.wte = cv(sd["transformer.wtes.0.weight"])
        self.wpe = cv(sd["transformer.wpe.weight"])
        self.w_spk = cv(sd["speaker_cond_pos.weight"])
        self.ln_f = cv(sd["transformer.ln_f.weight"])
        self.ln_f_b = opt("transformer.ln_f.bias") if self.layernorm else None
        self.head = cv(sd["lm_heads.0.weight"])           # == wtes.0 in a reference checkpoint (model.py:137-143)
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
        self.n_layer = len(self.layers)
        self.dim = self.wte.shape[1]
        self.head_dim = self.dim // n_head
        self.block_size = self.wpe.shape[0]
        self.k_cache, self.v_cache = [], []

    # layers/attn.py:20-44 (empty_kv_cache): one [rows, heads, block_size, head_dim] cache per layer
    def setup_caches(self) -> None:
        shape = (2, self.n_head, self.block_size, self.head_dim)
        self.k_cache = [torch.zeros(shape, dtype=self.dtype) for _ in range(self.n_layer)]
        self.v_cache = [torch.zeros(shape, dtype=self.dtype) for _ in range(self.n_layer)]
        self.causal = torch.tril(torch.ones(self.block_size, self.block_size, dtype=torch.bool))

    def _norm(self, x, g, b=None):
        if self.layernorm:      # layers.py:8-17
            return F.layer_norm(x, g.shape, g, b, 1e-5)
        return (x * torch.rsqrt(torch.mean(x * x, dim=-1, keepdim=True) + self.eps)) * g   # layers.py:20-30

    @staticmethod
    def _lin(x, w, b):          # nn.Linear(bias=config.bias)
        return x @ w.t() if b is None else x @ w.t() + b

    def _mlp(self, n, L):       # layers.py:63-72
        if self.gelu:
            h = F.gelu(self._lin(n, L["w1"], L["w1_b"]))                    # nn.GELU(): approximate='none'
        else:
            h = F.silu(self._lin(n, L["w1"], L["w1_b"])) * self._lin(n, L["w3"], L["w3_b"])   # layers.py:41-42
        return self._lin(h, L["w2"], L["w2_b"])

    def _attend(self, li: int, q, k, v, input_pos):
        # attn.py:84-115 (_update_kv_cache: k / v cached after c_attn and its bias), then attn.py:117-158: SDPA, causal
        # over the prefill, the whole cache for a decode step -- i.e. every position <= its own
        self.k_cache[li][:, :, input_pos] = k
        self.v_cache[li][:, :, input_pos] = v
        hi = int(input_pos.max()) + 1
        K, V = self.k_cache[li][:, :, :hi], self.v_cache[li][:, :, :hi]
        s = (q @ K.transpose(-1, -2)) * (1.0 / math.sqrt(self.head_dim))
        s = s.masked_fill(~self.causal[None, None, input_pos][..., :hi], float("-inf"))
        return torch.softmax(s, dim=-1) @ V

    @torch.no_grad()
    def forward(self, idx: torch.Tensor, spk_emb: torch.Tensor, input_pos: torch.Tensor) -> torch.Tensor:
        """idx int [2, S] (row 0 conditioned, row 1 without the speaker); spk_emb [1, spk_dim]; input_pos [S]
        consecutive.  Returns logits [2, S, vocab] at every position (model.py:232-314; the reference's inference keeps
        only the last, model.py:303-310) and appends to the cache at ``input_pos``."""
        B, S = idx.shape
        assert B == 2
        input_pos = input_pos.long()
        spk_mask = torch.zeros((2, 1, self.dim), dtype=torch.bool)
        spk_mask[0] = True
        x = self.wte[idx.long()] + self.wpe[input_pos] + (spk_emb.to(self.dtype) @ self.w_spk.t()) * spk_mask   # :246-291
        H, hd = self.n_head, self.head_dim
        for li, L in enumerate(self.layers):       # layers/combined.py:38-50
            n = self._norm(x, L["g1"], L["b1"])
            q, k, v = self._lin(n, L["qkv"], L["qkv_b"]).split([self.dim, self.dim, self.dim], dim=-1)   # attn.py:175
            q, k, v = (t.view(B, S, H, hd).transpose(1, 2) for t in (q, k, v))
            y = self._attend(li, q, k, v, input_pos).transpose(1, 2).contiguous().view(B, S, self.dim)
            x = x + self._lin(y, L["o"], L["o_b"])                                                  # attn.py:182-184
            x = x + self._mlp(self._norm(x, L["g2"], L["b2"]), L)
        return self._norm(x, self.ln_f, self.ln_f_b) @ self.head.t()                                 # model.py:293, 303-310


def teacher_forced(oracle: Stage1ArchOracle, prompt: torch.Tensor, spk: torch.Tensor, forced: torch.Tensor,
                   steps: Optional[list] = None):
    """Prefill ``prompt`` [T], then feed ``forced`` [n] one token per position.  Returns the last-position logits
    [1 + n, 2, vocab] of the prefill and of every step (or only of the prefill and ``steps``, 1-based)."""
    oracle.setup_caches()
    T = prompt.numel()
    out = [oracle.forward(prompt.view(1, -1).repeat(2, 1), spk, torch.arange(T))[:, -1]]
    want = set(range(1, forced.numel() + 1) if steps is None else steps)
    for i in range(forced.numel()):
        t = forced[i].view(1, 1).repeat(2, 1)
        lg = oracle.forward(t, spk, torch.tensor([T + i]))[:, -1]
        if i + 1 in want:
            out.append(lg)
    return torch.stack(out)
