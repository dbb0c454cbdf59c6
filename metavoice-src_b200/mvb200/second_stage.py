"""Host-side mirror of the stage-2 half of ``fam/llm/inference.py::Model`` over libmvb200.

``SecondStage.non_causal_sample`` keeps the argument meaning of ``Model.non_causal_sample``
(inference.py:248-338): texts + 2 stage-1 codebooks (+ speaker embeddings) -> 8 codebooks per utterance.
The vocoder call the reference makes next (``decoder.decode`` -> MBD, decoders.py:66-102) is outside this class.
Token adapters (integer bucketing, SURVEY.md rows a12/a16) stay on the host exactly as in the reference.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._engine import Engine, pack_arena_bytes

PAD = 1024  # _encodec_codes_pad_token (inference.py:125)


def flattened_interleaved_decode(tokens: Sequence[int], end_of_audio_token: int = PAD):
    """``FlattenedInterleavedEncodec2Codebook.decode`` (adapters/flattened_encodec.py:8-32)."""
    text, cb = [], [[], []]
    for t in tokens:
        if t < end_of_audio_token:
            cb[0].append(t)
        elif t < 2 * end_of_audio_token:
            cb[1].append(t - end_of_audio_token)
        elif t > 2 * end_of_audio_token:
            text.append(t)
    if len(cb[0]) != len(cb[1]):
        n = min(len(cb[0]), len(cb[1]))
        print("WARNING: Number of tokens at each hierarchy must be of the same length!")
        cb = [cb[0][:n], cb[1][:n]]
    return text[:-1], cb


def tilted_decode(hier: Sequence[Sequence[int]], end_of_audio_token: int = PAD):
    """``TiltedEncodec.decode`` (adapters/tilted_encodec.py:8-39)."""
    assert len(hier) > 1
    text = [t for t in hier[0] if t > end_of_audio_token]
    out = [[t for t in hier[0] if t < end_of_audio_token]] + [[t for t in h if t < end_of_audio_token] for h in hier[1:]]
    if len(set(len(x) for x in out)) != 1:
        n = min(len(x) for x in out)
        out = [x[:n] for x in out]
    return text[:-1], out


def build_stage2_input(text_ids: Sequence[int], codes: Sequence[Sequence[int]], block_size: int, pad: int = PAD) -> torch.Tensor:
    """The two input hierarchies of ``Model.non_causal_sample`` (inference.py:283-306): hierarchy 0 = text ++ codebook 0
    ++ pad, hierarchy 1 = pad x len(text) ++ codebook 1 ++ pad, each padded with ``pad`` / cut to ``block_size``."""
    h0 = list(text_ids) + list(codes[0]) + [pad]
    h1 = [pad] * len(text_ids) + list(codes[1]) + [pad]
    rows = []
    for h in (h0, h1):
        assert len(h) == len(h0)
        rows.append(h + [pad] * (block_size - len(h)) if len(h) < block_size else h[:block_size])
    return torch.tensor(rows, dtype=torch.int32)


_GLOBAL = lambda n_in, n_out: ([f"transformer.wtes.{i}.weight" for i in range(n_in)] +
                               ["transformer.wpe.weight", "speaker_cond_pos.weight", "transformer.ln_f.weight"] +
                               [f"lm_heads.{i}.weight" for i in range(n_out)])
_NORMS = {"rmsnorm": _lib.MVB_S2_NORM_RMS, "layernorm": _lib.MVB_S2_NORM_LAYER}
_MLPS = {"swiglu": _lib.MVB_S2_MLP_SWIGLU, "gelu": _lib.MVB_S2_MLP_GELU}


def stage2_arch(model_args: dict) -> Tuple[str, str, bool]:
    """(norm_type, nonlinearity_type, bias) of a second-stage ``model_args``, a missing key meaning GPTConfig's default
    (model.py:36-43: bias=True, norm_type="layernorm", nonlinearity_type="gelu"), as ``GPTConfig(**model_args)`` reads
    it.  A value libmvb200 does not build raises NotImplementedError naming it."""
    norm = model_args.get("norm_type", "layernorm")
    mlp = model_args.get("nonlinearity_type", "gelu")
    bias = model_args.get("bias", True)
    if norm not in _NORMS:
        raise NotImplementedError(f"libmvb200 stage 2: norm_type {norm!r} is not supported (rmsnorm, layernorm)")
    if mlp not in _MLPS:
        raise NotImplementedError(f"libmvb200 stage 2: nonlinearity_type {mlp!r} is not supported (swiglu, gelu)")
    if bias not in (True, False):
        raise NotImplementedError(f"libmvb200 stage 2: bias {bias!r} is not supported (True, False)")
    return norm, mlp, bool(bias)


def stage2_keys(n_in: int, n_out: int, n_layer: int, norm: str, mlp: str, bias: bool) -> List[str]:
    """State-dict keys in the order of mvb_s2_create_ex's offset list (include/mvb200.h)."""
    ffn = ["mlp.c_fc"] if mlp == "gelu" else ["mlp.swiglu.w1", "mlp.swiglu.w3"]
    layer = ["ln_1", "attn.c_attn", "attn.c_proj", "ln_2"] + ffn + ["mlp.c_proj"]
    keys = _GLOBAL(n_in, n_out) + [f"transformer.h.{l}.{k}.weight" for l in range(n_layer) for k in layer]
    if bias:
        ln = norm == "layernorm"
        keys += ["transformer.ln_f.bias"] if ln else []
        with_bias = [k for k in layer if ln or not k.startswith("ln_")]
        keys += [f"transformer.h.{l}.{k}.bias" for l in range(n_layer) for k in with_bias]
    return keys


class SecondStage(Engine):
    def __init__(self, checkpoint: dict, device="cuda", max_batch: int = 1, tokenizer=None, cuda_graph: bool = True):
        """``checkpoint`` = the second_stage.pt dict (model / model_args / meta), as ``Model._init_model`` reads it.
        ``cuda_graph=False`` (test hook): launch the forward pass kernel by kernel instead of replaying a captured graph."""
        a = checkpoint["model_args"]
        if a.get("causal", True):
            raise ValueError("second-stage checkpoint must be non-causal")
        norm, mlp, bias = stage2_arch(a)
        if not a.get("spk_emb_on_text", True):
            # model.py:104-107: the reference itself refuses a non-causal model with spk_emb_on_text=False
            raise NotImplementedError("spk_emb_on_text=False is not supported for the non-causal second stage (model.py:104-107)")
        sd = {(k[len("_orig_mod."):] if k.startswith("_orig_mod.") else k): v for k, v in checkpoint["model"].items()}
        self.args = a
        self.n_in, self.n_out = len(a["vocab_sizes"]), len(a["target_vocab_sizes"])
        keys = stage2_keys(self.n_in, self.n_out, a["n_layer"], norm, mlp, bias)
        super().__init__(device, *pack_arena_bytes([sd[k].to(torch.bfloat16) for k in keys]))
        hidden = sd["transformer.h.0.mlp.c_fc.weight" if mlp == "gelu" else "transformer.h.0.mlp.swiglu.w1.weight"].shape[0]
        cfg = _lib.S2Config()
        cfg.n_layer, cfg.n_head, cfg.n_embd, cfg.hidden = a["n_layer"], a["n_head"], a["n_embd"], hidden
        cfg.block_size, cfg.n_in, cfg.n_out = a["block_size"], self.n_in, self.n_out
        for i, v in enumerate(a["vocab_sizes"]):
            cfg.vocab_in[i] = v
        for i, v in enumerate(a["target_vocab_sizes"]):
            cfg.vocab_out[i] = v
        cfg.spk_dim = sd["speaker_cond_pos.weight"].shape[1]
        cfg.norm_eps = a.get("rmsnorm_eps") or 1e-5     # RMSNorm only: LayerNorm's eps is 1e-5 in the library
        cfg.max_batch = max_batch
        cfg.options = 0 if cuda_graph else _lib.MVB_S2_EAGER
        self.cfg = cfg
        self.arch = _lib.S2Arch(_NORMS[norm], _MLPS[mlp], int(bias))
        create = lambda cfg_p, *rest: self._lib.mvb_s2_create_ex(cfg_p, C.byref(self.arch), *rest)   # noqa: E731
        self._create(create, self._lib.mvb_s2_destroy, cfg, self._lib.mvb_s2_workspace_bytes)
        self.tokenizer = tokenizer
        self.block_size = a["block_size"]

    # inference.py:283-301
    def build_input(self, text_ids: Sequence[int], codes: Sequence[Sequence[int]]) -> torch.Tensor:
        return build_stage2_input(text_ids, codes, self.block_size)

    @torch.no_grad()
    def forward_tokens(self, idx: torch.Tensor, speaker_embs: Optional[torch.Tensor], temperature: float = 1.0,
                       top_k: Optional[int] = 200, noise: Optional[torch.Tensor] = None, seed: int = 0,
                       return_logits: bool = False):
        """idx int [b, 2, t] -> tokens int32 [b, 6, t] (== GPT.generate for causal=False, model.py:384-408)."""
        b = idx.shape[0]
        assert idx.shape[1] == self.n_in and idx.shape[2] == self.block_size
        idx_d = idx.to(device=self.device, dtype=torch.int32).contiguous()
        spk_d = None if speaker_embs is None else speaker_embs.reshape(b, -1).to(self.device, torch.float32).contiguous()
        V = self.args["target_vocab_sizes"][0]
        out = torch.empty((b, self.n_out, self.block_size), dtype=torch.int32, device=self.device)
        lg = torch.empty((self.n_out, b * self.block_size, V), dtype=torch.float32, device=self.device) if return_logits else None
        nz = None if noise is None else noise.to(self.device, torch.float32).contiguous()
        _lib.check(self._lib.mvb_s2_forward(self._h, b, idx_d.data_ptr(), None if spk_d is None else spk_d.data_ptr(),
                                            float(temperature), int(top_k or 0), None if nz is None else nz.data_ptr(),
                                            int(seed), out.data_ptr(), None if lg is None else lg.data_ptr(), self._st()))
        return (out, lg) if return_logits else out

    @torch.no_grad()
    def non_causal_sample(self, *, texts: List[str], encodec_tokens: List[torch.Tensor], batch_size: int = 1,
                          top_k: Optional[int] = 200, temperature: float = 1.0,
                          speaker_embs: Optional[torch.Tensor] = None, seed: Optional[int] = None) -> List[torch.Tensor]:
        """Same inputs as ``Model.non_causal_sample``; returns one int64 [8, T_f] code tensor per utterance (what the
        reference hands to ``mbd.tokens_to_wav`` after ``TiltedEncodec.decode``, decoders.py:70-79)."""
        if speaker_embs is not None:
            assert len(texts) == len(speaker_embs)
        if seed is None:
            seed = int(torch.randint(0, 2**62, (1,)).item())
        outs = []
        for s0 in range(0, len(texts), self.cfg.max_batch):
            chunk = range(s0, min(len(texts), s0 + self.cfg.max_batch))
            idx = torch.stack([self.build_input(self.tokenizer.encode(texts[i]), encodec_tokens[i][0].tolist()) for i in chunk])
            spk = None if speaker_embs is None else speaker_embs[s0:s0 + len(idx)]
            y = self.forward_tokens(idx, spk, temperature, top_k, seed=seed + s0).cpu()
            for j in range(len(idx)):
                allh = torch.cat([idx[j], y[j]], dim=0).tolist()          # b_tokens = cat([in_x, y], dim=1) (inference.py:329)
                _, codes = tilted_decode(allh)
                outs.append(torch.tensor(codes, dtype=torch.long))
        return outs
