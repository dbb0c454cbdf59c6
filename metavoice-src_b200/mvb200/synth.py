"""Synthetic checkpoints in the reference's on-disk layout.

No real MetaVoice weights exist offline, so every parity test and benchmark runs on
seeded synthetic checkpoints that are laid out exactly like the files the reference
loads (SURVEY.md App. B):

  * ``first_stage.pt``  -> dict(model=state_dict, model_args=..., config=..., meta=...)
    read by ``fam/llm/fast_inference_utils.py:243-280`` (key names are the slow-path
    ``GPT`` names: ``transformer.wtes.0.weight`` ... ``lm_heads.0.weight``).
  * ``second_stage.pt`` -> same container, non-causal ``GPT`` with 2 input / 6 output
    hierarchies, read by ``fam/llm/inference.py:102-141``.

The generator is deterministic for a given (config, seed) on a given torch build, so the
GPU box can regenerate bit-identical weights from the seed instead of shipping 2.5 GB.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, asdict
from typing import Dict, Optional

import torch


@dataclass
class Stage1Dims:
    """Shape parameters of the stage-1 causal LM (fam/llm/fast_model.py:52-94).  norm_type, nonlinearity_type and bias
    select the architecture of the reference's causal ``GPT`` (model.py:26-46); the defaults are the production model's."""

    n_layer: int = 24
    n_head: int = 16
    dim: int = 2048
    vocab_size: int = 2562
    block_size: int = 2048
    speaker_emb_dim: int = 256
    norm_eps: float = 1e-5
    intermediate_size: Optional[int] = None
    norm_type: str = "rmsnorm"
    nonlinearity_type: str = "swiglu"
    bias: bool = False

    def __post_init__(self):
        if self.intermediate_size is None and self.nonlinearity_type == "gelu":
            self.intermediate_size = 4 * self.dim        # fam/llm/layers/layers.py:46
        if self.intermediate_size is None:
            # fam/llm/fast_model.py:69-72: find_multiple(int(2*4*dim/3), 256)
            n_hidden = int(2 * 4 * self.dim / 3)
            self.intermediate_size = n_hidden if n_hidden % 256 == 0 else n_hidden + 256 - (n_hidden % 256)

    @property
    def head_dim(self) -> int:
        return self.dim // self.n_head

    def n_params(self) -> int:
        d, f, v = self.dim, self.intermediate_size, self.vocab_size
        n_mlp = 2 if self.nonlinearity_type == "gelu" else 3
        ln_beta = self.bias and self.norm_type == "layernorm"
        per_layer = 3 * d * d + d * d + n_mlp * d * f + 2 * d
        if self.bias:
            per_layer += 4 * d + (n_mlp - 1) * f + (2 * d if ln_beta else 0)
        return self.n_layer * per_layer + 2 * v * d + self.block_size * d + self.speaker_emb_dim * d + d + (d if ln_beta else 0)


FULL = Stage1Dims()
TINY = Stage1Dims(n_layer=2, n_head=2, dim=256)


def _normal(gen: torch.Generator, shape, std: float) -> torch.Tensor:
    t = torch.empty(shape, dtype=torch.float32)
    t.normal_(mean=0.0, std=std, generator=gen)
    return t.to(torch.bfloat16)


def stage1_state_dict(dims: Stage1Dims, seed: int = 0, tie_head: bool = False) -> Dict[str, torch.Tensor]:
    """bf16 state dict with the reference checkpoint's key names (SURVEY.md App. B).

    Init follows GPT-2 style used by the reference (fam/llm/model.py:151-176): N(0, 0.02),
    ``c_proj`` scaled by 1/sqrt(2*n_layer).  Norm gains are 1 + 0.1*N(0,1) rather than the
    reference's all-ones so that the gain path is actually exercised by parity tests.
    The LM head is drawn independently by default (the reference loads it as a separate
    tensor, fast_inference_utils.py:252) so head and embedding mistakes cannot cancel.
    A GELU MLP draws ``mlp.c_fc`` where SwiGLU draws w1 and has no w3; with ``dims.bias``, LayerNorm betas 0.1 N(0, 1)
    and Linear biases 0.02 N(0, 1) are drawn after every other tensor, non-zero so that a dropped bias changes the
    output.  The default architecture draws exactly the tensors it always has.
    """
    gen = torch.Generator().manual_seed(seed)
    d, f, v = dims.dim, dims.intermediate_size, dims.vocab_size
    gelu, ln = dims.nonlinearity_type == "gelu", dims.norm_type == "layernorm"
    proj_std = 0.02 / math.sqrt(2 * dims.n_layer)
    sd: Dict[str, torch.Tensor] = {}
    sd["transformer.wtes.0.weight"] = _normal(gen, (v, d), 0.02)
    sd["transformer.wpe.weight"] = _normal(gen, (dims.block_size, d), 0.02)
    sd["speaker_cond_pos.weight"] = _normal(gen, (d, dims.speaker_emb_dim), 0.02)
    for i in range(dims.n_layer):
        p = f"transformer.h.{i}."
        sd[p + "ln_1.weight"] = (1.0 + 0.1 * torch.empty(d).normal_(generator=gen)).to(torch.bfloat16)
        sd[p + "attn.c_attn.weight"] = _normal(gen, (3 * d, d), 0.02)
        sd[p + "attn.c_proj.weight"] = _normal(gen, (d, d), proj_std)
        sd[p + "ln_2.weight"] = (1.0 + 0.1 * torch.empty(d).normal_(generator=gen)).to(torch.bfloat16)
        if gelu:
            sd[p + "mlp.c_fc.weight"] = _normal(gen, (f, d), 0.02)
        else:
            sd[p + "mlp.swiglu.w1.weight"] = _normal(gen, (f, d), 0.02)
            sd[p + "mlp.swiglu.w3.weight"] = _normal(gen, (f, d), 0.02)
        sd[p + "mlp.c_proj.weight"] = _normal(gen, (d, f), proj_std)
    sd["transformer.ln_f.weight"] = (1.0 + 0.1 * torch.empty(d).normal_(generator=gen)).to(torch.bfloat16)
    if tie_head:
        sd["lm_heads.0.weight"] = sd["transformer.wtes.0.weight"]
    else:
        sd["lm_heads.0.weight"] = _normal(gen, (v, d), 0.02)
    if dims.bias:
        beta = lambda: _normal(gen, (d,), 0.1)      # noqa: E731
        lin = lambda n: _normal(gen, (n,), 0.02)    # noqa: E731
        if ln:
            sd["transformer.ln_f.bias"] = beta()
        for i in range(dims.n_layer):
            p = f"transformer.h.{i}."
            if ln:
                sd[p + "ln_1.bias"] = beta()
                sd[p + "ln_2.bias"] = beta()
            sd[p + "attn.c_attn.bias"] = lin(3 * d)
            sd[p + "attn.c_proj.bias"] = lin(d)
            if gelu:
                sd[p + "mlp.c_fc.bias"] = lin(f)
            else:
                sd[p + "mlp.swiglu.w1.bias"] = lin(f)
                sd[p + "mlp.swiglu.w3.bias"] = lin(f)
            sd[p + "mlp.c_proj.bias"] = lin(d)
    return sd


def state_dict_checksum(sd: Dict[str, torch.Tensor]) -> float:
    """Cheap order-dependent fingerprint used by golden fixtures to detect RNG drift."""
    acc = 0.0
    for i, (k, t) in enumerate(sorted(sd.items())):
        flat = t.reshape(-1)
        step = max(1, flat.numel() // 4096)
        acc += float(flat[::step].to(torch.float64).sum()) * (1.0 + 0.001 * (i % 97))
    return acc


def synthetic_tokenizer_meta(n_text_tokens: int = 512, offset: int = 2049) -> dict:
    """``meta["tokenizer"]`` kwargs for ``TrainedBPETokeniser`` (fam/quantiser/text/tokenise.py:4-12).

    256 single-byte tokens + (n_text_tokens-256) two-byte merges; EOT id = n_text_tokens so that
    EOT + offset = 2561 as in the real checkpoint (SURVEY.md App. D).
    """
    ranks = {bytes([b]): b for b in range(256)}
    letters = b"etaoinshrdlucmfwypvbgkjqxz "
    rank = 256
    for a in letters:
        for b in letters:
            if rank >= n_text_tokens:
                break
            ranks[bytes([a, b])] = rank
            rank += 1
    assert rank == n_text_tokens
    return dict(
        name="synthetic_bpe",
        pat_str=r"""'s|'t|'re|'ve|'m|'ll|'d| ?\w+| ?[^\s\w]+|\s+""",
        mergeable_ranks=ranks,
        special_tokens={"<|endoftext|>": n_text_tokens},
        offset=offset,
    )


def stage1_model_args(dims: Stage1Dims) -> dict:
    """``first_stage.pt["model_args"]``: the GPTConfig (fam/llm/model.py:26-46) the reference builds the model from."""
    return dict(
        n_layer=dims.n_layer,
        n_head=dims.n_head,
        n_embd=dims.dim,
        block_size=dims.block_size,
        bias=dims.bias,
        vocab_sizes=[dims.vocab_size],
        causal=True,
        target_vocab_sizes=None,
        norm_type=dims.norm_type,
        rmsnorm_eps=dims.norm_eps,
        nonlinearity_type=dims.nonlinearity_type,
        attn_kernel_type="torch_attn",
        spk_emb_on_text=True,
        swiglu_multiple_of=256,
        dropout=0.0,
    )


def stage1_checkpoint(dims: Stage1Dims, seed: int = 0, tie_head: bool = False) -> dict:
    """Full ``first_stage.pt`` container (SURVEY.md App. B)."""
    return dict(
        model=stage1_state_dict(dims, seed, tie_head=tie_head),
        model_args=stage1_model_args(dims),
        config=dict(causal=True),
        meta=dict(tokenizer=synthetic_tokenizer_meta(), speaker_cond=True, speaker_emb_size=dims.speaker_emb_dim),
        iter_num=0,
        best_val_loss=0.0,
    )


def write_stage1_checkpoint(path, dims: Stage1Dims = FULL, seed: int = 0) -> None:
    torch.save(stage1_checkpoint(dims, seed), str(path))


def synthetic_prompt(T: int, seed: int = 7, text_lo: int = 2049, eot: int = 2561) -> torch.Tensor:
    """T-1 text ids uniform in [2049, 2561) followed by EOT (SURVEY.md §8d)."""
    gen = torch.Generator().manual_seed(seed)
    ids = torch.randint(text_lo, eot, (T - 1,), generator=gen, dtype=torch.int64)
    return torch.cat([ids, torch.tensor([eot])]).to(torch.int32)


def synthetic_speaker(seed: int = 11, dim: int = 256) -> torch.Tensor:
    """relu(N(0,1)) L2-normalised: same structure as speaker_encoder/model.py:57-58,101-102."""
    gen = torch.Generator().manual_seed(seed)
    e = torch.relu(torch.randn(1, dim, generator=gen))
    return e / e.norm(dim=-1, keepdim=True)


def dims_as_dict(d: Stage1Dims) -> dict:
    return asdict(d)


# ------------------------------------------------------------------------------------------------ stage 2
@dataclass
class Stage2Dims:
    """Shape of the non-causal codebook-expansion model (fam/llm/model.py:26-46 GPTConfig, causal=False).
    The real values live in second_stage.pt["model_args"] (not available offline); these defaults give the
    "~10 Mn parameters" of README.md:164 and are only used for synthetic checkpoints.  norm_type, nonlinearity_type
    and bias select the architecture (GPTConfig's own defaults are "layernorm", "gelu", True)."""

    n_layer: int = 6
    n_head: int = 6
    n_embd: int = 384
    block_size: int = 1024
    vocab_sizes: tuple = (1538, 1025)        # hierarchy 0: 1024 codes + pad 1024 + 512 text + EOT 1537; hierarchy 1: codes + pad
    target_vocab_sizes: tuple = (1025,) * 6  # codebooks 2..7 (+ pad)
    speaker_emb_dim: int = 256
    rmsnorm_eps: float = 1e-5
    swiglu_multiple_of: int = 256
    norm_type: str = "rmsnorm"
    nonlinearity_type: str = "swiglu"
    bias: bool = False

    @property
    def hidden(self) -> int:
        if self.nonlinearity_type == "gelu":
            return 4 * self.n_embd           # fam/llm/layers/layers.py:46
        h = int(2 * 4 * self.n_embd / 3)    # fam/llm/layers/layers.py:51-52
        m = self.swiglu_multiple_of
        return m * ((h + m - 1) // m)


S2_FULL = Stage2Dims()
S2_TINY = Stage2Dims(n_layer=2, n_head=2, n_embd=128, block_size=256)


def stage2_model_args(d: Stage2Dims) -> dict:
    return dict(n_layer=d.n_layer, n_head=d.n_head, n_embd=d.n_embd, block_size=d.block_size, bias=d.bias,
                vocab_sizes=list(d.vocab_sizes), target_vocab_sizes=list(d.target_vocab_sizes), causal=False,
                norm_type=d.norm_type, rmsnorm_eps=d.rmsnorm_eps, nonlinearity_type=d.nonlinearity_type,
                swiglu_multiple_of=d.swiglu_multiple_of, attn_kernel_type="torch_attn", spk_emb_on_text=True, dropout=0.0)


def stage2_state_dict(d: Stage2Dims, seed: int = 1) -> Dict[str, torch.Tensor]:
    """bf16 state dict with the slow-path GPT key names (fam/llm/model.py:118-146).  The default architecture's tensors
    are drawn first, in a fixed order (GELU: c_fc in place of w1, no w3); then, with bias, LayerNorm betas 0.1 N(0, 1)
    and Linear biases 0.02 N(0, 1), non-zero so that a dropped bias changes the output."""
    gen = torch.Generator().manual_seed(seed)
    gelu, ln = d.nonlinearity_type == "gelu", d.norm_type == "layernorm"
    e, hd = d.n_embd, d.hidden
    proj_std = 0.02 / math.sqrt(2 * d.n_layer)
    gain = lambda: (1.0 + 0.1 * torch.empty(e).normal_(generator=gen)).to(torch.bfloat16)
    sd: Dict[str, torch.Tensor] = {}
    for i, v in enumerate(d.vocab_sizes):
        sd[f"transformer.wtes.{i}.weight"] = _normal(gen, (v, e), 0.02)
    sd["transformer.wpe.weight"] = _normal(gen, (d.block_size, e), 0.02)
    for i in range(d.n_layer):
        p = f"transformer.h.{i}."
        sd[p + "ln_1.weight"] = gain()
        sd[p + "ln_2.weight"] = gain()
        sd[p + "attn.c_attn.weight"] = _normal(gen, (3 * e, e), 0.02)
        sd[p + "attn.c_proj.weight"] = _normal(gen, (e, e), proj_std)
        if gelu:
            sd[p + "mlp.c_fc.weight"] = _normal(gen, (hd, e), 0.02)
        else:
            sd[p + "mlp.swiglu.w1.weight"] = _normal(gen, (hd, e), 0.02)
            sd[p + "mlp.swiglu.w3.weight"] = _normal(gen, (hd, e), 0.02)
        sd[p + "mlp.c_proj.weight"] = _normal(gen, (e, hd), proj_std)
    sd["transformer.ln_f.weight"] = gain()
    sd["speaker_cond_pos.weight"] = _normal(gen, (e, d.speaker_emb_dim), 0.02)
    for i, v in enumerate(d.target_vocab_sizes):
        sd[f"lm_heads.{i}.weight"] = _normal(gen, (v, e), 0.05)
    if d.bias:
        beta = lambda: _normal(gen, (e,), 0.1)      # noqa: E731
        lin = lambda n: _normal(gen, (n,), 0.02)    # noqa: E731
        if ln:
            sd["transformer.ln_f.bias"] = beta()
        for i in range(d.n_layer):
            p = f"transformer.h.{i}."
            if ln:
                sd[p + "ln_1.bias"] = beta()
                sd[p + "ln_2.bias"] = beta()
            sd[p + "attn.c_attn.bias"] = lin(3 * e)
            sd[p + "attn.c_proj.bias"] = lin(e)
            if gelu:
                sd[p + "mlp.c_fc.bias"] = lin(hd)
            else:
                sd[p + "mlp.swiglu.w1.bias"] = lin(hd)
                sd[p + "mlp.swiglu.w3.bias"] = lin(hd)
            sd[p + "mlp.c_proj.bias"] = lin(e)
    return sd


def stage2_checkpoint(d: Stage2Dims, seed: int = 1) -> dict:
    tok = synthetic_tokenizer_meta(offset=1025)  # stage-2 text ids = bpe id + 1025, EOT = 1537 (model.py:15)
    return dict(model=stage2_state_dict(d, seed), model_args=stage2_model_args(d), config=dict(causal=False),
                meta=dict(tokenizer=tok, speaker_cond=True, speaker_emb_size=d.speaker_emb_dim), iter_num=0, best_val_loss=0.0)


def synthetic_stage2_input(d: Stage2Dims, n_frames: int, n_text: int = 12, seed: int = 3):
    """(text ids incl. EOT, cb0[n_frames], cb1[n_frames]) in stage-2 token space (SURVEY.md App. D)."""
    gen = torch.Generator().manual_seed(seed)
    text = torch.randint(1025, 1537, (n_text - 1,), generator=gen).tolist() + [1537]
    cb = torch.randint(0, 1024, (2, n_frames), generator=gen)
    return text, cb[0].tolist(), cb[1].tolist()


# ------------------------------------------------------------------------------------------------ codec
def encodec_model_and_state_dict(seed: int = 0):
    """Random-init EnCodec 24 kHz in the layout of the ``facebook/encodec_24khz`` checkpoint that audiocraft's
    ``MultiBandDiffusion.get_mbd_24khz`` loads (fam/llm/decoders.py:13) through ``transformers.EncodecModel``.
    Returns (module, state_dict); the module is only used by tests as the reference implementation."""
    from transformers import EncodecConfig, EncodecModel
    torch.manual_seed(seed)
    m = EncodecModel(EncodecConfig()).eval()
    with torch.no_grad():
        for q in m.quantizer.layers:           # codebooks are zero-initialised buffers: give them content
            q.codebook.embed.normal_(0.0, 1.0)
    return m, {k: v.detach().clone() for k, v in m.state_dict().items()}


def speaker_encoder_state_dict(seed: int = 3) -> Dict[str, torch.Tensor]:
    """``speaker_encoder.pt["model_state"]`` layout (fam/quantiser/audio/speaker_encoder/model.py:30-32, 45-46):
    ``nn.LSTM(40, 256, 3, batch_first=True)`` + ``nn.Linear(256, 256)``, torch's default U(-1/sqrt(H), 1/sqrt(H)) init."""
    gen = torch.Generator().manual_seed(seed)
    H, k = 256, 1.0 / 16.0
    u = lambda *shape: (torch.rand(*shape, generator=gen) * 2 - 1) * k
    sd: Dict[str, torch.Tensor] = {}
    for l in range(3):
        sd[f"lstm.weight_ih_l{l}"] = u(4 * H, 40 if l == 0 else H)
        sd[f"lstm.weight_hh_l{l}"] = u(4 * H, H)
        sd[f"lstm.bias_ih_l{l}"] = u(4 * H)
        sd[f"lstm.bias_hh_l{l}"] = u(4 * H)
    sd["linear.weight"] = u(H, H)
    sd["linear.bias"] = u(H).abs()          # keeps a healthy fraction of the ReLU outputs alive
    return sd


def synthetic_waveform(seconds: float, sr: int, seed: int = 5):
    """Deterministic speech-like test signal (sum of drifting harmonics + noise bursts), float32 in [-1, 1]."""
    import numpy as np
    rng = np.random.default_rng(seed)
    n = int(seconds * sr)
    t = np.arange(n) / sr
    f0 = 110 + 40 * np.sin(2 * np.pi * 0.7 * t) + 15 * np.sin(2 * np.pi * 3.1 * t)
    phase = 2 * np.pi * np.cumsum(f0) / sr
    sig = sum((0.5 ** h) * np.sin((h + 1) * phase + rng.uniform(0, 6.28)) for h in range(6))
    env = 0.5 * (1 + np.sin(2 * np.pi * 2.3 * t)) * (0.6 + 0.4 * np.sin(2 * np.pi * 0.31 * t + 1.0))
    sig = sig * env + 0.02 * rng.standard_normal(n)
    return (0.3 * sig / np.abs(sig).max()).astype(np.float32)


# ------------------------------------------------------------------------------------------------ multi-band diffusion
def mbd_checkpoint(cfg, seed: int = 0) -> dict:
    """Synthetic multi-band-diffusion checkpoint for a parametrised config (oracle/mbd_port.MBDConfig): per band model a
    DiffusionUnet state dict with audiocraft's module names (models/unet.py) and MultiBandProcessor statistics.  Weights
    are scaled by 1/sqrt(fan_in) so that activations stay O(1) through the 20-step sampler."""
    gen = torch.Generator().manual_seed(seed)
    u = cfg.unet
    ch = u.channels()
    rn = lambda *shape, std=1.0: torch.randn(*shape, generator=gen) * std
    models, proc = [], []
    for _ in range(cfg.n_models):
        sd: Dict[str, torch.Tensor] = {}

        def res(prefix, C):
            for n in ("1", "2"):
                sd[f"{prefix}norm{n}.weight"] = 1.0 + 0.1 * rn(C)
                sd[f"{prefix}norm{n}.bias"] = 0.1 * rn(C)
                sd[f"{prefix}conv{n}.weight"] = rn(C, C, 3, std=0.5 / math.sqrt(3 * C))
                sd[f"{prefix}conv{n}.bias"] = 0.05 * rn(C)

        cin = u.chin
        for i, C in enumerate(ch):
            p = f"encoders.{i}."
            sd[p + "conv.weight"] = rn(C, cin, u.kernel, std=1.0 / math.sqrt(cin * u.kernel))
            sd[p + "norm.weight"] = 1.0 + 0.1 * rn(C)
            sd[p + "norm.bias"] = 0.1 * rn(C)
            for j in range(u.res_blocks):
                res(f"{p}res_blocks.{j}.", C)
            if i == 0:
                sd["embedding.weight"] = 0.3 * rn(u.num_steps, C)
            elif u.emb_all_layers:
                sd[f"embeddings.{i - 1}.weight"] = 0.3 * rn(u.num_steps, C)
            cin = C
        sd["conv_codec.weight"] = rn(ch[-1], u.codec_dim, 1, std=1.0 / math.sqrt(u.codec_dim))
        sd["conv_codec.bias"] = 0.05 * rn(ch[-1])
        for i in range(u.depth):
            lvl = u.depth - 1 - i
            C, cout = ch[lvl], (u.chin if lvl == 0 else ch[lvl - 1])
            p = f"decoders.{i}."
            for j in range(u.res_blocks):
                res(f"{p}res_blocks.{j}.", C)
            sd[p + "norm.weight"] = 1.0 + 0.1 * rn(C)
            sd[p + "norm.bias"] = 0.1 * rn(C)
            sd[p + "convtr.weight"] = rn(C, cout, u.kernel, std=1.0 / math.sqrt(2 * C))
        models.append(sd)
        proc.append(dict(mean=0.01 * rn(cfg.proc_bands), std=1.0 + 0.2 * torch.rand(cfg.proc_bands, generator=gen),
                         target_std=1.0 + 0.2 * torch.rand(cfg.proc_bands, generator=gen)))
    return dict(models=models, proc=proc)
