"""Host-side mirror of ``fam/llm/fast_model.py`` over libmvb200.

Same names and call signatures as the reference (``ModelArgs``, ``Transformer.from_name``,
``setup_spk_cond_mask``, ``setup_caches``, ``forward(idx, spk_emb, input_pos)``) so that
``fam/llm/fast_inference.py`` works by changing one import; the arithmetic runs in
``libmvb200.so``.  PyTorch is used for device memory and streams only.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, List, Optional, Union

import torch

from . import _lib
from ._engine import Engine, pack_arena_bytes


def find_multiple(n: int, k: int) -> int:
    return n if n % k == 0 else n + k - (n % k)


@dataclass
class ModelArgs:
    """fam/llm/fast_model.py:52-84."""
    block_size: int = 2048
    vocab_size: int = 32000
    n_layer: int = 32
    n_head: int = 32
    dim: int = 4096
    speaker_emb_dim: int = 256
    intermediate_size: Optional[int] = None
    n_local_heads: int = -1
    head_dim: int = 64
    norm_eps: float = 1e-5
    dtype: torch.dtype = torch.bfloat16
    # GPTConfig's architecture fields (fam/llm/model.py:36-43); the defaults are the production model's, which is the
    # only architecture the reference's fast path builds.  Any other runs on the engine's per-layer paths.
    norm_type: str = "rmsnorm"
    nonlinearity_type: str = "swiglu"
    bias: bool = False

    def __post_init__(self):
        if self.n_local_heads == -1:
            self.n_local_heads = self.n_head
        if self.intermediate_size is None:
            if self.nonlinearity_type == "gelu":
                self.intermediate_size = 4 * self.dim                   # layers/layers.py:46
            else:
                self.intermediate_size = find_multiple(int(2 * 4 * self.dim / 3), 256)
        self.head_dim = self.dim // self.n_head

    @property
    def production_arch(self) -> bool:
        return (self.norm_type, self.nonlinearity_type, self.bias) == ("rmsnorm", "swiglu", False)

    @classmethod
    def from_name(cls, name: str):
        if name in transformer_configs:
            return cls(**transformer_configs[name])
        config = [c for c in transformer_configs if c in str(name).upper() or c in str(name)]
        assert len(config) == 1, name
        return cls(**transformer_configs[config[0]])


transformer_configs = {"metavoice-1B": dict(n_layer=24, n_head=16, dim=2048, vocab_size=2562)}

# arena order == MVB_S1_GLOBAL_TENSORS / MVB_S1_LAYER_TENSORS in include/mvb200.h; names are the
# checkpoint's (fast_inference_utils.py:250-278 maps them onto the fast model's names)
_GLOBAL_KEYS = ["transformer.wtes.0.weight", "transformer.wpe.weight", "speaker_cond_pos.weight",
                "transformer.ln_f.weight", "lm_heads.0.weight"]
_LAYER_KEYS = ["ln_1.weight", "attn.c_attn.weight", "attn.c_proj.weight", "ln_2.weight",
               "mlp.swiglu.w1.weight", "mlp.swiglu.w3.weight", "mlp.c_proj.weight"]


_KV_DTYPES = {"bf16": _lib.MVB_KV_BF16, "fp32": _lib.MVB_KV_FP32, "fp8": _lib.MVB_KV_FP8}
_NORMS = {"rmsnorm": _lib.MVB_S1_NORM_RMS, "layernorm": _lib.MVB_S1_NORM_LAYER}
_MLPS = {"swiglu": _lib.MVB_S1_MLP_SWIGLU, "gelu": _lib.MVB_S1_MLP_GELU}


def stage1_keys(n_layer: int, norm_type: str = "rmsnorm", nonlinearity_type: str = "swiglu", bias: bool = False) -> List[str]:
    """State-dict keys in the order of mvb_s1_create_ex's offset list (include/mvb200.h): the production list, GELU's
    ``mlp.c_fc`` in place of the two SwiGLU matrices, then the biases (LayerNorm betas only for LayerNorm)."""
    ffn = ["mlp.c_fc"] if nonlinearity_type == "gelu" else ["mlp.swiglu.w1", "mlp.swiglu.w3"]
    layer = ["ln_1", "attn.c_attn", "attn.c_proj", "ln_2"] + ffn + ["mlp.c_proj"]
    keys = list(_GLOBAL_KEYS) + [f"transformer.h.{i}.{k}.weight" for i in range(n_layer) for k in layer]
    if bias:
        ln = norm_type == "layernorm"
        keys += ["transformer.ln_f.bias"] if ln else []
        with_bias = [k for k in layer if ln or not k.startswith("ln_")]
        keys += [f"transformer.h.{i}.{k}.bias" for i in range(n_layer) for k in with_bias]
    return keys


def _layer_keys(i: int, norm_type: str = "rmsnorm", nonlinearity_type: str = "swiglu", bias: bool = False) -> List[str]:
    """Keys of block i: its weights in arena order, then (bias) its biases in arena order."""
    ffn = ["mlp.c_fc"] if nonlinearity_type == "gelu" else ["mlp.swiglu.w1", "mlp.swiglu.w3"]
    layer = ["ln_1", "attn.c_attn", "attn.c_proj", "ln_2"] + ffn + ["mlp.c_proj"]
    keys = [f"transformer.h.{i}.{k}.weight" for k in layer]
    if bias:
        keys += [f"transformer.h.{i}.{k}.bias" for k in layer if norm_type == "layernorm" or not k.startswith("ln_")]
    return keys


def stage1_shapes(c: "ModelArgs") -> List[tuple]:
    """Shapes of the tensors of stage1_keys(c's architecture), in the same order."""
    D, F, V = c.dim, c.intermediate_size, c.vocab_size
    gelu, ln = c.nonlinearity_type == "gelu", c.norm_type == "layernorm"
    ffn = [(F, D)] if gelu else [(F, D), (F, D)]
    layer = [(D,), (3 * D, D), (D, D), (D,)] + ffn + [(D, F)]
    shapes = [(V, D), (c.block_size, D), (D, c.speaker_emb_dim), (D,), (V, D)] + layer * c.n_layer
    if c.bias:
        shapes += [(D,)] if ln else []
        lb = ([(D,)] if ln else []) + [(3 * D,), (D,)] + ([(D,)] if ln else []) + ([(F,)] if gelu else [(F,), (F,)]) + [(D,)]
        shapes += lb * c.n_layer
    return shapes


def overlay_keys(n_layer: int, first_layer: int, norm_type: str = "rmsnorm", nonlinearity_type: str = "swiglu",
                 bias: bool = False) -> List[str]:
    """State-dict keys of a voice overlay in mvb_s1_add_voice's offset order (include/mvb200.h): every tensor of blocks
    [first_layer, n_layer) block by block (weights, then biases), then ln_f.weight and (LayerNorm with bias) ln_f.bias."""
    keys = [k for i in range(first_layer, n_layer) for k in _layer_keys(i, norm_type, nonlinearity_type, bias)]
    keys.append("transformer.ln_f.weight")
    if bias and norm_type == "layernorm":
        keys.append("transformer.ln_f.bias")
    return keys


def strip_compile_prefix(state_dict: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The checkpoint's keys without torch.compile's ``_orig_mod.`` prefix (as _load_model reads them)."""
    return {(k[len("_orig_mod."):] if k.startswith("_orig_mod.") else k): v for k, v in state_dict.items()}


def overlay_first_layer(base: Dict[str, torch.Tensor], finetune: Dict[str, torch.Tensor], config: "ModelArgs") -> int:
    """The first block of the overlay that turns ``base`` into ``finetune``: the longest run of blocks, ending at the last,
    in which every block differs from the base (exact equality of the host tensors), or the last block alone when only
    ln_f differs.  ValueError names the first tensor that is missing, has another shape, or differs outside ln_f and
    that run (an embedding, speaker_cond_pos, the head, or an earlier block): the finetune would not be an overlay."""
    c = config
    keys = stage1_keys(c.n_layer, c.norm_type, c.nonlinearity_type, c.bias)
    for k in keys:
        if k not in finetune:
            raise ValueError(f"the voice checkpoint is missing {k}")
        if tuple(finetune[k].shape) != tuple(base[k].shape):
            raise ValueError(f"{k} has shape {tuple(finetune[k].shape)} in the voice checkpoint, {tuple(base[k].shape)} in the base")
    same = lambda k: torch.equal(base[k].to(torch.bfloat16), finetune[k].to(torch.bfloat16))   # noqa: E731
    block_same = [all(same(k) for k in _layer_keys(i, c.norm_type, c.nonlinearity_type, c.bias)) for i in range(c.n_layer)]
    first = c.n_layer
    while first > 0 and not block_same[first - 1]:
        first -= 1
    first = min(first, c.n_layer - 1)
    overlaid = set(overlay_keys(c.n_layer, first, c.norm_type, c.nonlinearity_type, c.bias))
    for k in keys:
        if k not in overlaid and not same(k):
            raise ValueError(f"the voice checkpoint differs from the base in {k}: only ln_f and a run of blocks ending at the "
                             f"last (blocks {first}..{c.n_layer - 1} here) can be a voice")
    return first


def pack_arena(state_dict: Dict[str, torch.Tensor], n_layer: int, config: Optional["ModelArgs"] = None):
    """Checkpoint state dict -> one contiguous bf16 byte arena (CPU) + byte offsets.
    Replaces the module construction of ``_load_model`` (fast_inference_utils.py:236-281).  ``config`` selects the
    architecture's tensors (default: the production model's)."""
    sd = {(k[len("_orig_mod."):] if k.startswith("_orig_mod.") else k): v for k, v in state_dict.items()}
    c = config or ModelArgs(n_layer=n_layer)
    keys = stage1_keys(n_layer, c.norm_type, c.nonlinearity_type, c.bias)
    for k in keys:
        if k not in sd:
            raise KeyError(f"checkpoint is missing {k}")
    return pack_arena_bytes([sd[k].to(torch.bfloat16) for k in keys])


class KVCache:
    """Placeholder with the reference's attribute names (fast_model.py:97-113); the cache itself is a
    single device buffer owned by the Transformer (layout in DESIGN.md)."""

    def __init__(self, k_cache: torch.Tensor, v_cache: torch.Tensor):
        self.k_cache, self.v_cache = k_cache, v_cache


class Transformer(Engine):
    """Mirror of fam/llm/fast_model.py:116-167 backed by an ``mvb_s1`` engine handle."""

    _voices = ()        # (device overlay, offsets, first_layer) of voices 1, 2, ... (a list once __init__ has run)

    def __init__(self, config: ModelArgs, arena: torch.Tensor, offsets: List[int], device="cuda",
                 quantisation_mode: Optional[str] = None):
        self._check_mode(config, quantisation_mode)
        super().__init__(device, arena, offsets)
        self.config = config
        self.quantisation_mode = quantisation_mode
        self.max_batch_size = -1
        self.max_seq_length = -1
        self.max_utts = 0
        self._spk_key = None
        self.kv_dtype = "bf16"
        self._voices: List[tuple] = []

    # ---- construction ------------------------------------------------------------------------
    @staticmethod
    def _check_mode(config: ModelArgs, quantisation_mode: Optional[str]) -> None:
        if quantisation_mode not in (None, "int4", "int8", "fp8"):
            raise NotImplementedError(f"quantisation_mode={quantisation_mode!r} is not implemented (only None, 'int4', 'int8' "
                                      "and 'fp8')")
        if quantisation_mode is not None and not config.production_arch:
            raise NotImplementedError(f"quantisation_mode={quantisation_mode!r} is implemented for the production architecture "
                                      "(rmsnorm, swiglu, no bias) only")

    @classmethod
    def from_name(cls, name: str):
        raise RuntimeError("mvb200.Transformer holds device weights; use Transformer.from_state_dict(...)")

    @classmethod
    def from_state_dict(cls, state_dict, config: ModelArgs, device="cuda", quantisation_mode: Optional[str] = None):
        """``quantisation_mode="int4"`` quantises wqkv / wo / w1 / w3 / w2 at load (mvb200/quantize.py) and builds an int4
        engine: decode streams the packed weights through k_gemv_w4, prefill dequantises one layer at a time.
        ``quantisation_mode="int8"`` quantises every Linear per output channel at load and builds an int8 engine: decode
        streams the int8 weights through k_gemv_w8, prefill widens one layer's q at a time and scales the GEMM outputs.
        ``quantisation_mode="fp8"`` quantises every Linear to e4m3 per output channel at load and builds an fp8 engine:
        decode of up to 8 utterances reads the weights once per step for all of them through k_gemv_f8, prefill (and a
        larger decode batch) widens one layer's q at a time as int8 does.
        ``config``'s norm_type / nonlinearity_type / bias select the architecture (mvb_s1_create_ex); only the production
        one takes a quantisation mode."""
        cls._check_mode(config, quantisation_mode)   # before the weights are quantised
        from . import quantize as Q
        pack = {None: lambda sd, n: pack_arena(sd, n, config), "int4": Q.pack_arena_int4, "int8": Q.pack_arena_int8,
                "fp8": Q.pack_arena_fp8}[quantisation_mode]
        arena, offsets = pack(state_dict, config.n_layer)[:2]
        return cls(config, arena, offsets, device, quantisation_mode)

    @staticmethod
    def bf16_model_size_bytes(c: ModelArgs) -> int:
        n_mlp = 2 if c.nonlinearity_type == "gelu" else 3
        per_layer = 4 * c.dim * c.dim + n_mlp * c.dim * c.intermediate_size + 2 * c.dim
        if c.bias:   # c_attn, attn.c_proj, the MLP Linears, and the LayerNorm betas
            per_layer += 4 * c.dim + (n_mlp - 1) * c.intermediate_size + (2 * c.dim if c.norm_type == "layernorm" else 0)
        n = c.n_layer * per_layer + 2 * c.vocab_size * c.dim + c.block_size * c.dim + c.speaker_emb_dim * c.dim + c.dim
        if c.bias and c.norm_type == "layernorm":
            n += c.dim
        return n * 2

    @staticmethod
    def int4_model_size_bytes(c: ModelArgs) -> int:
        """Bytes of the int4 arena's tensors: 4-bit weights plus one bf16 (scale, zero) pair per 128 of them for the five
        layer matrices, bf16 for everything else (speaker_cond_pos is held as its dequantised bf16 weight)."""
        mats = 4 * c.dim * c.dim + 3 * c.dim * c.intermediate_size
        per_layer = mats // 2 + mats // 128 * 4 + 2 * c.dim * 2
        rest = 2 * c.vocab_size * c.dim + c.block_size * c.dim + c.speaker_emb_dim * c.dim + c.dim
        return c.n_layer * per_layer + rest * 2

    @staticmethod
    def int8_model_size_bytes(c: ModelArgs) -> int:
        """Bytes of the int8 arena's tensors == the reference's ``model_size`` of its int8 model: int8 weights plus one bf16
        scale per output row for every Linear (the five layer matrices, speaker_cond_pos, lm_head), bf16 for the rest."""
        D, F, V = c.dim, c.intermediate_size, c.vocab_size
        per_layer = 4 * D * D + 3 * D * F + (3 * D + D + 2 * F + D) * 2 + 2 * D * 2
        linear_rest = c.speaker_emb_dim * D + D * 2 + V * D + V * 2
        return c.n_layer * per_layer + linear_rest + (V * D + c.block_size * D + D) * 2

    def model_size_bytes(self) -> int:
        """Σ numel*itemsize of parameters == the reference's ``model_size`` (utils:348) before caches; for an int4 engine
        the bytes its arena's tensors occupy, so that main()'s bandwidth figure counts the bytes actually read."""
        if self.quantisation_mode == "int4":
            return self.int4_model_size_bytes(self.config)
        if self.quantisation_mode in ("int8", "fp8"):   # one byte per weight plus one bf16 scale per row, either way
            return self.int8_model_size_bytes(self.config)
        return self.bf16_model_size_bytes(self.config)

    def setup_spk_cond_mask(self):
        # fast_model.py:132-134: row 0 conditioned, row 1 unconditioned -- built into the kernels.
        self.spk_cond_mask = torch.zeros((2, 1, self.config.dim), dtype=torch.bool)
        self.spk_cond_mask[0] = 1

    def setup_caches(self, max_batch_size: int, max_seq_length: int, kv_dtype: str = "bf16", max_new: Optional[int] = None,
                     tensor_core_path: Union[None, bool, str] = None, unfused_sampler: Optional[bool] = None,
                     trace: Optional[bool] = None):
        """fast_model.py:136-148.  ``max_batch_size`` counts rows: 2 per utterance (CFG pair).
        ``kv_dtype``: "bf16" (the reference's cache), "fp32" (validation) or "fp8" (e4m3 codes with one bf16 scale per head
          vector, half the bytes; mvb200/quantize.py quantize_kv_fp8); any other string is a ValueError.
        Test / tool hooks, the engine's ``options`` (include/mvb200.h); any of them given creates a new engine:
          ``tensor_core_path``: True / "BC" = every engine path, False / "" = CUDA-core kernels only, "B" = tensor-core rows
            path without the resident decode kernel, "C" = resident decode kernel with CUDA-core prefill;
          ``unfused_sampler``: the resident kernel leaves the logits to k_sample;
          ``trace``: the resident kernel records per-phase clocks for mvb_s1_trace_fetch."""
        if kv_dtype not in _KV_DTYPES:
            raise ValueError(f"kv_dtype={kv_dtype!r}: expected one of {sorted(_KV_DTYPES)}")
        if (self._h is not None and self.max_seq_length >= max_seq_length and self.max_batch_size >= max_batch_size
                and kv_dtype == self.kv_dtype and tensor_core_path is None and unfused_sampler is None and trace is None):
            return
        c = self.config
        if max_batch_size % 2:
            raise ValueError("max_batch_size must be even: every utterance owns a {cond, uncond} row pair")
        if find_multiple(max_seq_length, 8) != c.block_size:
            raise ValueError("the engine sizes the KV cache to block_size slots per row")
        self.close()
        self.max_seq_length, self.max_batch_size = c.block_size, max_batch_size
        self.max_utts = max_batch_size // 2
        self.kv_dtype = kv_dtype
        if tensor_core_path is None or isinstance(tensor_core_path, bool):
            paths = "" if tensor_core_path is False else "BC"
        else:
            paths = str(tensor_core_path)
        options = ((0 if "B" in paths else _lib.MVB_S1_NO_ROWS_PATH) | (0 if "C" in paths else _lib.MVB_S1_NO_RESIDENT) |
                   (_lib.MVB_S1_UNFUSED_SAMPLER if unfused_sampler else 0) | (_lib.MVB_S1_TRACE if trace else 0))
        cfg = _lib.S1Config(c.n_layer, c.n_head, c.head_dim, c.dim, c.intermediate_size, c.vocab_size, c.block_size,
                            c.speaker_emb_dim, c.norm_eps, self.max_utts,
                            _KV_DTYPES[kv_dtype], max_new or c.block_size, options)
        self._cfg = cfg
        workspace_bytes, create = {None: (self._lib.mvb_s1_workspace_bytes, self._lib.mvb_s1_create),
                                   "int4": (self._lib.mvb_s1_int4_workspace_bytes, self._lib.mvb_s1_create_int4),
                                   "int8": (self._lib.mvb_s1_int8_workspace_bytes, self._lib.mvb_s1_create_int8),
                                   "fp8": (self._lib.mvb_s1_fp8_workspace_bytes, self._lib.mvb_s1_create_fp8)}[self.quantisation_mode]
        if not c.production_arch:
            self._arch = _lib.S1Arch(_NORMS[c.norm_type], _MLPS[c.nonlinearity_type], int(c.bias))
            create = lambda cfg_p, *rest: self._lib.mvb_s1_create_ex(cfg_p, C.byref(self._arch), *rest)   # noqa: E731
        self._create(create, self._lib.mvb_s1_destroy, cfg, self._lib.mvb_s1_kv_bytes, workspace_bytes)
        self._spk_key = None
        for i, v in enumerate(self._voices):          # a new handle: the voices keep their ids
            self._register_voice(*v, want=i + 1)

    # ---- voices ---------------------------------------------------------------------------------
    @property
    def n_voices(self) -> int:
        """Voices the engine serves, voice 0 (the base checkpoint) included."""
        return 1 + len(self._voices)

    def add_voice(self, checkpoint) -> int:
        """Register a last-N-block finetune of the base checkpoint (fam/llm/finetune.py trains ln_f and the last
        ``last_n_blocks_to_finetune`` blocks) and return its voice id.  ``checkpoint``: a ``first_stage.pt`` dict (its
        ``model_args`` must describe the base's architecture) or a bare state dict; ``_orig_mod.`` prefixes are stripped as
        _load_model strips them.  Only the overlaid blocks and ln_f are packed into their own device tensor, kept alive
        with the engine.  ValueError when the checkpoint is not such a finetune (overlay_first_layer); NotImplementedError
        on a quantised engine, before any weight is read."""
        if self.quantisation_mode is not None:
            raise NotImplementedError(f"voices are served by bf16-weight engines only (quantisation_mode="
                                      f"{self.quantisation_mode!r})")
        if self.n_voices >= _lib.MVB_S1_MAX_VOICES:
            raise ValueError(f"the engine already serves {self.n_voices} voices (at most {_lib.MVB_S1_MAX_VOICES})")
        c = self.config
        sd = checkpoint
        if isinstance(checkpoint, dict) and "model" in checkpoint:
            from .fast_inference_utils import stage1_arch
            sd = strip_compile_prefix(checkpoint["model"])
            args = checkpoint.get("model_args", {})
            arch = stage1_arch(args, sd)
            if arch != (c.norm_type, c.nonlinearity_type, c.bias):
                raise ValueError(f"the voice checkpoint's architecture {arch} is not the base's "
                                 f"{(c.norm_type, c.nonlinearity_type, c.bias)}")
            for key, want in (("n_layer", c.n_layer), ("n_head", c.n_head), ("n_embd", c.dim), ("block_size", c.block_size)):
                if args.get(key, want) != want:
                    raise ValueError(f"the voice checkpoint's model_args[{key!r}] = {args[key]!r}, the base's is {want!r}")
        else:
            sd = strip_compile_prefix(sd)
        first = overlay_first_layer(self._base_tensors(), sd, c)
        arena, offsets = pack_arena_bytes([sd[k].to(torch.bfloat16)
                                           for k in overlay_keys(c.n_layer, first, c.norm_type, c.nonlinearity_type, c.bias)])
        voice = (arena.to(self.device), offsets, first)
        if self._h is not None:
            self._register_voice(*voice, want=self.n_voices)
        self._voices.append(voice)
        return len(self._voices)

    def _base_tensors(self) -> Dict[str, torch.Tensor]:
        """The base checkpoint's bf16 tensors, read back from the engine's arena (one host copy, freed with the result)."""
        c = self.config
        arena = self._arena.cpu()
        out = {}
        for k, o, shape in zip(stage1_keys(c.n_layer, c.norm_type, c.nonlinearity_type, c.bias), self._offsets,
                               stage1_shapes(c)):
            n = 1
            for d in shape:
                n *= d
            out[k] = arena[o:o + 2 * n].view(torch.bfloat16).view(shape)
        return out

    def _register_voice(self, overlay: torch.Tensor, offsets: List[int], first_layer: int, want: int) -> None:
        offs = (C.c_uint64 * len(offsets))(*offsets)
        vid = C.c_int32()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.mvb_s1_add_voice(self.handle, overlay.data_ptr(), overlay.numel(), first_layer, offs,
                                                  len(offsets), C.byref(vid)))
        assert vid.value == want, (vid.value, want)

    def voice_id(self, voice) -> int:
        """A voice id of this engine (None: the base, 0) -> int; KeyError for any other value."""
        if voice is None:
            return 0
        if isinstance(voice, bool) or not isinstance(voice, int) or not 0 <= voice < self.n_voices:
            raise KeyError(f"voice {voice!r} is not registered (ids 0 .. {self.n_voices - 1})")
        return voice

    def set_voice(self, utt: int, voice) -> None:
        """Select the voice of slot ``utt`` for its next admission (mvb_s1_set_voice)."""
        _lib.check(self._lib.mvb_s1_set_voice(self.handle, utt, self.voice_id(voice)))

    # ---- helpers --------------------------------------------------------------------------------
    @property
    def handle(self):
        if self._h is None:
            raise RuntimeError("call setup_caches() first")
        return self._h

    @property
    def _kv(self):
        """The KV cache: the first device buffer the handle is created over."""
        return self._ws[0]

    _stream = Engine._st

    def set_speaker(self, utt: int, spk_emb: torch.Tensor):
        e = spk_emb.detach().reshape(-1).to(device=self.device, dtype=torch.float32).contiguous()
        assert e.numel() == self.config.speaker_emb_dim
        _lib.check(self._lib.mvb_s1_set_speaker(self.handle, utt, e.data_ptr(), self._stream()))
        self._keepalive = e

    # ---- Transformer.forward (fast_model.py:150-163) -------------------------------------------
    def forward(self, idx: torch.Tensor, spk_emb: torch.Tensor, input_pos: torch.Tensor, utt: int = 0) -> torch.Tensor:
        """idx int [2,S]; spk_emb [1,speaker_emb_dim]; input_pos int [S] (must be consecutive).
        Returns fp32 logits [2,S,vocab] and updates the KV cache at ``input_pos``."""
        B, S = idx.shape
        if B != 2:
            raise ValueError("idx must hold the {cond, uncond} row pair of one utterance")
        ip = input_pos.detach().to("cpu", torch.int64)
        pos0 = int(ip[0])
        if S > 1 and not torch.equal(ip, torch.arange(pos0, pos0 + S)):
            raise ValueError("input_pos must be consecutive positions")
        self.set_speaker(utt, spk_emb)
        idx_d = idx.detach().to(device=self.device, dtype=torch.int32).contiguous()
        logits = torch.empty((2, S, self.config.vocab_size), dtype=torch.float32, device=self.device)
        _lib.check(self._lib.mvb_s1_forward(self.handle, utt, idx_d.data_ptr(), S, pos0, logits.data_ptr(), 1,
                                            self._stream()))
        return logits

    __call__ = forward
