"""Host-side mirror of ``fam/llm/fast_inference_utils.py`` over libmvb200.

Same seams as the reference: ``sample``, ``prefill``, ``decode_one_token``, ``decode_n_tokens``,
``generate``, ``build_model``, ``main`` keep their names, argument meaning and error behaviour.
There is no ``torch.compile`` step: ``build_model`` returns in the time it takes to read the
checkpoint (the reference needs 30-120 s, README.md:98).
"""
from __future__ import annotations

import ctypes as C
import math
import time
import warnings
from pathlib import Path
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _lib
from .fast_model import ModelArgs, Transformer


def device_sync(device):
    if "cuda" in str(device):
        torch.cuda.synchronize()


def _f(v, default=None) -> Optional[float]:
    if v is None:
        return default
    return float(v.item()) if isinstance(v, torch.Tensor) else float(v)


def _sampling_struct(guidance_scale, temperature, top_p=None, top_k=None, end_of_audio_token=2048, seed=0):
    return _lib.Sampling(_f(guidance_scale), _f(temperature), _f(top_p, -1.0), int(top_k) if top_k else 0,
                         int(end_of_audio_token), int(seed) & (2**64 - 1))


def split_guidance(guidance_scale, end_of_text_token: Optional[int] = None, *, need_eot: bool = True
                   ) -> Tuple[float, Optional[float]]:
    """``guidance_scale`` as the fast path's scalar g, or as the reference's pair ``(s, p)`` of speaker and prompt guidance
    (mixins/causal.py:89-105) -> ``(s, p)`` with ``p = None`` when there is no prompt guidance: a scalar, or ``p == 1``,
    which is the scalar ``s`` exactly.  A pair must have finite scales >= 1 (the reference asserts both), and ``p > 1``
    needs ``end_of_text_token`` (unless ``need_eot`` is False): the uncond-prompt row sees every text token as
    end-of-text (causal.py:259-262)."""
    if not isinstance(guidance_scale, (tuple, list)):
        return guidance_scale, None
    if len(guidance_scale) != 2:
        raise ValueError(f"guidance_scale must be a float or a pair (speaker, prompt), got {guidance_scale!r}")
    s, p = (_f(v) for v in guidance_scale)
    if not (math.isfinite(s) and math.isfinite(p) and s >= 1 and p >= 1):
        raise ValueError(f"guidance_scale {(s, p)}: both scales must be finite and >= 1")
    if p == 1:
        return s, None
    if need_eot and end_of_text_token is None:
        raise ValueError("prompt guidance (guidance_scale=(s, p) with p > 1) needs end_of_text_token=")
    return s, p


# ---- fast_inference_utils.py:107-120 --------------------------------------------------------------
def sample(logits: torch.Tensor, guidance_scale, temperature, top_p=None, top_k=None, *, model: Transformer = None,
           q: Optional[torch.Tensor] = None):
    """logits [2, S, V] -> (idx_next int32 [1], probs [V]).  The Exp(1) noise ``q`` is drawn with torch's
    generator exactly where the reference draws it (``multinomial_sample_one_no_sync``, utils:61-65) unless
    supplied, then everything else runs in one CUDA kernel.  ``guidance_scale=(s, p)`` with p > 1 takes logits
    [3, S, V] = {cond, uncond speaker, uncond prompt} and mixes them as the reference's ``_sample_next_token``
    (mixins/causal.py:89-105); ``(s, 1.0)`` is ``s``."""
    model = model or sample.default_model
    s, p = split_guidance(guidance_scale, need_eot=False)
    rows = 2 if p is None else 3
    if logits.shape[0] < rows:
        raise ValueError(f"logits have {logits.shape[0]} rows; guidance_scale={guidance_scale!r} needs {rows}")
    lg = logits[:, -1].to(torch.float32).contiguous()
    V = lg.shape[-1]
    if q is None:
        q = torch.empty(V, dtype=torch.float32, device=lg.device).exponential_(1)
    q = q.to(device=lg.device, dtype=torch.float32).contiguous()
    tok = torch.empty(1, dtype=torch.int32, device=lg.device)
    probs = torch.empty(V, dtype=torch.float32, device=lg.device)
    sp = _sampling_struct(s, temperature, top_p, top_k)
    if p is None:
        _lib.check(model._lib.mvb_s1_sample(model.handle, lg.data_ptr(), C.byref(sp), q.data_ptr(), 0, tok.data_ptr(),
                                            probs.data_ptr(), model._stream()))
    else:
        _lib.check(model._lib.mvb_s1_sample_guided(model.handle, lg.data_ptr(), C.byref(sp), p, q.data_ptr(), 0,
                                                   tok.data_ptr(), probs.data_ptr(), model._stream()))
    return tok, probs


sample.default_model = None


# ---- fast_inference_utils.py:123-145 --------------------------------------------------------------
def prefill(model: Transformer, x: torch.Tensor, spk_emb: torch.Tensor, input_pos: torch.Tensor, **sampling_kwargs):
    logits = model(x, spk_emb, input_pos)
    return sample(logits, model=model, **sampling_kwargs)[0]


def decode_one_token(model: Transformer, x: torch.Tensor, spk_emb: torch.Tensor, input_pos: torch.Tensor,
                     **sampling_kwargs) -> Tuple[torch.Tensor, torch.Tensor]:
    assert input_pos.shape[-1] == 1
    logits = model(x, spk_emb, input_pos)
    return sample(logits, model=model, **sampling_kwargs)


# ---- fast_inference_utils.py:148-174 (step-at-a-time seam, kept for callers that drive the loop) ----
def decode_n_tokens(model: Transformer, cur_token: torch.Tensor, spk_emb: torch.Tensor, input_pos: torch.Tensor,
                    num_new_tokens: int, callback=lambda _: _, return_probs: bool = False,
                    end_of_audio_token: int = 2048, **sampling_kwargs):
    new_tokens, new_probs = [], []
    for _ in range(num_new_tokens):
        if (cur_token == end_of_audio_token).any():
            break
        next_token, next_prob = decode_one_token(model, cur_token, spk_emb, input_pos, **sampling_kwargs)
        input_pos += 1
        new_tokens.append(next_token.clone())
        callback(new_tokens[-1])
        if return_probs:
            new_probs.append(next_prob.clone())
        cur_token = next_token.view(1, -1).repeat(2, 1)
    return new_tokens, new_probs


# ---- fast_inference_utils.py:181-228 --------------------------------------------------------------
@torch.no_grad()
def generate(model: Transformer, prompt: torch.Tensor, spk_emb: torch.Tensor, *, max_new_tokens: Optional[int] = None,
             callback=lambda x: x, end_of_audio_token: int = 2048, noise: Optional[torch.Tensor] = None,
             forced: Optional[torch.Tensor] = None, voice: Optional[int] = None, **sampling_kwargs) -> torch.Tensor:
    """Same contract as the reference: returns prompt ++ generated tokens (EOA included if emitted).
    The whole decode loop (sampler, EOA latch, position bump) runs on the device; ``noise`` / ``forced``
    are parity-test hooks (Exp(1) draws in the reference's call order / teacher-forced feedback).
    ``callback`` is invoked once per generated token, in order, like the reference's (utils:168) -- after the device
    loop has finished, since there is no per-token host round trip to hook into."""
    out = generate_batch(model, [prompt], spk_emb.reshape(1, -1), max_new_tokens=max_new_tokens,
                         end_of_audio_token=end_of_audio_token, noise=None if noise is None else noise[None],
                         forced=None if forced is None else forced[None], voices=None if voice is None else [voice], **sampling_kwargs)[0]
    for t in out[1:]:          # decode_n_tokens calls back for every token after the prefill sample (utils:166-168)
        callback(t.view(1))
    seq = torch.cat([prompt.to(torch.int32).cpu(), out]).to(prompt.device)
    return seq


def draw_reference_noise(n_utts: int, n_steps: int, vocab: int, device, rng: str) -> torch.Tensor:
    """The Exp(1) draws ``multinomial_sample_one_no_sync`` makes (utils:61-65: ``torch.empty_like(probs).exponential_(1)``,
    ONE [vocab]-sized draw per generated token) taken from torch's global generator in the reference's call order, so
    that ``torch.manual_seed(s); generate(...)`` yields the reference's token ids.
      rng="torch"     : the generator of the device the model lives on -- what the reference consumes when it runs on
                        a GPU (one exponential_ call per token: CUDA Philox offsets advance per call);
      rng="torch-cpu" : the CPU generator -- what the reference consumes when it runs on CPU (the golden vectors under
                        tests/golden were produced that way).  Returns a DEVICE tensor [n_utts, n_steps, vocab]."""
    if rng == "torch-cpu":
        q = torch.stack([torch.stack([torch.empty(vocab).exponential_(1) for _ in range(n_steps)]) for _ in range(n_utts)])
        return q.to(device)
    q = torch.empty((n_utts, n_steps, vocab), dtype=torch.float32, device=device)
    for u in range(n_utts):
        for s in range(n_steps):
            q[u, s].exponential_(1)
    return q


@torch.no_grad()
def generate_batch(model: Transformer, prompts, spk_embs: torch.Tensor, *, max_new_tokens: Optional[int] = None,
                   end_of_audio_token: int = 2048, noise=None, forced=None, seed: Optional[int] = None,
                   guidance_scale=3.0, temperature=1.0, top_p=None, top_k=None, return_sampled: bool = False,
                   rng: Optional[str] = None, end_of_text_token: Optional[int] = None, voices=None):
    """N independent utterances decoded together with per-utterance positions (the batching semantics of
    fam/llm/mixins/causal.py:179-287, numerically equal to running each utterance alone).  Goes through the
    HOST-buffer plugin call ``mvb_s1_generate``: prompts/speakers are copied host->device and the tokens
    device->host inside the call.

    Randomness: ``noise`` (explicit Exp(1) draws) > ``seed`` (on-device Philox stream keyed by it) > ``rng``.
    With neither ``noise`` nor ``seed`` the draws come from torch's global generator exactly where the reference
    takes them (``rng="torch"``, see ``draw_reference_noise``); ``rng="philox"`` selects the on-device stream keyed
    from torch's generator instead (no noise buffer, used by the throughput benchmark).

    Prompt guidance: ``guidance_scale=(s, p)`` with p > 1 is the reference's three-row CFG (mixins/causal.py:89-105,
    224-262) and needs ``end_of_text_token``; each utterance i then takes slot i plus companion slot n + i, so the engine
    needs 2 n slots, and the loop runs through ``mvb_s1_admit_guided`` / ``mvb_s1_decode`` / ``mvb_s1_poll``.
    ``(s, 1.0)`` is ``s``.

    ``voices``: one voice id per utterance (``Transformer.add_voice``; None = the base checkpoint), or None for all on
    the base.  A prompt-guided utterance's companion runs on its voice too."""
    n = len(prompts)
    vids = None if voices is None else [model.voice_id(v) for v in voices]   # KeyError before any work
    if vids is not None and len(vids) != n:
        raise ValueError(f"{len(vids)} voices for {n} prompts")
    s_g, p_g = split_guidance(guidance_scale, end_of_text_token)
    if p_g is not None:
        if 2 * n > model.max_utts:
            raise ValueError(f"{n} prompt-guided utterances need {2 * n} slots; setup_caches set up {model.max_utts}")
        if forced is not None:
            raise ValueError("teacher forcing is not available with prompt guidance")
    guidance_scale = s_g
    if n > model.max_utts:
        raise ValueError(f"{n} utterances exceed the {model.max_utts} slots set up by setup_caches")
    lens = np.asarray([int(p.numel()) for p in prompts], dtype=np.int32)
    block = model.config.block_size
    if max_new_tokens is None:
        max_new = block - int(lens.min())
    else:
        max_new = int(max_new_tokens)
    for T in lens:  # utils:196-204
        if min(T + max_new, block) - T <= 0:
            raise ValueError("Prompt is too long to generate more tokens")
    max_new = min(max_new, model._cfg.max_new)
    flat = np.concatenate([p.detach().cpu().numpy().astype(np.int32).reshape(-1) for p in prompts])
    spk = np.ascontiguousarray(spk_embs.detach().to("cpu", torch.float32).numpy().reshape(n, -1))
    if rng is None:
        rng = "philox" if seed is not None else "torch"
    d_noise = None
    if noise is None and seed is None and rng in ("torch", "torch-cpu"):
        d_noise = draw_reference_noise(n, max_new, model.config.vocab_size, model.device, rng)
    if seed is None:  # tie the on-device Philox stream to torch's global generator (torch.manual_seed reproducible)
        seed = int(torch.randint(0, 2**62, (1,)).item()) if d_noise is None else 0
    params = (_lib.Sampling * n)(*[_sampling_struct(guidance_scale, temperature, top_p, top_k, end_of_audio_token,
                                                    seed + 7919 * i) for i in range(n)])
    out = np.zeros((n, max_new), dtype=np.int32)
    out_lens = np.zeros(n, dtype=np.int32)
    nz = None if noise is None else np.ascontiguousarray(noise.detach().cpu().numpy().astype(np.float32))
    fc = None if forced is None else np.ascontiguousarray(forced.detach().cpu().numpy().astype(np.int32))
    if nz is not None:
        assert nz.shape == (n, max_new, model.config.vocab_size), nz.shape
    if fc is not None:
        assert fc.shape == (n, max_new), fc.shape
    vp = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    if getattr(model, "n_voices", 1) > 1:
        for i in range(n):
            model.set_voice(i, 0 if vids is None else vids[i])
    if p_g is not None:
        if nz is not None:
            d_noise = torch.from_numpy(nz).to(model.device)
        offs = np.concatenate([[0], np.cumsum(lens)])
        return _generate_guided(model, [flat[offs[i]:offs[i + 1]] for i in range(n)], spk, params, p_g, int(end_of_text_token),
                                max_new, d_noise, return_sampled)
    noise_arg, on_dev = (C.c_void_p(d_noise.data_ptr()), 1) if d_noise is not None else (vp(nz), 0)
    _lib.check(model._lib.mvb_s1_generate(model.handle, n, vp(flat), vp(lens), vp(spk), params, max_new, noise_arg, on_dev,
                                          vp(fc), vp(out), vp(out_lens), model._stream()))
    fed = [torch.from_numpy(out[i, :out_lens[i]].copy()) for i in range(n)]
    if not return_sampled:
        return fed
    # test hook: the sampler's own draws (they differ from the fed-back tokens only under teacher forcing)
    sampled = []
    for i in range(n):
        buf = np.zeros(int(out_lens[i]), dtype=np.int32)
        _lib.check(model._lib.mvb_s1_fetch_sampled(model.handle, i, vp(buf), int(out_lens[i]), model._stream()))
        sampled.append(torch.from_numpy(buf))
    return fed, sampled


def _generate_guided(model: Transformer, prompts, spk: np.ndarray, params, prompt_guidance: float, end_of_text_token: int,
                     max_new: int, d_noise: Optional[torch.Tensor], return_sampled: bool):
    """generate_batch's prompt-guided loop: utterance i in slot i with companion slot n + i, decoded in bursts until every
    done flag latches.  ``d_noise``: DEVICE Exp(1) draws [n, max_new, vocab] or None (on-device Philox)."""
    lib, h, st = model._lib, model.handle, model._stream()
    n = len(prompts)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    for i in range(n):
        pr = np.ascontiguousarray(prompts[i], dtype=np.int32)
        sv = np.ascontiguousarray(spk[i], dtype=np.float32)
        dn = None if d_noise is None else C.c_void_p(d_noise[i].data_ptr())
        _lib.check(lib.mvb_s1_admit_guided(h, i, n + i, vp(pr), int(pr.size), vp(sv), C.byref(params[i]), prompt_guidance,
                                           end_of_text_token, max_new, dn, st))
    done = np.zeros(2 * n, dtype=np.int32)
    n_gen = np.zeros(2 * n, dtype=np.int32)
    while True:
        _lib.check(lib.mvb_s1_poll(h, 2 * n, vp(done), vp(n_gen), st))
        if done[:n].all():
            break
        _lib.check(lib.mvb_s1_decode(h, 2 * n, 32, st))
    fed, sampled = [], []
    for i in range(n):
        buf = np.zeros(int(n_gen[i]), dtype=np.int32)
        _lib.check(lib.mvb_s1_fetch(h, i, vp(buf), int(buf.size), None, None, st))
        fed.append(torch.from_numpy(buf))
        if return_sampled:
            sb = np.zeros(int(n_gen[i]), dtype=np.int32)
            _lib.check(lib.mvb_s1_fetch_sampled(h, i, vp(sb), int(sb.size), st))
            sampled.append(torch.from_numpy(sb))
    return (fed, sampled) if return_sampled else fed


def encode_tokens(tokenizer, text: str, device="cuda") -> torch.Tensor:
    return torch.tensor(tokenizer.encode(text), dtype=torch.int, device=device)


# ---- fast_inference_utils.py:236-321 ---------------------------------------------------------------
_ARCH_VALUES = {"norm_type": ("rmsnorm", "layernorm"), "nonlinearity_type": ("swiglu", "gelu"), "bias": (False, True)}
_PRODUCTION_ARCH = {"norm_type": "rmsnorm", "nonlinearity_type": "swiglu", "bias": False}


def stage1_arch(model_args: dict, state_dict: Dict[str, torch.Tensor]) -> Tuple[str, str, bool]:
    """(norm_type, nonlinearity_type, bias) of a first-stage checkpoint, the GPTConfig fields (model.py:36-43) the
    reference's slow path builds ``GPT(GPTConfig(**model_args))`` from (inference.py:102-156).

    A key present in ``model_args`` is taken as it is.  A missing key means what the fast path has always assumed
    (rmsnorm, swiglu, no bias), not GPTConfig's own default (layernorm, gelu, bias): checkpoints the reference writes
    always carry all three keys (finetune.py).  A state dict that contradicts an assumed value -- ``mlp.c_fc`` weights
    without ``nonlinearity_type``, any ``.bias`` tensor without ``bias`` -- raises ValueError naming the missing key.
    What the engine does not build raises NotImplementedError naming the key: an unknown value, spk_emb_on_text=False,
    more than one input hierarchy."""
    arch = {}
    for key, values in _ARCH_VALUES.items():
        v = model_args.get(key, _PRODUCTION_ARCH[key])
        if not any(v is x or (type(v) is type(x) and v == x) for x in values):
            raise NotImplementedError(f"model_args[{key!r}] = {v!r} is not supported (one of {values})")
        arch[key] = v
    if "nonlinearity_type" not in model_args and any(k.endswith(".mlp.c_fc.weight") for k in state_dict):
        raise ValueError("model_args has no 'nonlinearity_type' but the state dict holds mlp.c_fc weights (a GELU MLP): "
                         "set nonlinearity_type")
    if "bias" not in model_args and any(k.endswith(".bias") for k in state_dict):
        raise ValueError("model_args has no 'bias' but the state dict holds .bias tensors: set bias")
    if model_args.get("spk_emb_on_text", True) is not True:
        raise NotImplementedError("model_args['spk_emb_on_text'] = False is not supported (speaker on text tokens only)")
    if len(model_args.get("vocab_sizes") or [None]) > 1:
        raise NotImplementedError(f"model_args['vocab_sizes'] = {model_args['vocab_sizes']!r}: more than one input "
                                  "hierarchy is not supported")
    return arch["norm_type"], arch["nonlinearity_type"], arch["bias"]


def _load_model(checkpoint_path, spk_emb_ckpt_path, device, precision, quantisation_mode=None, n_head: int = None):
    if quantisation_mode is not None:
        if quantisation_mode not in ("int4", "int8", "fp8"):
            raise Exception(f"Invalid quantisation mode {quantisation_mode}! Must be one of 'int4', 'int8' or 'fp8'!")
        if quantisation_mode in ("int8", "fp8") and torch.device(device).type != "cuda":
            raise NotImplementedError(f"{quantisation_mode} weight-only quantisation runs on the CUDA engine only; there is no "
                                      "CPU engine")
    checkpoint = torch.load(str(checkpoint_path), mmap=True, weights_only=False)
    sd = checkpoint["model"]
    args = checkpoint.get("model_args", {})
    sd0 = {(k[len("_orig_mod."):] if k.startswith("_orig_mod.") else k): v for k, v in sd.items()}
    norm_type, nonlinearity_type, bias = stage1_arch(args, sd0)
    if quantisation_mode is not None and (norm_type, nonlinearity_type, bias) != ("rmsnorm", "swiglu", False):
        # before any weight is read (the checkpoint is memory-mapped)
        raise NotImplementedError(f"quantisation_mode={quantisation_mode!r} is implemented for the production architecture "
                                  f"only; model_args['norm_type', 'nonlinearity_type', 'bias'] = "
                                  f"{(norm_type, nonlinearity_type, bias)!r}")
    vocab, dim = sd0["transformer.wtes.0.weight"].shape
    n_layer = args.get("n_layer") or sum(1 for k in sd0 if k.endswith(".ln_1.weight"))
    n_head = n_head or args.get("n_head") or dim // 128
    mlp_in = "mlp.c_fc" if nonlinearity_type == "gelu" else "mlp.swiglu.w1"
    config = ModelArgs(block_size=sd0["transformer.wpe.weight"].shape[0], vocab_size=vocab, n_layer=n_layer,
                       n_head=n_head, dim=dim, speaker_emb_dim=sd0["speaker_cond_pos.weight"].shape[1],
                       intermediate_size=sd0[f"transformer.h.0.{mlp_in}.weight"].shape[0],
                       norm_eps=args.get("rmsnorm_eps") or 1e-5,
                       norm_type=norm_type, nonlinearity_type=nonlinearity_type, bias=bias)
    if quantisation_mode == "int8":   # measured: 0.84x the bf16 decode rate at batch 1 on an H100 (DESIGN.md section 8)
        warnings.warn("int8 quantisation is slower than bf16/fp16 for undebugged reasons! Please set optimisation_mode to "
                      "`None` or to `int4`.")
    if quantisation_mode is not None:   # utils:283-306: quantised at load from the bf16 checkpoint
        warnings.warn("quantisation will degrade the quality of the audio! Please set optimisation_mode to `None` for best quality.")
    model = Transformer.from_state_dict(sd0, config, device=device, quantisation_mode=quantisation_mode)
    tokenizer = None
    tok_info = checkpoint.get("meta", {}).get("tokenizer", {})
    if tok_info:
        from .tokenise import TrainedBPETokeniser
        tokenizer = TrainedBPETokeniser(**tok_info)
    smodel = None  # speaker encoder: out of scope row N3 (runs once per speaker, disk-cached by the reference)
    return model, tokenizer, smodel


# ---- fast_inference_utils.py:324-392 ---------------------------------------------------------------
def build_model(*, precision: torch.dtype = torch.bfloat16, checkpoint_path: Path = Path(""),
                spk_emb_ckpt_path: Path = Path(""), compile_prefill: bool = False, compile: bool = True,
                device: str = "cuda", quantisation_mode=None, max_utts: int = 1, kv_dtype: str = "bf16"):
    assert Path(checkpoint_path).is_file(), checkpoint_path
    print(f"Using device={device}")
    print("Loading model ...")
    t0 = time.time()
    model, tokenizer, smodel = _load_model(checkpoint_path, spk_emb_ckpt_path, device, precision, quantisation_mode)
    device_sync(device)
    print(f"Time to load model: {time.time() - t0:.02f} seconds")
    torch.manual_seed(1234)  # utils:347
    model_size = model.model_size_bytes()
    model.setup_spk_cond_mask()
    model.setup_caches(max_batch_size=2 * max_utts, max_seq_length=model.config.block_size, kv_dtype=kv_dtype)
    sample.default_model = model
    # `compile` / `compile_prefill` are accepted and ignored: kernels are ahead-of-time sm_90a code.
    return model, tokenizer, smodel, model_size


# ---- fast_inference_utils.py:395-445 ---------------------------------------------------------------
def main(*, model, tokenizer, model_size, prompt: str, guidance_scale, temperature, spk_emb, top_k=None, top_p=None,
         device: str = "cuda", voice: Optional[int] = None) -> list:
    encoded = encode_tokens(tokenizer, prompt, device="cpu")
    prompt_length = encoded.size(0)
    device_sync(device)
    t0 = time.perf_counter()
    y = generate(model, encoded, spk_emb, temperature=temperature, top_k=top_k, top_p=top_p,
                 guidance_scale=guidance_scale, end_of_text_token=getattr(tokenizer, "eot_token", None), voice=voice)
    device_sync(device)
    t = time.perf_counter() - t0
    tokens_generated = y.size(0) - prompt_length
    tokens_sec = tokens_generated / t
    print(f"Time for 1st stage LLM inference: {t:.02f} sec total, {tokens_sec:.02f} tokens/sec")
    print(f"Bandwidth achieved: {model_size * tokens_sec / 1e9:.02f} GB/s")
    print(f"Memory used: {torch.cuda.max_memory_reserved() / 1e9:.02f} GB\n")
    return y.tolist()
