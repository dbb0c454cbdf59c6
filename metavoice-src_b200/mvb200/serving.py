"""Request-level batching for the stage-1 engine (SURVEY.md row N4).

The reference serves one request at a time (``serving.py:59-109`` calls the blocking ``TTS.synthesise`` from an
``async`` handler) and truncates text at 220 characters (``fam/llm/inference.py:535-541``: "Long form synthesis coming
soon").  Here utterances are admitted into free KV-cache slots of the persistent decode kernel between bursts
(continuous batching), and long text is cut into <= 220-character chunks that are synthesised as one batch.

  chunk_text(text)            sentence-aware splitter, every chunk <= max_chars (the reference's MAX_CHARS)
  ContinuousBatcher(model)    submit() requests at any time, step() = admit + one decode burst + harvest

Every utterance is decoded exactly as if it ran alone (per-row positions, per-utterance sampler state, no
cross-utterance math: fam/llm/mixins/causal.py:389-424), so batching changes throughput, not results.
"""
from __future__ import annotations

import ctypes as C
import re
from collections import deque
from dataclasses import dataclass, field
from typing import Deque, Dict, List, Optional

import numpy as np
import torch

from . import _lib
from .fast_inference_utils import _sampling_struct, split_guidance

MAX_CHARS = 220  # fam/llm/inference.py:537


def chunk_text(text: str, max_chars: int = MAX_CHARS) -> List[str]:
    """Split `text` into chunks of at most `max_chars` characters: sentence boundaries first (.!?;:), then commas,
    then spaces, and only as a last resort inside a word.  Concatenating the chunks with single spaces gives the
    whitespace-normalised input back."""
    text = re.sub(r"\s+", " ", text).strip()
    if not text:
        return []

    def split(piece: str, seps: List[str]) -> List[str]:
        if len(piece) <= max_chars:
            return [piece]
        if not seps:
            return [piece[i:i + max_chars] for i in range(0, len(piece), max_chars)]
        parts = [p.strip() for p in re.split(seps[0], piece) if p.strip()]
        out: List[str] = []
        for p in parts:
            out.extend(split(p, seps[1:]))
        return out

    atoms = split(text, [r"(?<=[.!?])\s+", r"(?<=[;:])\s+", r"(?<=,)\s+", r"\s+"])
    chunks: List[str] = []
    cur = ""
    for a in atoms:                       # greedy re-packing: as few chunks as possible
        if not cur:
            cur = a
        elif len(cur) + 1 + len(a) <= max_chars:
            cur = cur + " " + a
        else:
            chunks.append(cur)
            cur = a
    if cur:
        chunks.append(cur)
    return chunks


def seeded_noise(model, prompt_len: int, seed: int, max_new_tokens: Optional[int] = None) -> torch.Tensor:
    """Exp(1) draws [max_new, vocab] on the model's device from torch's Philox generator seeded with ``seed``, for
    ``ContinuousBatcher.submit(..., max_new_tokens=max_new, noise=...)``.  A request's tokens then depend on its seed
    alone, not on the slot it is admitted to (the engine's own on-device stream is keyed on the slot).  Returns the
    draws; their first dimension is the ``max_new`` to submit with."""
    block = model.config.block_size
    max_new = block - int(prompt_len) if max_new_tokens is None else int(max_new_tokens)
    max_new = max(1, min(max_new, model._cfg.max_new))
    g = torch.Generator(device=model.device).manual_seed(int(seed))
    return torch.empty((max_new, model.config.vocab_size), dtype=torch.float32, device=model.device).exponential_(1, generator=g)


@dataclass
class _Request:
    rid: int
    prompt: np.ndarray
    spk: np.ndarray
    sampling: dict
    max_new: int
    seed: int
    noise: Optional[torch.Tensor] = None
    prompt_guidance: Optional[float] = None      # p > 1 of guidance_scale = (s, p): the request needs a companion slot
    end_of_text: int = 0
    voice: int = 0                               # voice id of the stage-1 engine (Transformer.add_voice); 0 = the base
    slot: int = -1
    companion: int = -1
    tokens: Optional[torch.Tensor] = None


@dataclass
class ContinuousBatcher:
    """Admit-between-bursts scheduler over one ``mvb200.fast_model.Transformer`` (``setup_caches(2 * slots, ...)``).
    A prompt-guided request (``guidance_scale=(s, p)``, p > 1) occupies two slots, its own and a companion, from
    admission until it finishes; requests are admitted in submission order."""
    model: object
    burst: int = 32
    _next: int = 0
    _pending: Deque[_Request] = field(default_factory=deque)
    _active: Dict[int, _Request] = field(default_factory=dict)   # slot -> request
    _done: Dict[int, torch.Tensor] = field(default_factory=dict)
    _companions: Dict[int, int] = field(default_factory=dict)   # companion slot -> its request's slot

    def __post_init__(self):
        self.slots = self.model.max_utts
        lib, h, st = self.model._lib, self.model.handle, self.model._stream()
        for s in range(self.slots):                     # every slot starts parked
            _lib.check(lib.mvb_s1_release(h, s, st))

    # ---- client side -----------------------------------------------------------------------------
    def submit(self, prompt: torch.Tensor, spk_emb: torch.Tensor, *, max_new_tokens: Optional[int] = None,
               guidance_scale=3.0, temperature=1.0, top_p=0.95, top_k=None, end_of_audio_token: int = 2048,
               seed: Optional[int] = None, noise: Optional[torch.Tensor] = None,
               end_of_text_token: Optional[int] = None, voice: Optional[int] = None) -> int:
        """``guidance_scale``: a float, or the reference's ``(s, p)``; p > 1 needs ``end_of_text_token`` and two free
        slots at admission, and ``(s, 1.0)`` is ``s``.  ``voice``: a voice id of the model (None: the base checkpoint);
        requests of different voices share decode bursts."""
        vid = 0 if voice is None else self.model.voice_id(voice)
        s_g, p_g = split_guidance(guidance_scale, end_of_text_token)
        if p_g is not None and self.slots < 2:
            raise ValueError(f"a prompt-guided request needs 2 slots; setup_caches set up {self.slots}")
        T = int(prompt.numel())
        block = self.model.config.block_size
        max_new = block - T if max_new_tokens is None else int(max_new_tokens)
        if min(T + max_new, block) - T <= 0:
            raise ValueError("Prompt is too long to generate more tokens")      # utils:203-204
        max_new = min(max_new, self.model._cfg.max_new)
        if seed is None:
            seed = int(torch.randint(0, 2**62, (1,)).item())
        rid = self._next
        self._next += 1
        self._pending.append(_Request(rid, prompt.detach().cpu().numpy().astype(np.int32).reshape(-1),
                                      np.ascontiguousarray(spk_emb.detach().to("cpu", torch.float32).numpy().reshape(-1)),
                                      dict(guidance_scale=s_g, temperature=temperature, top_p=top_p, top_k=top_k,
                                           end_of_audio_token=end_of_audio_token), max_new, seed, noise, p_g,
                                      int(end_of_text_token) if p_g is not None else 0, vid))
        return rid

    @property
    def idle(self) -> bool:
        return not self._pending and not self._active

    # ---- engine side -----------------------------------------------------------------------------
    def _admit(self):
        lib, h, st = self.model._lib, self.model.handle, self.model._stream()
        free = [s for s in range(self.slots) if s not in self._active and s not in self._companions]
        while self._pending and len(free) >= (1 if self._pending[0].prompt_guidance is None else 2):
            r = self._pending.popleft()
            r.slot = free.pop(0)
            sp = _sampling_struct(seed=r.seed, **r.sampling)
            d_noise = None
            if r.noise is not None:
                r.noise = r.noise.to(self.model.device, torch.float32).contiguous()     # keep alive while the slot is active
                assert r.noise.shape == (r.max_new, self.model.config.vocab_size)
                d_noise = C.c_void_p(r.noise.data_ptr())
            if getattr(self.model, "n_voices", 1) > 1:
                self.model.set_voice(r.slot, r.voice)
            if r.prompt_guidance is None:
                _lib.check(lib.mvb_s1_admit(h, r.slot, r.prompt.ctypes.data_as(C.c_void_p), int(r.prompt.size),
                                            r.spk.ctypes.data_as(C.c_void_p), C.byref(sp), r.max_new, d_noise, st))
            else:
                r.companion = free.pop(0)
                _lib.check(lib.mvb_s1_admit_guided(h, r.slot, r.companion, r.prompt.ctypes.data_as(C.c_void_p),
                                                   int(r.prompt.size), r.spk.ctypes.data_as(C.c_void_p), C.byref(sp),
                                                   r.prompt_guidance, r.end_of_text, r.max_new, d_noise, st))
                self._companions[r.companion] = r.slot
            self._active[r.slot] = r

    def step(self) -> List[int]:
        """Admit waiting requests into free slots, run one decode burst for all slots, harvest finished utterances.
        Returns the ids of the requests that finished in this step."""
        self._admit()
        if not self._active:
            return []
        lib, h, st = self.model._lib, self.model.handle, self.model._stream()
        n_slots = max([*self._active, *self._companions]) + 1
        _lib.check(lib.mvb_s1_decode(h, n_slots, self.burst, st))
        done = np.zeros(n_slots, dtype=np.int32)
        n_gen = np.zeros(n_slots, dtype=np.int32)
        _lib.check(lib.mvb_s1_poll(h, n_slots, done.ctypes.data_as(C.c_void_p), n_gen.ctypes.data_as(C.c_void_p), st))
        finished = []
        for s in list(self._active):
            if done[s]:
                r = self._active.pop(s)
                self._companions.pop(r.companion, None)     # the engine parked it with its request
                buf = np.zeros(int(n_gen[s]), dtype=np.int32)
                n, d = C.c_int32(0), C.c_int32(0)
                _lib.check(lib.mvb_s1_fetch(h, s, buf.ctypes.data_as(C.c_void_p), int(buf.size), C.byref(n), C.byref(d), st))
                self._done[r.rid] = torch.from_numpy(buf[: int(n.value)].copy())
                finished.append(r.rid)
        return finished

    def run_until_done(self) -> Dict[int, torch.Tensor]:
        while not self.idle:
            self.step()
        out, self._done = self._done, {}
        return out

    def result(self, rid: int) -> Optional[torch.Tensor]:
        return self._done.get(rid)
