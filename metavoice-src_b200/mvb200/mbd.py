"""Host-side wrapper of the multi-band-diffusion vocoder in libmvb200 (SURVEY.md row a17): the part of
``mbd.tokens_to_wav`` (fam/llm/decoders.py:84-85, audiocraft 1.2.0 ``MultiBandDiffusion``) that follows the codec decode.
PARITY UNPINNED -- see oracle/mbd_port.py: the configuration is a parameter (``MBDSettings``), the checkpoint layout
follows audiocraft's module names (``models`` = one ``DiffusionUnet`` state dict per band model, ``proc`` = the
``MultiBandProcessor`` statistics)."""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional

import torch

from . import _lib
from ._engine import Engine, pack_arena_bytes


@dataclass
class UnetSettings:
    chin: int = 1
    hidden: int = 48
    depth: int = 4
    growth: float = 4.0
    kernel: int = 8
    stride: int = 4
    res_blocks: int = 1
    norm_groups: int = 4
    emb_all_layers: bool = True
    codec_dim: int = 128
    num_steps: int = 1000
    max_channels: int = 10_000

    def channels(self) -> List[int]:
        ch, h = [], self.hidden
        for _ in range(self.depth):
            ch.append(h)
            h = min(int(h * self.growth), self.max_channels)
        return ch


@dataclass
class ScheduleSettings:
    beta_t0: float = 1e-5
    beta_t1: float = 2.9e-2
    beta_exp: float = 7.5
    num_steps: int = 1000
    clip: float = 5.0
    rescale: float = 1.0
    noise_scale: float = 1.0


@dataclass
class MBDSettings:
    sample_rate: int = 24000
    n_models: int = 4
    unet: UnetSettings = field(default_factory=UnetSettings)
    schedule: ScheduleSettings = field(default_factory=ScheduleSettings)
    proc_bands: int = 8
    power_std: float = 1.0
    eq_bands: int = 32
    step_list: Optional[List[int]] = None

    def steps(self) -> List[int]:
        return self.step_list if self.step_list is not None else list(range(self.schedule.num_steps))[::-50] + [0]


def _lowpass_bank(n_bands: int, sample_rate: int, zeros: float = 8.0) -> torch.Tensor:
    """julius.SplitBands(sample_rate, n_bands): low-pass filters at the mel-spaced band edges (windowed sinc, Hann, 8 zero
    crossings of the lowest cutoff on each side), normalised to unit DC gain.  [n_bands - 1, taps] fp32."""
    mel = lambda f: 2595 * math.log10(1 + f / 700)
    inv = lambda m: 700 * (10 ** (m / 2595) - 1)
    top = mel(sample_rate / 2)
    cuts = [inv(top * i / n_bands) / sample_rate for i in range(1, n_bands)]
    half = int(zeros / min(cuts) / 2)
    t = torch.arange(-half, half + 1, dtype=torch.float64)
    win = torch.hann_window(2 * half + 1, periodic=False, dtype=torch.float64)
    rows = []
    for c in cuts:
        arg = 2 * c * math.pi * t
        f = 2 * c * win * torch.where(arg == 0, torch.ones_like(arg), torch.sin(arg) / arg)
        rows.append(f / f.sum())
    return torch.stack(rows).float()


def _schedule_table(s: ScheduleSettings, steps: List[int]) -> torch.Tensor:
    """NoiseSchedule.generate_subsampled folded into one row per model call: previous = (current - a * estimate) * b
    + sigma * noise; columns {a, b, sigma, step}."""
    betas = torch.linspace(s.beta_t0 ** (1 / s.beta_exp), s.beta_t1 ** (1 / s.beta_exp), s.num_steps, dtype=torch.float32) ** s.beta_exp
    abar = (1 - betas).cumprod(dim=0)
    sub = abar[list(reversed(steps))]
    beta_sub = 1 - torch.cat([sub[:1], sub[1:] / sub[:-1]])
    cur_abar = abar[s.num_steps - 1]
    rows = []
    for i, step in enumerate(steps[:-1]):
        alpha = 1 - beta_sub[-1 - i]
        last = step == steps[-2]
        nxt = torch.tensor(1.0) if last else abar[steps[i + 1]]
        sigma2 = torch.tensor(0.0) if last else (1 - nxt) / (1 - cur_abar) * (1 - alpha)
        rows.append([float((1 - alpha) / (1 - cur_abar).sqrt()), float(1 / alpha.sqrt()), float(sigma2.clamp(min=0).sqrt()), float(step)])
        cur_abar = nxt
    return torch.tensor(rows, dtype=torch.float32)


_RES = ["norm1.weight", "norm1.bias", "conv1.weight", "conv1.bias", "norm2.weight", "norm2.bias", "conv2.weight", "conv2.bias"]


class MultiBandDiffusionEngine(Engine):
    def __init__(self, checkpoint: dict, settings: MBDSettings, device="cuda", max_seconds: float = 12.0,
                 tensor_cores: bool = True, band_streams: bool = True):
        """``tensor_cores=False`` (test hook): every convolution on the fp32 CUDA-core kernels; ``band_streams=False``: the
        band models back to back on the caller's stream instead of one stream each."""
        self.s = settings
        u = settings.unet
        tensors = []
        for sd, pr in zip(checkpoint["models"], checkpoint["proc"]):
            g = lambda k: sd[k].detach().float().contiguous()
            for i in range(u.depth):
                p = f"encoders.{i}."
                tensors += [g(p + "conv.weight"), g(p + "norm.weight"), g(p + "norm.bias")]
                for j in range(u.res_blocks):
                    tensors += [g(f"{p}res_blocks.{j}.{k}") for k in _RES]
                if i == 0:
                    tensors.append(g("embedding.weight"))
                elif u.emb_all_layers:
                    tensors.append(g(f"embeddings.{i - 1}.weight"))
                else:
                    tensors.append(torch.zeros(u.num_steps, u.channels()[i]))
            tensors += [g("conv_codec.weight"), g("conv_codec.bias")]
            for i in range(u.depth):
                p = f"decoders.{i}."
                for j in range(u.res_blocks):
                    tensors += [g(f"{p}res_blocks.{j}.{k}") for k in _RES]
                tensors += [g(p + "norm.weight"), g(p + "norm.bias"), g(p + "convtr.weight")]
            tensors += [((pr["std"] / pr["target_std"]) ** settings.power_std).float(), pr["mean"].float()]
        bank_p = _lowpass_bank(settings.proc_bands, settings.sample_rate)
        bank_e = _lowpass_bank(settings.eq_bands, settings.sample_rate)
        sched = _schedule_table(settings.schedule, settings.steps())
        tensors += [bank_p, bank_e, sched]
        super().__init__(device, *pack_arena_bytes(tensors))
        cfg = _lib.MbdConfig(settings.n_models, u.chin, u.hidden, u.depth, u.res_blocks, u.norm_groups, u.kernel, u.stride,
                             float(u.growth), int(u.emb_all_layers), u.codec_dim, u.num_steps, sched.shape[0],
                             float(settings.schedule.noise_scale), float(settings.schedule.clip), settings.proc_bands,
                             bank_p.shape[1], settings.eq_bands, bank_e.shape[1], int(max_seconds * settings.sample_rate),
                             (0 if tensor_cores else _lib.MVB_MBD_CUDA_CORES) | (0 if band_streams else _lib.MVB_MBD_ONE_STREAM))
        self.cfg = cfg
        self._create(self._lib.mvb_mbd_create, self._lib.mvb_mbd_destroy, cfg, self._lib.mvb_mbd_workspace_bytes)
        self.n_calls = sched.shape[0]

    def flops(self, n_samples: int, n_frames: int) -> float:
        """FLOPs (2 x multiply-adds) of the convolutions of one ``tokens_to_wav`` call: every band model x every sampler call."""
        u, ch = self.s.unet, self.s.unet.channels()
        t, cin, per = n_samples, u.chin, 0.0
        for c in ch:
            t = -(-t // u.stride)
            per += 2.0 * u.kernel * cin * c * t                       # strided encoder conv
            per += 2 * u.res_blocks * 2 * (2.0 * 3 * c * c * t)       # encoder + decoder ResBlocks (two k = 3 convs each)
            per += 2.0 * u.kernel * c * cin * t                       # transposed conv back to the level above
            cin = c
        per += 2.0 * u.codec_dim * ch[-1] * n_frames
        return per * self.s.n_models * (len(self.s.steps()) - 1)

    def check_shape(self, n_frames: int, n_samples: int) -> None:
        """The library's shape checks of ``tokens_to_wav``, as ValueError before anything reaches the device: n_samples
        within 16 x stride .. the workspace capacity, and at most the frames the workspace's condition buffer holds
        (capacity / 320 + 8), and at most twice the UNet bottleneck length."""
        u, cap = self.s.unet, self.cfg.max_samples
        if not 16 * u.stride <= n_samples <= cap:
            raise ValueError(f"mbd: n_samples {n_samples} out of range ({16 * u.stride} .. {cap})")
        tl = n_samples
        for _ in range(u.depth):
            tl = -(-tl // u.stride)
        limit = min(cap // 320 + 8, 2 * tl)
        if not 1 <= n_frames <= limit:
            raise ValueError(f"mbd: n_frames {n_frames} out of range (1 .. {limit} for {n_samples} samples)")

    @torch.no_grad()
    def tokens_to_wav(self, cond: torch.Tensor, wav_encodec: torch.Tensor, noise: Optional[torch.Tensor] = None, seed: int = 0) -> torch.Tensor:
        """cond fp32 [codec_dim, T_frames] (``decode_latent``), wav_encodec fp32 [T] (codec decode) -> refined wav fp32 [T].
        ``noise`` [n_models, n_calls, T]: the standard-normal draws of the sampler (parity tests); else on-device Philox."""
        self.check_shape(cond.shape[1], wav_encodec.numel())
        c = cond.to(self.device, torch.float32).contiguous()
        w = wav_encodec.to(self.device, torch.float32).reshape(-1).contiguous()
        nz = None
        if noise is not None:
            nz = noise.to(self.device, torch.float32).contiguous()
            assert nz.shape == (self.s.n_models, self.n_calls, w.numel()), nz.shape
        out = torch.empty_like(w)
        _lib.check(self._lib.mvb_mbd_tokens_to_wav(self._h, c.data_ptr(), c.shape[1], w.data_ptr(), w.numel(),
                                                   None if nz is None else nz.data_ptr(), int(seed) & (2**64 - 1), out.data_ptr(),
                                                   self._st()))
        return out
