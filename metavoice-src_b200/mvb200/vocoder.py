"""Host-side wrapper of the EnCodec-24 kHz decode path in libmvb200 (RVQ decode + SEANet decoder), the first half
of what ``EncodecDecoder.decode`` -> ``mbd.tokens_to_wav`` computes (fam/llm/decoders.py:66-102).  Loads the
``facebook/encodec_24khz`` checkpoint layout (transformers ``EncodecModel`` state dict, either weight-norm naming).
The multi-band diffusion stage is not implemented (unpinned: no source, no weights)."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional

import torch

from . import _lib
from ._engine import Engine, pack_arena_bytes, split_runs

RATIOS = (8, 5, 4, 2)


def _fold(sd, prefix):
    if prefix + ".parametrizations.weight.original0" in sd:
        g, v = sd[prefix + ".parametrizations.weight.original0"], sd[prefix + ".parametrizations.weight.original1"]
    elif prefix + ".weight_g" in sd:
        g, v = sd[prefix + ".weight_g"], sd[prefix + ".weight_v"]
    else:
        return sd[prefix + ".weight"].float()
    v = v.float()
    n = v.reshape(v.shape[0], -1).norm(dim=1).reshape(-1, *([1] * (v.dim() - 1)))
    return v * (g.float() / n)


class EncodecDecodeEngine(Engine):
    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda", max_frames: int = 2048, n_q: int = 8,
                 max_batch: int = 1, max_total_frames: Optional[int] = None):
        """``max_batch`` > 1 allocates the workspace of ``decode_batch`` / ``decode_latent_batch`` for up to ``max_batch``
        (<= 32) utterances and ``max_total_frames`` frames in all (default ``max_batch * max_frames``); larger requests
        are split into several launch sets."""
        sd = state_dict
        tensors = [sd[f"quantizer.layers.{q}.codebook.embed"].float() for q in range(n_q)]
        cw = lambda p: [_fold(sd, p + ".conv"), sd[p + ".conv.bias"].float()]
        tensors += cw("decoder.layers.0")
        for l in range(2):
            g = lambda k: sd[f"decoder.layers.1.lstm.{k}_l{l}"].float()
            tensors += [g("weight_ih"), g("weight_hh"), g("bias_ih") + g("bias_hh")]
        i = 3
        for _ in RATIOS:
            tensors += cw(f"decoder.layers.{i}") + cw(f"decoder.layers.{i + 1}.block.1") + \
                cw(f"decoder.layers.{i + 1}.block.3") + cw(f"decoder.layers.{i + 1}.shortcut")
            i += 3
        tensors += cw(f"decoder.layers.{i}")
        super().__init__(device, *pack_arena_bytes(tensors))
        cfg = _lib.VocConfig()
        cfg.n_q, cfg.hidden, cfg.n_filters, cfg.n_ratios = n_q, tensors[0].shape[1], 32, len(RATIOS)
        for k, r in enumerate(RATIOS):
            cfg.ratios[k] = r
        cfg.kernel, cfg.res_kernel, cfg.last_kernel, cfg.compress, cfg.max_frames = 7, 3, 7, 2, max_frames
        self.cfg = cfg
        self._create(self._lib.mvb_voc_create, self._lib.mvb_voc_destroy, cfg, self._lib.mvb_voc_workspace_bytes)
        self.max_batch, self.max_total_frames, self._bws = max_batch, max_total_frames or max_batch * max_frames, None
        if max_batch > 1:
            self._bws = self._batch_workspace_of(
                self._lib.mvb_voc_batch_workspace_bytes(C.byref(cfg), max_batch, self.max_total_frames))
        self.upsample = 1
        for r in RATIOS:
            self.upsample *= r
        # multiply-add accounting for the roofline in bench.py: (weight elements, output-rate multiplier) per layer
        terms, mult, k = [(tensors[n_q].numel(), 1)], 1, n_q + 2
        terms += [(tensors[k + 3 * l].numel() + tensors[k + 3 * l + 1].numel(), 1) for l in range(2)]
        k += 6
        for r in RATIOS:
            terms.append((tensors[k].numel(), mult))              # transposed conv: every input sample meets every tap
            mult *= r
            terms += [(tensors[k + 2 * j].numel(), mult) for j in (1, 2, 3)]
            k += 8
        terms.append((tensors[k].numel(), mult))
        self._flop_terms = terms

    def flops(self, n_frames: int) -> float:
        """fp32 FLOPs (2 x multiply-adds) of one SEANet decode of ``n_frames`` code frames."""
        return float(sum(2.0 * n * m * n_frames for n, m in self._flop_terms))

    @torch.no_grad()
    def decode_latent(self, codes: torch.Tensor) -> torch.Tensor:
        """codes int [n_q, T] -> [hidden, T] (the MBD condition, audiocraft ``get_condition``)."""
        c = codes.to(self.device, torch.int32).contiguous()
        out = torch.empty((self.cfg.hidden, c.shape[1]), dtype=torch.float32, device=self.device)
        _lib.check(self._lib.mvb_voc_decode_latent(self._h, c.data_ptr(), c.shape[1], out.data_ptr(), self._st()))
        return out

    @torch.no_grad()
    def decode(self, codes: torch.Tensor) -> torch.Tensor:
        """codes int [n_q, T] -> waveform fp32 [T * 320] at 24 kHz."""
        c = codes.to(self.device, torch.int32).contiguous()
        out = torch.empty(c.shape[1] * self.upsample, dtype=torch.float32, device=self.device)
        _lib.check(self._lib.mvb_voc_decode(self._h, c.data_ptr(), c.shape[1], out.data_ptr(), self._st()))
        return out

    def _batch(self, fn: str, codes: List[torch.Tensor], rows: int, per_frame: int) -> List[torch.Tensor]:
        cs = [c.to(self.device, torch.int32).contiguous() for c in codes]
        lens = [int(c.shape[1]) for c in cs]
        out = torch.empty(rows * sum(lens) * per_frame, dtype=torch.float32, device=self.device)
        pos = 0
        for g in split_runs(lens, self.max_batch, self.max_total_frames):
            flat = torch.cat([cs[i].reshape(-1) for i in g])
            T = (C.c_int32 * len(g))(*[lens[i] for i in g])
            _lib.check(getattr(self._lib, fn)(self._h, len(g), flat.data_ptr(), T, self._bws.data_ptr(), self.max_batch,
                                              self.max_total_frames, out[pos:].data_ptr(), self._st()))
            pos += rows * per_frame * sum(lens[i] for i in g)
        res, pos = [], 0
        for t in lens:
            n = rows * t * per_frame
            res.append(out[pos:pos + n].view(rows, t * per_frame) if rows > 1 else out[pos:pos + n])
            pos += n
        return res

    @torch.no_grad()
    def decode_batch(self, codes: List[torch.Tensor]) -> List[torch.Tensor]:
        """[codes int [n_q, T_i]] -> [waveform fp32 [T_i * 320]], each bit-identical to ``decode(codes[i])``.  One launch set
        per group of utterances that fits the batch workspace (``max_batch``); with ``max_batch=1`` a loop over ``decode``."""
        if not codes:
            return []
        if self._bws is None:
            return [self.decode(c) for c in codes]
        return self._batch("mvb_voc_decode_batch", codes, 1, self.upsample)

    @torch.no_grad()
    def decode_latent_batch(self, codes: List[torch.Tensor]) -> List[torch.Tensor]:
        """[codes int [n_q, T_i]] -> [latent [hidden, T_i]], each bit-identical to ``decode_latent(codes[i])``."""
        if not codes:
            return []
        if self._bws is None:
            return [self.decode_latent(c) for c in codes]
        return self._batch("mvb_voc_decode_latent_batch", codes, self.cfg.hidden, 1)


def _encoder_tensors(sd: Dict[str, torch.Tensor], n_q: int) -> List[torch.Tensor]:
    """The ``mvb_enc_create`` arena order (include/mvb200.h) from an ``EncodecModel`` state dict."""
    tensors = [sd[f"quantizer.layers.{q}.codebook.embed"].float() for q in range(n_q)]
    cw = lambda p: [_fold(sd, p + ".conv"), sd[p + ".conv.bias"].float()]   # noqa: E731
    tensors += cw("encoder.layers.0")
    i = 1
    for _ in RATIOS:                      # encoder.layers: resnet block i, ELU i + 1, strided conv i + 2
        tensors += cw(f"encoder.layers.{i}.block.1") + cw(f"encoder.layers.{i}.block.3") + \
            cw(f"encoder.layers.{i}.shortcut") + cw(f"encoder.layers.{i + 2}")
        i += 3
    for l in range(2):
        g = lambda k: sd[f"encoder.layers.{i}.lstm.{k}_l{l}"].float()      # noqa: E731
        tensors += [g("weight_ih"), g("weight_hh"), g("bias_ih") + g("bias_hh")]
    tensors += cw(f"encoder.layers.{i + 2}")
    return tensors


class EncodecEncodeEngine(Engine):
    """EnCodec-24 kHz encode path on the device (csrc/encoder.cu): waveform fp32 at 24 kHz -> SEANet encoder -> RVQ codes,
    i.e. ``EncodecModel.encode(wav, bandwidth)`` of the default 24 kHz config (normalize=False, one chunk) that
    ``EncodecDecoder.get_tokens`` (fam/llm/decoders.py:49-64) and the fine-tuning loader call.  Reads the same
    ``facebook/encodec_24khz`` state dict as ``EncodecDecodeEngine``; ``n_q = floor(bandwidth * 1000 / 750)`` (8 at 6 kbps).
    An input of L samples gives ``ceil(L / 320)`` frames; any L >= 1 up to ``320 * max_frames`` is accepted."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda", max_frames: int = 2048, n_q: int = 8,
                 max_batch: int = 1, max_total_frames: Optional[int] = None):
        """``max_batch`` > 1 allocates the workspace of ``encode_batch`` for up to ``max_batch`` (<= 32) utterances and
        ``max_total_frames`` frames in all (default ``max_batch * max_frames``); larger requests are split."""
        tensors = _encoder_tensors(state_dict, n_q)
        super().__init__(device, *pack_arena_bytes(tensors))
        cfg = _lib.EncConfig()
        cfg.n_q, cfg.hidden, cfg.n_filters, cfg.n_ratios = n_q, tensors[0].shape[1], 32, len(RATIOS)
        for k, r in enumerate(RATIOS):
            cfg.ratios[k] = r
        cfg.kernel, cfg.res_kernel, cfg.last_kernel, cfg.compress, cfg.max_frames = 7, 3, 7, 2, max_frames
        self.cfg = cfg
        self.hop = 1
        for r in RATIOS:
            self.hop *= r
        self._create(self._lib.mvb_enc_create, self._lib.mvb_enc_destroy, cfg, self._lib.mvb_enc_workspace_bytes)
        self.max_batch, self.max_total_frames, self._bws = max_batch, max_total_frames or max_batch * max_frames, None
        if max_batch > 1:
            self._bws = self._batch_workspace_of(
                self._lib.mvb_enc_batch_workspace_bytes(C.byref(cfg), max_batch, self.max_total_frames))
        # multiply-adds per output sample of every layer, with the layer's output rate in samples per frame
        terms, m, k = [(tensors[n_q].numel(), self.hop)], self.hop, n_q + 2
        for r in reversed(RATIOS):
            terms += [(tensors[k + 2 * j].numel(), m) for j in range(3)]       # resnet block k3, k1, shortcut
            m //= r
            terms.append((tensors[k + 6].numel(), m))                          # strided conv
            k += 8
        terms += [(tensors[k + 3 * l].numel() + tensors[k + 3 * l + 1].numel(), 1) for l in range(2)]
        terms.append((tensors[k + 6].numel(), 1))
        self._flop_terms = terms
        self._rvq_macs = n_q * tensors[0].numel()                              # every codebook row meets every frame

    def frames(self, n_samples: int) -> int:
        return -(-int(n_samples) // self.hop)

    def flops(self, n_samples: int) -> float:
        """fp32 FLOPs (2 x multiply-adds) of one encode of ``n_samples`` samples, counted from shapes: the conv stack,
        the LSTM and the codebook search."""
        F = self.frames(n_samples)
        return float(sum(2.0 * n * m * F for n, m in self._flop_terms) + 2.0 * self._rvq_macs * F)

    def _run(self, wav: torch.Tensor, emb: bool):
        x = wav.to(self.device, torch.float32).contiguous().reshape(-1)
        F = self.frames(x.numel())
        codes = torch.empty((self.cfg.n_q, F), dtype=torch.int32, device=self.device)
        e = torch.empty((self.cfg.hidden, F), dtype=torch.float32, device=self.device) if emb else None
        _lib.check(self._lib.mvb_enc_encode(self._h, x.data_ptr(), x.numel(), codes.data_ptr(),
                                            e.data_ptr() if emb else None, self._st()))
        return codes, e

    @torch.no_grad()
    def encode(self, wav: torch.Tensor) -> torch.Tensor:
        """waveform fp32 [L] at 24 kHz -> codes int32 [n_q, ceil(L / 320)] (the layout ``EncodecDecodeEngine.decode`` takes)."""
        return self._run(wav, False)[0]

    @torch.no_grad()
    def embed(self, wav: torch.Tensor) -> torch.Tensor:
        """waveform fp32 [L] -> the encoder output before quantisation, fp32 [128, ceil(L / 320)]."""
        return self._run(wav, True)[1]

    @torch.no_grad()
    def encode_mono(self, wav: torch.Tensor) -> torch.Tensor:
        """[channels, L] -> codes of the channel mean: ``_extract_encodec_tokens`` (fam/llm/loaders/training_data.py:98-112)."""
        return self.encode(wav.float().mean(dim=0) if wav.dim() == 2 else wav)

    @torch.no_grad()
    def encode_batch(self, wavs: List[torch.Tensor]) -> List[torch.Tensor]:
        """[waveform fp32 [L_i]] -> [codes int32 [n_q, ceil(L_i / 320)]], each bit-identical to ``encode(wavs[i])``.  One
        launch set per group of utterances that fits the batch workspace (``max_batch``); with ``max_batch=1`` a loop over
        ``encode``."""
        if not wavs:
            return []
        if self._bws is None:
            return [self.encode(w) for w in wavs]
        xs = [w.to(self.device, torch.float32).contiguous().reshape(-1) for w in wavs]
        lens = [int(x.numel()) for x in xs]
        n_q = self.cfg.n_q
        out = torch.empty(n_q * sum(self.frames(n) for n in lens), dtype=torch.int32, device=self.device)
        pos = 0
        for g in split_runs([self.frames(n) for n in lens], self.max_batch, self.max_total_frames):
            flat = torch.cat([xs[i] for i in g])
            L = (C.c_int32 * len(g))(*[lens[i] for i in g])
            _lib.check(self._lib.mvb_enc_encode_batch(self._h, len(g), flat.data_ptr(), L, self._bws.data_ptr(), self.max_batch,
                                                      self.max_total_frames, out[pos:].data_ptr(), None, self._st()))
            pos += n_q * sum(self.frames(lens[i]) for i in g)
        res, pos = [], 0
        for n in lens:
            F = self.frames(n)
            res.append(out[pos:pos + n_q * F].view(n_q, F))
            pos += n_q * F
        return res


def get_tokens(engine: EncodecEncodeEngine, audio_path: str) -> List[List[int]]:
    """``EncodecDecoder.get_tokens`` (fam/llm/decoders.py:49-64): audio file -> codes [n_q][F] as nested lists.

    RIFF/WAVE only (PCM16 / PCM32 / float32); mp3 and flac raise ``NotImplementedError`` as the speaker-reference reader
    does.  The reference passes the channels as the batch and returns the first one (``tokens[0][0]``), so a
    multi-channel file gives the codes of its first channel.  A file not at 24 kHz is resampled on the host with the
    polyphase resampler of the speaker encoder; the reference uses ``julius.resample_frac``, so that path is not pinned.
    The fine-tuning loader's variant (``_extract_encodec_tokens``, training_data.py:98-112) encodes the channel mean
    instead: ``engine.encode_mono``."""
    from .speaker_encoder import read_wav, resample
    x, sr = read_wav(audio_path, mono=False)
    x = resample(x[0], sr, 24000)
    return engine.encode(torch.from_numpy(x)).tolist()
