"""Host-side wrapper of the EnCodec-24 kHz decode path in libmvb200 (RVQ decode + SEANet decoder), the first half
of what ``EncodecDecoder.decode`` -> ``mbd.tokens_to_wav`` computes (fam/llm/decoders.py:66-102).  Loads the
``facebook/encodec_24khz`` checkpoint layout (transformers ``EncodecModel`` state dict, either weight-norm naming).
The multi-band diffusion stage is not implemented (unpinned: no source, no weights)."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional

import torch

from . import _lib

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


class EncodecDecodeEngine:
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
        offs, total = [], 0
        for t in tensors:
            offs.append(total)
            total = (total + t.numel() * 4 + 255) // 256 * 256
        arena = torch.zeros(total, dtype=torch.uint8)
        for t, o in zip(tensors, offs):
            arena[o:o + t.numel() * 4] = t.contiguous().reshape(-1).view(torch.uint8)
        self.device = torch.device(device)
        self._arena = arena.to(self.device)
        cfg = _lib.VocConfig()
        cfg.n_q, cfg.hidden, cfg.n_filters, cfg.n_ratios = n_q, tensors[0].shape[1], 32, len(RATIOS)
        for k, r in enumerate(RATIOS):
            cfg.ratios[k] = r
        cfg.kernel, cfg.res_kernel, cfg.last_kernel, cfg.compress, cfg.max_frames = 7, 3, 7, 2, max_frames
        self.cfg, self._lib = cfg, _lib.load()
        wsb = self._lib.mvb_voc_workspace_bytes(C.byref(cfg))
        if wsb == 0:
            _lib.check(_lib.MVB_ERR_UNSUPPORTED)
        self._ws = torch.zeros(wsb, dtype=torch.uint8, device=self.device)
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.mvb_voc_create(C.byref(cfg), self._arena.data_ptr(), self._arena.numel(),
                                                (C.c_uint64 * len(offs))(*offs), self._ws.data_ptr(), C.byref(h)))
        self._h = h
        self.max_batch, self.max_total_frames, self._bws = max_batch, max_total_frames or max_batch * max_frames, None
        if max_batch > 1:
            bwsb = self._lib.mvb_voc_batch_workspace_bytes(C.byref(cfg), max_batch, self.max_total_frames)
            if bwsb == 0:
                _lib.check(_lib.MVB_ERR_ARG)
            self._bws = torch.zeros(bwsb, dtype=torch.uint8, device=self.device)
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

    def close(self):
        if getattr(self, "_h", None) is not None:
            self._lib.mvb_voc_destroy(self._h)
            self._h = None

    __del__ = close

    def _st(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

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

    def _groups(self, lens: List[int]) -> List[range]:
        """Consecutive runs of utterances that fit the batch workspace (<= max_batch of them, <= max_total_frames)."""
        groups, s0, tot = [], 0, 0
        for i, t in enumerate(lens):
            if i > s0 and (i - s0 == self.max_batch or tot + t > self.max_total_frames):
                groups.append(range(s0, i))
                s0, tot = i, 0
            tot += t
        groups.append(range(s0, len(lens)))
        return groups

    def _batch(self, fn: str, codes: List[torch.Tensor], rows: int, per_frame: int) -> List[torch.Tensor]:
        cs = [c.to(self.device, torch.int32).contiguous() for c in codes]
        lens = [int(c.shape[1]) for c in cs]
        out = torch.empty(rows * sum(lens) * per_frame, dtype=torch.float32, device=self.device)
        pos = 0
        for g in self._groups(lens):
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
