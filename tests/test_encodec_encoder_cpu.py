"""CPU: a float64 restatement of the EnCodec-24 kHz encode path (`EncodecEncodeOracle`, the reference the GPU tests of
csrc/encoder.cu measure against) pinned to transformers.EncodecModel run in float64 on the synthetic checkpoint.

  * SEANet encoder                                          EncodecEncoder            (modeling_encodec.py:285-313)
  * causal Conv1d, reflect padding of k - stride on the left and ceil(L / s) s - L on the right, with _pad1d's
    zero extension of a tensor no longer than the padding  EncodecConv1d             (:126-176)
  * residual block, 2-layer LSTM with skip                  EncodecResnetBlock / EncodecLSTM
  * RVQ encode: argmin_j |e_j|^2 - 2 x.e_j, first index on ties, residual -= e_idx
                                                            EncodecResidualVectorQuantizer.encode (:424-438)

Embeddings must agree to 1e-12 (relative, normwise) and codes exactly, at L = 1 .. 24000 samples (every length class
of the zero-extension rule at the short end, the frame seams at 320 and 640) and n_q = 2, 8 and 32 (1.5, 6 and 24 kbps).
"""
from __future__ import annotations

from typing import Dict, List

import pytest
import torch
import torch.nn.functional as F

from mvb200 import synth

RATIOS = (8, 5, 4, 2)
LENGTHS = (1, 2, 7, 8, 15, 16, 39, 40, 41, 319, 320, 321, 641, 24000)
BANDWIDTH = {2: 1.5, 8: 6.0, 32: 24.0}


def pad1d_reflect(x: torch.Tensor, left: int, right: int) -> torch.Tensor:
    """EncodecConv1d._pad1d in reflect mode: a tensor no longer than the larger padding is first zero-extended to one
    sample more than it, reflected, and trimmed by the extension again."""
    length = x.shape[-1]
    max_pad = max(left, right)
    extra = 0
    if length <= max_pad:
        extra = max_pad - length + 1
        x = F.pad(x, (0, extra))
    p = F.pad(x, (left, right), mode="reflect")
    return p[..., : p.shape[-1] - extra]


def enc_conv1d(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, stride: int = 1) -> torch.Tensor:
    """EncodecConv1d.forward, causal: padding_total = k - stride on the left, ceil(L / stride) stride - L on the right."""
    k, L = w.shape[-1], x.shape[-1]
    extra = -(-L // stride) * stride - L
    return F.conv1d(pad1d_reflect(x, k - stride, extra), w, b, stride=stride)


def fold_weight_norm(sd: Dict[str, torch.Tensor], prefix: str, dtype) -> torch.Tensor:
    """w = g v / ||v|| (norm over every dim but 0) evaluated in `dtype`, as torch's weight-norm parametrisation evaluates
    it for a model cast to that dtype; either weight-norm naming."""
    if prefix + ".parametrizations.weight.original0" in sd:
        g, v = sd[prefix + ".parametrizations.weight.original0"], sd[prefix + ".parametrizations.weight.original1"]
    elif prefix + ".weight_g" in sd:
        g, v = sd[prefix + ".weight_g"], sd[prefix + ".weight_v"]
    else:
        return sd[prefix + ".weight"].to(dtype)
    g, v = g.to(dtype), v.to(dtype)
    return v * (g / v.reshape(v.shape[0], -1).norm(dim=1).reshape(-1, *([1] * (v.dim() - 1))))


class EncodecEncodeOracle:
    """Float64 (by default) EncodecModel.encode of the default 24 kHz config from its state dict."""

    def __init__(self, sd: Dict[str, torch.Tensor], n_q: int = 8, dtype=torch.float64, device="cpu"):
        d = lambda t: t.to(device, dtype)     # noqa: E731
        cw = lambda p: (d(fold_weight_norm(sd, p + ".conv", dtype)), d(sd[p + ".conv.bias"]))   # noqa: E731
        self.n_q = n_q
        self.codebooks = [d(sd[f"quantizer.layers.{q}.codebook.embed"]) for q in range(n_q)]
        self.conv_in = cw("encoder.layers.0")
        self.levels = []
        i = 1
        for r in reversed(RATIOS):
            p = f"encoder.layers.{i}"
            self.levels.append(dict(r=r, c1=cw(p + ".block.1"), c2=cw(p + ".block.3"), sc=cw(p + ".shortcut"),
                                    down=cw(f"encoder.layers.{i + 2}")))
            i += 3
        self.lstm = [{k: d(sd[f"encoder.layers.{i}.lstm.{k}_l{l}"]) for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")}
                     for l in range(2)]
        self.conv_out = cw(f"encoder.layers.{i + 2}")

    def _lstm(self, x: torch.Tensor) -> torch.Tensor:       # x [B, C, T]
        seq = x.permute(2, 0, 1)
        out = seq
        for L in self.lstm:
            H = L["weight_hh"].shape[1]
            h = seq.new_zeros(seq.shape[1], H)
            c = seq.new_zeros(seq.shape[1], H)
            ys = []
            for t in range(out.shape[0]):
                g = out[t] @ L["weight_ih"].t() + L["bias_ih"] + h @ L["weight_hh"].t() + L["bias_hh"]
                i, f, gg, o = g.chunk(4, dim=-1)
                c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
                h = torch.sigmoid(o) * torch.tanh(c)
                ys.append(h)
            out = torch.stack(ys)
        return (out + seq).permute(1, 2, 0)

    @torch.no_grad()
    def embed(self, wav: torch.Tensor, taps: dict = None) -> torch.Tensor:
        """wav [B, 1, L] -> embeddings [B, 128, ceil(L / 320)]."""
        x = enc_conv1d(wav, *self.conv_in)
        for lv in self.levels:
            h = enc_conv1d(F.elu(x), *lv["c1"])
            h = enc_conv1d(F.elu(h), *lv["c2"])
            x = enc_conv1d(x, *lv["sc"]) + h
            x = enc_conv1d(F.elu(x), *lv["down"], stride=lv["r"])
            if taps is not None:
                taps[f"down{lv['r']}"] = x.clone()
        x = self._lstm(x)
        return enc_conv1d(F.elu(x), *self.conv_out)

    @torch.no_grad()
    def quantize(self, emb: torch.Tensor, n_q: int = None) -> List[torch.Tensor]:
        """emb [128, F] -> [(codes [F], sorted scores [F, 2]) per codebook]: the chosen index (first on ties) and the best
        two values of |e_j|^2 - 2 r.e_j, in the oracle's dtype, with r the oracle's own residual."""
        r = emb.t()
        out = []
        for cb in self.codebooks[: n_q or self.n_q]:
            s = (cb * cb).sum(1)[None] - 2 * r @ cb.t()
            idx = torch.argmin(s, dim=1)            # first minimal index
            out.append((idx, torch.topk(s, 2, dim=1, largest=False).values))
            r = r - cb[idx]
        return out

    def encode(self, wav: torch.Tensor, n_q: int = None) -> torch.Tensor:
        """wav [L] -> codes [n_q, ceil(L / 320)]."""
        emb = self.embed(wav.reshape(1, 1, -1))[0]
        return torch.stack([c for c, _ in self.quantize(emb, n_q)])


@pytest.fixture(scope="module")
def model_and_oracle():
    m, sd = synth.encodec_model_and_state_dict(seed=0)
    return m.double(), EncodecEncodeOracle(sd, n_q=32)


def _wav(L: int) -> torch.Tensor:
    return torch.from_numpy(synth.synthetic_waveform(1.01, 24000, seed=5))[:L].double()


@pytest.mark.parametrize("L", LENGTHS)
def test_encode_oracle_matches_transformers_float64(model_and_oracle, L):
    m, o = model_and_oracle
    x = _wav(L)
    assert x.shape == (L,)
    with torch.no_grad():
        ref_emb = m.encoder(x.view(1, 1, L))
    emb = o.embed(x.view(1, 1, L))
    Fr = -(-L // 320)
    assert emb.shape == ref_emb.shape == (1, 128, Fr)
    err = float((emb - ref_emb).norm() / ref_emb.norm())
    assert err < 1e-12, f"L={L}: embeddings normwise {err:.2e}"
    for n_q, bw in BANDWIDTH.items():
        with torch.no_grad():
            ref = m.encode(x.view(1, 1, L), bandwidth=bw).audio_codes[0, 0]
        got = o.encode(x, n_q)
        assert ref.shape == got.shape == (n_q, Fr)
        assert torch.equal(got, ref), f"L={L} n_q={n_q}: codes differ"


def test_short_inputs_hit_the_zero_extension_rule():
    """The oracle's padding restatement against torch's reflect padding where it is defined, and the zero-extension
    branch where it is not (a sensitivity check of the rule itself)."""
    x = torch.arange(1.0, 4.0, dtype=torch.float64).view(1, 1, 3)
    assert pad1d_reflect(x, 2, 0).flatten().tolist() == [3.0, 2.0, 1.0, 2.0, 3.0]
    # length 3 <= pad 4: zero-extended to 5 samples, reflected, trimmed back
    assert pad1d_reflect(x, 4, 1).flatten().tolist() == [0.0, 0.0, 3.0, 2.0, 1.0, 2.0, 3.0, 0.0]
