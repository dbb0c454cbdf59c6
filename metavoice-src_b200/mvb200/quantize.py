"""Weight-only quantisation of the stage-1 model: int4 (``quantisation_mode="int4"``, fast_inference_utils.py:297-306) and
int8 (``quantisation_mode="int8"``, fast_inference_utils.py:283-296).

int4 semantics, defined once here and in include/mvb200.h ("int4 packed matrix"):

* Which tensors.  A Linear weight [out, in] is quantised when ``out % 8 == 0`` and ``in % 128 == 0`` (the rule of the
  reference's ``WeightOnlyInt4QuantHandler``, fast_quantize.py:270-299, with groupsize 128).  A Linear with
  ``out % 8 == 0`` whose ``in`` is not a multiple of 128 is rejected (the reference would pad it through a module that does
  not exist).  For MetaVoice-1B that quantises wqkv, wo, w1, w3, w2 of every layer and speaker_cond_pos; lm_head
  (2562 outputs), the embeddings and the norms stay bf16.
* Quantiser.  Per group of 128 consecutive inputs of a row, with every intermediate rounded to bf16 as the reference's
  bf16 tensor arithmetic does: ``s = bf16(bf16(max - min).clamp(1e-6) / 15)``, ``z = bf16(min + 8 s)``,
  ``q = clamp(round_half_even(bf16(bf16(w - bf16(z - 8 s)) / s)), 0, 15)``.  Bit-identical to the reference's
  ``group_quantize_tensor(w, 4, 128)`` (pinned by tests/golden/int4_quant.npz).
* Dequantised weight.  ``W_deq = bf16_rn((q - 8) s + z)``: the exact value rounded once to bf16 (a fused multiply-add
  with a single rounding, ``fma.rn.bf16x2``), the value both CUDA kernels (k_gemv_w4 and k_w4_dequant) use.  The
  reference's Python dequantiser ``group_dequantize_tensor_from_qparams`` rounds twice instead (bf16 after the multiply
  and after the add); how its CUDA int4 matmul (``_weight_int4pack_mm``) rounds could not be checked.  The two values are
  equal wherever the reference's product rounding is exact; elsewhere they differ by at most half a bf16 ulp of the product
  (the reference's first rounding, which cancellation against z can make larger than an ulp of the result) plus one ulp of
  the result (tests/test_int4_quant.py).
* Consequence.  An int4 engine computes the same function as a bf16 engine whose arena holds ``W_deq``.

int8 semantics, defined once here and in include/mvb200.h ("int8 matrix"):

* Which tensors.  Every ``nn.Linear`` of the stage-1 model, as the reference's ``WeightOnlyInt8QuantHandler`` walks
  ``named_modules()`` (fast_quantize.py:151-170): wqkv, wo, w1, w3, w2 of every layer, speaker_cond_pos and lm_head.
  Embeddings and norms stay bf16.
* Quantiser.  The reference quantises the bf16 model, so ``w = fp32(bf16 weight)``; then in fp32
  ``s32 = clamp(max(|min_row|, max_row) / 127.5, min=FLT_EPSILON)``, ``q = clamp(round_half_even(w / s32), -128, 127)``,
  and the stored scale is ``s = bf16_rn(s32)``: q is computed with the fp32 scale, the function uses the bf16 one.
  Bit-identical to the reference's ``dynamically_quantize_per_channel(w.float(), -128, 127, torch.int8)`` with the scales
  cast to bf16 as ``create_quantized_state_dict`` does (pinned by tests/golden/int8_quant.npz).
* Function.  ``WeightOnlyInt8Linear.forward`` is ``F.linear(x, q) * s``; every kernel computes ``y_j = s_j sum_k x_k q_jk``
  with fp32 accumulation over the exact integer weights and the scale applied once per output after the whole sum.
* Consequence.  Where every scale is a power of two, ``s q`` is exact in bf16 and an int8 engine computes the same function
  as a bf16 engine whose arena holds ``W' = s q`` (``int8_dequantized_state_dict``).

fp8 semantics (``quantisation_mode="fp8"``, an extension: the reference has no fp8 mode), defined once here and in
include/mvb200.h ("fp8 matrix"):

* Which tensors.  Those int8 quantises: every ``nn.Linear``.
* Quantiser, per output row j of ``w = fp32(bf16 weight)``: ``s_j = bf16(max(amax_j / 448, FLT_EPSILON))`` and
  ``q_jk = float8_e4m3fn(clamp(w_jk / fp32(s_j), -448, 448))`` (round to nearest even).  Dividing by the rounded scale
  keeps q consistent with the scale stored; the clamp is needed because torch's cast does not saturate (500 -> NaN) and a
  scale rounded down can put |w / s| above 448.  NaN or Inf weights are rejected.
* Function.  ``y_j = s_j sum_k x_k q_jk``: fp32 sums over the exact e4m3 values, the scale applied once per output.
* Layout.  The int8 matrix layout with the codes in a fragment-native order (``pack_fp8_matrix``), so that the decode GEMV
  loads each lane's tensor-core operand with one 128-bit load.
* Consequence.  Where every scale is a power of two, ``s q`` is exact in bf16 and an fp8 engine computes the same function
  as a bf16 engine whose arena holds ``W' = s q`` (``fp8_dequantized_state_dict``).
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch

from ._engine import align_up, pack_arena_bytes
from .fast_model import _GLOBAL_KEYS, _LAYER_KEYS

GROUP = 128
N_BIT = 4


def is_quantised(out_features: int, in_features: int, name: str = "") -> bool:
    """The tensor-selection rule.  Raises for a Linear int4 cannot represent without padding."""
    if out_features % 8 != 0:
        return False
    if in_features % GROUP != 0:
        raise ValueError(f"int4 quantisation needs in_features % {GROUP} == 0; {name or 'a Linear'} has "
                         f"in_features={in_features} (padding is not supported)")
    return True


def group_quantize(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """w [M, K] -> (q uint8 [M, K] in [0, 15], scales bf16 [M, K/128], zeros bf16 [M, K/128])."""
    M, K = w.shape
    if K % GROUP:
        raise ValueError(f"K={K} is not a multiple of {GROUP}")
    g = w.detach().to("cpu", torch.bfloat16).reshape(M * (K // GROUP), GROUP)
    if torch.isnan(g).any():
        raise ValueError("cannot quantise a weight holding NaN")
    lo = g.amin(dim=1, keepdim=True)
    hi = g.amax(dim=1, keepdim=True)
    rng = (hi - lo).clamp(min=1e-6)                  # bf16 tensors: every step below rounds to bf16
    s = rng / (2 ** N_BIT - 1)
    z = lo + s * (2 ** (N_BIT - 1))
    base = z - s * (2 ** (N_BIT - 1))
    q = ((g - base) / s).round().clamp(0, 2 ** N_BIT - 1).to(torch.uint8)
    return q.reshape(M, K), s.reshape(M, K // GROUP), z.reshape(M, K // GROUP)


def _round_to_bf16(v: torch.Tensor) -> torch.Tensor:
    """float64 -> bf16 with ONE round-to-nearest-even at bf16's 8-bit significand (torch's own conversion goes through fp32
    and would round twice).  Exact for results in bf16's normal range."""
    b = v.contiguous().view(torch.int64)
    keep = 52 - 7                                       # float64 fraction bits below bf16's 7
    b = (b + ((1 << (keep - 1)) - 1) + ((b >> keep) & 1)) & ~((1 << keep) - 1)
    return b.view(torch.float64).to(torch.float32).to(torch.bfloat16)   # now exact in fp32 and in bf16


def dequantize(q: torch.Tensor, s: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
    """W_deq = bf16_rn((q - 8) s + z), bf16 [M, K].  The float64 value (q - 8) s + z is exact for every bf16 (s, z) pair
    whose exponents are less than 41 apart (every group the quantiser produces from finite weights)."""
    M, K = q.shape
    qd = q.to(torch.float64).reshape(M, K // GROUP, GROUP) - 2 ** (N_BIT - 1)
    v = qd * s.to(torch.float64)[..., None] + z.to(torch.float64)[..., None]
    return _round_to_bf16(v).reshape(M, K)


# nibble slot n (bits 4n..4n+3) of a little-endian 32-bit word holds k = 8w + _SLOT_K[n]: the even k of the word in slots
# 0-3, the odd ones in slots 4-7, so pair (2i, 2i + 1) sits at bits 4i and 16 + 4i (one shift and mask per bf16x2 pair)
_SLOT_K = [0, 2, 4, 6, 1, 3, 5, 7]


def pack_nibbles(q: torch.Tensor) -> torch.Tensor:
    """q uint8 [M, K] -> uint8 [M, K/2] in the word layout of include/mvb200.h (8 consecutive k per 32-bit word)."""
    M, K = q.shape
    g = q.to(torch.int64).reshape(M, K // 8, 8)
    w = torch.zeros(M, K // 8, dtype=torch.int64)
    for n, k in enumerate(_SLOT_K):
        w |= g[..., k] << (4 * n)
    return w.to(torch.int32).contiguous().view(torch.uint8).reshape(M, K // 2)


def unpack_nibbles(p: torch.Tensor) -> torch.Tensor:
    M, Kh = p.shape
    w = p.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    out = torch.empty(M, Kh // 4, 8, dtype=torch.uint8)
    for n, k in enumerate(_SLOT_K):
        out[..., k] = ((w >> (4 * n)) & 0xF).to(torch.uint8)
    return out.reshape(M, 2 * Kh)


def packed_bytes(M: int, K: int) -> int:
    """Bytes of one packed matrix: the nibble block padded to 256 bytes, then the (scale, zero) block."""
    return align_up(M * K // 2) + M * (K // GROUP) * 4


def pack_matrix(q: torch.Tensor, s: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
    """The int4 packed matrix of include/mvb200.h: nibbles [M, K/2] bytes, then at the next 256-byte boundary
    bf16 [M, K/128, 2] = {scale, zero} of every group."""
    M, K = q.shape
    buf = torch.zeros(packed_bytes(M, K), dtype=torch.uint8)
    nb = M * K // 2
    buf[:nb] = pack_nibbles(q).reshape(-1)
    sz = torch.stack([s, z], dim=-1).contiguous().reshape(-1)
    so = align_up(nb)
    buf[so:] = sz.view(torch.uint8)
    return buf


def unpack_matrix(buf: torch.Tensor, M: int, K: int):
    """Inverse of pack_matrix: (q, scales, zeros)."""
    nb = M * K // 2
    so = align_up(nb)
    q = unpack_nibbles(buf[:nb].reshape(M, K // 2))
    sz = buf[so:so + M * (K // GROUP) * 4].clone().view(torch.bfloat16).reshape(M, K // GROUP, 2)
    return q, sz[..., 0].contiguous(), sz[..., 1].contiguous()


# which entries of the arena (order: fast_model._GLOBAL_KEYS / _LAYER_KEYS) are Linear weights, and which of those the
# int4 engine streams packed
_GLOBAL_LINEAR = {2, 4}            # speaker_cond_pos, lm_head
_LAYER_PACKED = {1, 2, 4, 5, 6}    # wqkv, wo, w1, w3, w2: int4 packed matrices read by k_gemv_w4 / k_w4_dequant


def _keys(n_layer: int) -> List[Tuple[str, bool, bool]]:
    """(checkpoint key, is a Linear weight, stored packed) in arena order."""
    out = [(k, i in _GLOBAL_LINEAR, False) for i, k in enumerate(_GLOBAL_KEYS)]
    for l in range(n_layer):
        out += [(f"transformer.h.{l}.{k}", t in _LAYER_PACKED, t in _LAYER_PACKED) for t, k in enumerate(_LAYER_KEYS)]
    return out


def _strip(state_dict: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    return {(k[len("_orig_mod."):] if k.startswith("_orig_mod.") else k): v for k, v in state_dict.items()}


def pack_arena_int4(state_dict: Dict[str, torch.Tensor], n_layer: int):
    """Checkpoint state dict -> (uint8 arena, byte offsets, bytes the arena's tensors occupy without padding).
    Per layer wqkv / wo / w1 / w3 / w2 become int4 packed matrices (the offset points at the nibble block); a quantised
    Linear the engine does not stream in int4 (speaker_cond_pos, and lm_head when its out % 8 == 0) is stored as W_deq in
    bf16, so it computes what the reference's int4 Linear computes; everything else is the bf16 tensor."""
    sd = _strip(state_dict)
    blobs: List[torch.Tensor] = []
    payload = 0
    for k, linear, packed in _keys(n_layer):
        if k not in sd:
            raise KeyError(f"checkpoint is missing {k}")
        t = sd[k].detach().to(torch.bfloat16)
        if linear and is_quantised(t.shape[0], t.shape[1], k):
            q, s, z = group_quantize(t)
            if packed:
                blob = pack_matrix(q, s, z)
                payload += t.numel() // 2 + s.numel() * 4
                blobs.append(blob)
                continue
            t = dequantize(q, s, z)
        elif packed:
            raise ValueError(f"{k}: the int4 engine streams this matrix packed, but out % 8 != 0")
        blobs.append(t)
        payload += t.numel() * 2
    arena, offsets = pack_arena_bytes(blobs)
    return arena, offsets, payload


def dequantized_state_dict(state_dict: Dict[str, torch.Tensor], n_layer: int) -> Dict[str, torch.Tensor]:
    """The checkpoint with every quantised Linear replaced by W_deq (bf16): the bf16 model an int4 engine equals."""
    sd = _strip(state_dict)
    out = dict(sd)
    for k, linear, _ in _keys(n_layer):
        t = sd[k]
        if linear and is_quantised(t.shape[0], t.shape[1], k):
            out[k] = dequantize(*group_quantize(t.to(torch.bfloat16)))
    return out


# ---- weight-only int8 -------------------------------------------------------------------------------------------------
_FLT_EPS = torch.finfo(torch.float32).eps


def quantize_per_channel(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """w [M, K] -> (q int8 [M, K], s bf16 [M]): the reference's dynamically_quantize_per_channel(bf16 w -> fp32, -128, 127)
    with the scales cast to bf16 (fast_quantize.py:38-67, 160-162)."""
    wf = w.detach().to("cpu", torch.bfloat16).float()
    if torch.isnan(wf).any():
        raise ValueError("cannot quantise a weight holding NaN")
    lo, hi = torch.aminmax(wf, dim=1)
    amax = torch.maximum(-torch.clamp(lo, max=0.0), torch.clamp(hi, min=0.0))
    s32 = torch.clamp(amax / 127.5, min=_FLT_EPS)
    q = torch.clamp(torch.round(wf / s32[:, None]), -128, 127).to(torch.int8)
    return q, s32.to(torch.bfloat16)


def dequantize_int8(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """W' = bf16_rn(s q), bf16 [M, K] (s q is exact in fp32: 8 + 8 significant bits)."""
    return (q.float() * s.float()[:, None]).to(torch.bfloat16)


def int8_matrix_bytes(M: int, K: int) -> int:
    """Bytes of one int8 matrix: int8 [M, K] padded to 256 bytes, then bf16 [M] scales."""
    return align_up(M * K) + 2 * M


def pack_int8_matrix(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """The int8 matrix of include/mvb200.h: int8 [M][K] row-major, then at the next 256-byte boundary bf16 [M] scales."""
    M, K = q.shape
    buf = torch.zeros(int8_matrix_bytes(M, K), dtype=torch.uint8)
    buf[:M * K] = q.contiguous().reshape(-1).view(torch.uint8)
    so = align_up(M * K)
    buf[so:] = s.contiguous().view(torch.uint8)
    return buf


def unpack_int8_matrix(buf: torch.Tensor, M: int, K: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Inverse of pack_int8_matrix: (q, s)."""
    so = align_up(M * K)
    q = buf[:M * K].clone().view(torch.int8).reshape(M, K)
    return q, buf[so:so + 2 * M].clone().view(torch.bfloat16)


def _pack_arena_per_channel(state_dict: Dict[str, torch.Tensor], n_layer: int, quantise, pack):
    """Checkpoint state dict -> (uint8 arena, byte offsets, payload bytes).  Every Linear weight w becomes the one-byte
    matrix pack(*quantise(w)) (its offset points at the code block); embeddings and norms are the bf16 tensors.  The
    payload is the reference's ``model_size``: one byte per weight plus the bf16 scales plus the bf16 tensors."""
    sd = _strip(state_dict)
    blobs: List[torch.Tensor] = []
    payload = 0
    for k, linear, _ in _keys(n_layer):
        if k not in sd:
            raise KeyError(f"checkpoint is missing {k}")
        t = sd[k].detach()
        if linear:
            q, s = quantise(t)
            blobs.append(pack(q, s))
            payload += q.numel() + 2 * s.numel()
        else:
            t = t.to(torch.bfloat16)
            blobs.append(t)
            payload += t.numel() * 2
    arena, offsets = pack_arena_bytes(blobs)
    return arena, offsets, payload


def _per_channel_dequantized_state_dict(state_dict: Dict[str, torch.Tensor], n_layer: int, quantise, dequantise):
    """The checkpoint with every Linear w replaced by dequantise(*quantise(w))."""
    sd = _strip(state_dict)
    out = dict(sd)
    for k, linear, _ in _keys(n_layer):
        if linear:
            out[k] = dequantise(*quantise(sd[k]))
    return out


def pack_arena_int8(state_dict: Dict[str, torch.Tensor], n_layer: int):
    """Checkpoint state dict -> (uint8 arena, byte offsets, payload bytes) with every Linear weight an int8 matrix
    (_pack_arena_per_channel)."""
    return _pack_arena_per_channel(state_dict, n_layer, quantize_per_channel, pack_int8_matrix)


def int8_dequantized_state_dict(state_dict: Dict[str, torch.Tensor], n_layer: int) -> Dict[str, torch.Tensor]:
    """The checkpoint with every Linear replaced by bf16_rn(s q): the bf16 model an int8 engine equals when every scale is
    a power of two (and approximates to the rounding of s q otherwise)."""
    return _per_channel_dequantized_state_dict(state_dict, n_layer, quantize_per_channel, dequantize_int8)


# ---- weight-only fp8 (e4m3) -------------------------------------------------------------------------------------------
E4M3_MAX = 448.0


def quantize_fp8_per_channel(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """w [M, K] -> (q float8_e4m3fn [M, K], s bf16 [M]): s = bf16(max(amax / 448, FLT_EPSILON)) per row, q =
    e4m3(clamp(w / s, -448, 448))."""
    wf = w.detach().to("cpu", torch.bfloat16).float()
    if not torch.isfinite(wf).all():
        raise ValueError("cannot quantise a weight holding NaN or Inf")
    amax = wf.abs().amax(dim=1)
    s = torch.clamp(amax / E4M3_MAX, min=_FLT_EPS).to(torch.bfloat16)
    q = torch.clamp(wf / s.float()[:, None], -E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q, s


def dequantize_fp8(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """W' = bf16_rn(s q), bf16 [M, K] (s q is exact in fp32: 8 + 4 significant bits)."""
    return (q.float() * s.float()[:, None]).to(torch.bfloat16)


# Fragment-native order of the codes of a 16-row block (include/mvb200.h, "fp8 matrix"): the block [16, K] viewed as
# (row >> 3, row & 7, k >> 5, k >> 4 & 1, k >> 3 & 1, k >> 1 & 3, k & 1) -> (chunk, lane = (row & 7, k >> 1 & 3),
# word = (k >> 4 & 1, k >> 3 & 1), byte = (k & 1, row >> 3)).
_F8_PERM = (0, 3, 2, 6, 4, 5, 7, 1)
_F8_UNPERM = (0, 7, 2, 1, 4, 5, 3, 6)


def pack_fp8_codes(q: torch.Tensor) -> torch.Tensor:
    """q float8_e4m3fn [M, K] -> uint8 [M * K]: rows [0, M & ~15) in the fragment-native order, the rest row-major."""
    M, K = q.shape
    if M % 2 or K % 256:
        raise ValueError(f"an fp8 matrix needs an even M and K % 256 == 0 (got {M} x {K})")
    u = q.contiguous().view(torch.uint8)
    M16 = M // 16 * 16
    blocks = u[:M16].reshape(M16 // 16, 2, 8, K // 32, 2, 2, 4, 2).permute(*_F8_PERM).reshape(-1)
    return torch.cat([blocks, u[M16:].reshape(-1)])


def unpack_fp8_codes(codes: torch.Tensor, M: int, K: int) -> torch.Tensor:
    """Inverse of pack_fp8_codes: uint8 [M * K] -> float8_e4m3fn [M, K]."""
    M16 = M // 16 * 16
    blocks = codes[:M16 * K].reshape(M16 // 16, K // 32, 8, 4, 2, 2, 2, 2).permute(*_F8_UNPERM).reshape(M16, K)
    return torch.cat([blocks, codes[M16 * K:M * K].reshape(M - M16, K)]).contiguous().view(torch.float8_e4m3fn)


def pack_fp8_matrix(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """The fp8 matrix of include/mvb200.h: the codes of pack_fp8_codes, then at the next 256-byte boundary bf16 [M]
    scales (the int8 matrix layout, int8_matrix_bytes(M, K) bytes)."""
    M, K = q.shape
    buf = torch.zeros(int8_matrix_bytes(M, K), dtype=torch.uint8)
    buf[:M * K] = pack_fp8_codes(q)
    so = align_up(M * K)
    buf[so:] = s.contiguous().view(torch.uint8)
    return buf


def unpack_fp8_matrix(buf: torch.Tensor, M: int, K: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Inverse of pack_fp8_matrix: (q, s)."""
    so = align_up(M * K)
    return unpack_fp8_codes(buf[:M * K], M, K), buf[so:so + 2 * M].clone().view(torch.bfloat16)


def pack_arena_fp8(state_dict: Dict[str, torch.Tensor], n_layer: int):
    """Checkpoint state dict -> (uint8 arena, byte offsets, payload bytes) with every Linear weight an fp8 matrix
    (_pack_arena_per_channel)."""
    return _pack_arena_per_channel(state_dict, n_layer, quantize_fp8_per_channel, pack_fp8_matrix)


def quantize_kv_fp8(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The fp8 KV cache's quantiser (``kv_dtype="fp8"``, include/mvb200.h at mvb_s1_kv_bytes): x [..., 128] fp32 head
    vectors -> (codes float8_e4m3fn [..., 128], scales bf16 [...]) with, per vector,
    ``s = bf16_rn(max(amax|x| / 448, FLT_EPSILON))`` and ``q = e4m3_rn(clamp(x / s, -448, 448))``: quantize_fp8_per_channel
    without the bf16 rounding of the input.  Non-finite input has one encoding, which k_kv_store_f8 stores too: a NaN
    anywhere in x gives s = NaN (bits 0x7fc0) and every code 0x7f; otherwise an infinite element makes s = +inf, its own
    code 0x7f (inf / inf) and every finite element's a signed zero."""
    xf = x.detach().to("cpu", torch.float32)
    nan_row = torch.isnan(xf).any(-1)
    amax = xf.abs().amax(-1)
    s = torch.clamp(amax / E4M3_MAX, min=_FLT_EPS).to(torch.bfloat16)
    r = xf / s.float()[..., None]
    codes = torch.clamp(r, -E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8)
    codes = torch.where(torch.isnan(r) | nan_row[..., None], torch.full_like(codes, 0x7F), codes)
    s = torch.where(nan_row, torch.full_like(s.view(torch.int16), 0x7FC0), s.view(torch.int16)).view(torch.bfloat16)
    return codes.view(torch.float8_e4m3fn), s


def dequantize_kv_fp8(codes: torch.Tensor, scales: torch.Tensor) -> torch.Tensor:
    """fp32 s q of the fp8 KV cache, exactly (8 + 4 significant bits): codes [..., 128], scales [...]."""
    return codes.float() * scales.float()[..., None]


def fp8_dequantized_state_dict(state_dict: Dict[str, torch.Tensor], n_layer: int) -> Dict[str, torch.Tensor]:
    """The checkpoint with every Linear replaced by bf16_rn(s q): the bf16 model an fp8 engine equals when every scale is
    a power of two (and approximates to the rounding of s q otherwise)."""
    return _per_channel_dequantized_state_dict(state_dict, n_layer, quantize_fp8_per_channel, dequantize_fp8)
