"""CPU: the weight-arena layout every libmvb200 engine reads (mvb200/_engine.py pack_arena_bytes) -- each tensor's raw
bytes at the next 256-byte boundary, in order, zero padding -- and the stage-1 arenas of all three formats (bf16, int4,
int8) against a restatement of that layout built with numpy."""
import numpy as np
import pytest
import torch

from mvb200 import quantize as Q, synth
from mvb200._engine import pack_arena_bytes, split_runs
from mvb200.fast_model import _GLOBAL_KEYS, _LAYER_KEYS, pack_arena


def _raw(t: torch.Tensor) -> bytes:
    """The tensor's bytes in row-major order (bf16 through its int16 bit pattern: numpy has no bf16)."""
    t = t.detach().contiguous()
    if t.dtype == torch.bfloat16:
        t = t.view(torch.int16)
    return t.numpy().tobytes()


def _restated(blobs):
    """(arena bytes, offsets): the layout restated from its definition."""
    out, offsets = bytearray(), []
    for b in blobs:
        offsets.append(len(out))
        out += _raw(b)
        out += bytes(-len(out) % 256)
    return bytes(out), offsets


def _check(arena, offsets, blobs):
    want, want_offsets = _restated(blobs)
    assert arena.dtype == torch.uint8 and arena.device.type == "cpu" and arena.dim() == 1
    assert offsets == want_offsets and all(o % 256 == 0 for o in offsets)
    assert arena.numpy().tobytes() == want
    ends = [o + len(_raw(b)) for o, b in zip(offsets, blobs)]
    for end, nxt in zip(ends, offsets[1:] + [arena.numel()]):
        assert not arena[end:nxt].any(), "padding must be zero"


def test_mixed_dtypes():
    g = torch.Generator().manual_seed(0)
    blobs = [torch.randn(3, generator=g).to(torch.bfloat16),          # 6 bytes
             torch.randn(5, generator=g),                               # 20 bytes
             torch.randint(0, 256, (300,), generator=g, dtype=torch.uint8),
             torch.randn(64, generator=g),                              # exactly 256 bytes: no padding
             torch.randint(-128, 128, (7, 9), generator=g, dtype=torch.int8),
             torch.empty(0, dtype=torch.float32),                       # no bytes: shares the next tensor's offset
             torch.randn(6, 4, generator=g).t(),                        # not contiguous: packed in row-major order
             torch.randn(2, 3, generator=g, dtype=torch.float64)]
    arena, offsets = pack_arena_bytes(blobs)
    _check(arena, offsets, blobs)
    assert offsets == [0, 256, 512, 1024, 1280, 1536, 1536, 1792] and arena.numel() == 2048
    assert torch.equal(arena[1536:1536 + 96].view(torch.float32).view(4, 6), blobs[6])


def test_empty_list():
    arena, offsets = pack_arena_bytes([])
    assert arena.numel() == 0 and offsets == []


def _tiny():
    d = synth.TINY
    sd = synth.stage1_state_dict(d, 0)
    keys = list(_GLOBAL_KEYS) + [f"transformer.h.{l}.{k}" for l in range(d.n_layer) for k in _LAYER_KEYS]
    return d, sd, keys


def test_stage1_bf16_arena():
    d, sd, keys = _tiny()
    arena, offsets = pack_arena({"_orig_mod." + k: v for k, v in sd.items()}, d.n_layer)
    _check(arena, offsets, [sd[k].to(torch.bfloat16) for k in keys])


def test_stage1_int4_arena():
    d, sd, keys = _tiny()
    arena, offsets, _ = Q.pack_arena_int4(sd, d.n_layer)
    packed = {f"transformer.h.{l}.{k}" for l in range(d.n_layer) for k in _LAYER_KEYS if k.startswith(("attn.", "mlp."))}
    blobs = []
    for k in keys:
        t = sd[k].to(torch.bfloat16)
        if k in packed:
            blobs.append(Q.pack_matrix(*Q.group_quantize(t)))
        elif k == "speaker_cond_pos.weight":              # a quantised Linear the engine reads as W_deq in bf16
            blobs.append(Q.dequantize(*Q.group_quantize(t)))
        else:                                             # lm_head (2562 outputs), embeddings, norms
            blobs.append(t)
    _check(arena, offsets, blobs)


def test_stage1_int8_arena():
    d, sd, keys = _tiny()
    arena, offsets, _ = Q.pack_arena_int8(sd, d.n_layer)
    linear = {"speaker_cond_pos.weight", "lm_heads.0.weight"} | \
        {f"transformer.h.{l}.{k}" for l in range(d.n_layer) for k in _LAYER_KEYS if k.startswith(("attn.", "mlp."))}
    blobs = [Q.pack_int8_matrix(*Q.quantize_per_channel(sd[k])) if k in linear else sd[k].to(torch.bfloat16) for k in keys]
    _check(arena, offsets, blobs)


@pytest.mark.parametrize("sizes,max_items,max_total,want", [
    ([], 4, 10, []),
    ([3, 3, 3], 4, 10, [[0, 1, 2]]),
    ([3, 3, 3, 3, 3], 2, 100, [[0, 1], [2, 3], [4]]),
    ([4, 4, 4], 8, 8, [[0, 1], [2]]),
    ([2, 20, 2, 2], 8, 10, [[0], [1], [2, 3]]),           # an item over max_total runs alone
    ([20], 8, 10, [[0]]),
])
def test_split_runs(sizes, max_items, max_total, want):
    assert [list(r) for r in split_runs(sizes, max_items, max_total)] == want
