"""Decode ms / token of the stage-1 engine with a bf16 KV cache against an fp8 KV cache, one process, CUDA events.

    python tools/kv_fp8_step_time.py [repeats] [--steps N]

Production 1.2 B synthetic checkpoint, bf16 weights (one device arena shared by every engine).  For 1, 8, 32 and 64
utterances and two contexts -- mean context ~423 (a 48-token prompt plus 750 generated tokens: positions 391 .. 454) and
long-form ~1500 (1468 .. 1531) -- every slot is placed at the window's first position with mvb_s1_begin over a zeroed
cache (attention reads [0, pos] whatever the values, so no prefill is needed) and mvb_s1_decode runs `--steps` positions
(default 64), timed with CUDA events.  Engines: bf16 KV on the per-layer paths (path A at one utterance, the tensor-core
rows path above), fp8 KV (the same paths: an fp8 cache never takes the resident kernel), and at one utterance the
default bf16-KV engine, which decodes on the resident kernel (path C).  Each engine is created for the batch, warmed up
(graph capture) and closed again, since a 64-slot bf16 cache (51.5 GB) and a 64-slot fp8 cache (26.2 GB) do not fit on
one 80 GB card together; the engines alternate for `repeats` rounds (default 3).  Prints one JSON object: per cell the
median ms / token, all repeats, and the algorithmic weight and cache bytes one decode step reads, with the card's name and
power limit read in the same call."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from int4_step_time import card, weight_bytes_per_token  # noqa: E402
from mvb200 import _lib, synth  # noqa: E402
from mvb200.fast_model import ModelArgs, Transformer, pack_arena  # noqa: E402

UTTS = (1, 8, 32, 64)
CONTEXTS = {"mean_423": 391, "long_1500": 1468}     # first position of the timed window
# engine -> (kv_dtype, tensor_core_path); "bf16_path_c" only at one utterance
ENGINES = {"bf16": ("bf16", "B"), "fp8": ("fp8", None), "bf16_path_c": ("bf16", None)}


def cache_bytes_per_step(c: ModelArgs, kv: str, n_utts: int, first: int, steps: int) -> float:
    """Mean bytes of K / V one decode step reads: 2 rows x layers x {K, V} x heads per context position, 128 elements
    (plus one bf16 scale per vector for fp8) each, over the window's context lengths first + 1 .. first + steps."""
    per_vec = {"bf16": 256, "fp8": 130}[kv]
    mean_L = first + (steps + 1) / 2
    return n_utts * 2 * c.n_layer * 2 * c.n_head * per_vec * mean_L


def timed(m: Transformer, n_utts: int, first: int, steps: int) -> float:
    lib, h, st = m._lib, m.handle, m._stream()
    m._kv.zero_()
    sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 99999, 1)
    for u in range(n_utts):
        _lib.check(lib.mvb_s1_begin(h, u, 17 + u, first, C.byref(sp), None, None, st))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _lib.check(lib.mvb_s1_decode(h, n_utts, steps, st))
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("repeats", type=int, nargs="?", default=3)
    ap.add_argument("--steps", type=int, default=64)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    cfg = ModelArgs.from_name("metavoice-1B")
    arena, offsets = pack_arena(synth.stage1_state_dict(synth.FULL, 0), cfg.n_layer)
    arena = arena.cuda()
    wb = weight_bytes_per_token(cfg, False)
    out = {"workload": f"bf16 weights, {a.steps} decode steps per window, top-p 0.95, guidance 3", "card": card(),
           "repeats": a.repeats}
    for n_utts in UTTS:
        for ctx, first in CONTEXTS.items():
            kinds = [k for k in ENGINES if k != "bf16_path_c" or n_utts == 1]
            times = {k: [] for k in kinds}
            for r in range(a.repeats):
                for k in kinds:
                    kv, tc = ENGINES[k]
                    m = Transformer(cfg, arena, offsets, device="cuda:0")
                    try:
                        m.setup_caches(2 * n_utts, cfg.block_size, kv_dtype=kv, tensor_core_path=tc)
                    except (RuntimeError, _lib.MvbError) as e:   # the card's free memory: the cell is not measured
                        print(f"{k} at {n_utts} utterances: {e}", file=sys.stderr)
                        m.close()
                        continue
                    timed(m, n_utts, first, 4)                  # warm-up: graph capture, first launches
                    times[k].append(timed(m, n_utts, first, a.steps))
                    m.close()
                    torch.cuda.empty_cache()
            cell = {}
            for k, ts in times.items():
                kv = ENGINES[k][0]
                if not ts:
                    cell[k] = "not measured"
                    continue
                ms = sorted(ts)[len(ts) // 2]
                cb = cache_bytes_per_step(cfg, kv, n_utts, first, a.steps)
                cell[k] = {"ms_per_token_step": round(ms, 4), "ms_all": [round(t, 4) for t in ts],
                           "tokens_per_s": round(n_utts * 1e3 / ms, 1), "weight_bytes_per_step": wb,
                           "cache_bytes_per_step": int(cb), "GBps_over_weight_and_cache": round((wb + cb) / ms / 1e6, 1)}
            if any(isinstance(v, str) for v in cell.values()):
                out[f"utts_{n_utts}_{ctx}"] = cell
                continue
            cell["speed_fp8_over_bf16"] = round(cell["bf16"]["ms_per_token_step"] / cell["fp8"]["ms_per_token_step"], 3)
            if "bf16_path_c" in cell:
                cell["speed_fp8_over_bf16_path_c"] = round(cell["bf16_path_c"]["ms_per_token_step"] / cell["fp8"]["ms_per_token_step"], 3)
            out[f"utts_{n_utts}_{ctx}"] = cell
            print(json.dumps({f"utts_{n_utts}_{ctx}": cell}), file=sys.stderr, flush=True)
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
