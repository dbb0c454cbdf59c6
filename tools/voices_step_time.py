"""Decode ms / step of one stage-1 engine serving several voices (last-N-block finetunes), one process, CUDA events.

    python tools/voices_step_time.py [repeats] [--steps N]

Production 1.2 B synthetic checkpoint, bf16 weights and bf16 KV cache; seven voices that overlay the last block and ln_f
(N = 1, 103 MB each; their values are the base's scaled by 1.01, which only the timing sees).  Every slot is placed at
position 391 with mvb_s1_begin over a zeroed cache (attention reads [0, pos] whatever the values) and mvb_s1_decode runs
`--steps` positions (default 64).  Arms, alternated for `repeats` rounds (default 5), median reported:
  utts8_one_voice     8 utterances on voice 0, default paths (the resident decode kernel);
  utts8_one_voice_B   8 utterances on voice 0 on the tensor-core rows path (no resident kernel);
  utts8_eight_voices  8 utterances on voices 0..7 (the rows path; the last block's projections are grouped launches
                      over 8 units, the head one GEMM);
  utts1_voice0        1 utterance on voice 0 (the resident kernel);
  utts1_finetuned     1 utterance on voice 1 (path A, the CUDA-core GEMVs).
Prints one JSON object with the card's name and power limit read in the same call."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from int4_step_time import card  # noqa: E402
from mvb200 import _lib, synth  # noqa: E402
from mvb200.fast_model import ModelArgs, Transformer  # noqa: E402

FIRST = 391


def timed(m: Transformer, voices, steps: int) -> float:
    lib, h, st = m._lib, m.handle, m._stream()
    m._kv.zero_()
    sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 99999, 1)
    for u, v in enumerate(voices):
        m.set_voice(u, v)
        _lib.check(lib.mvb_s1_begin(h, u, 17 + u, FIRST, C.byref(sp), None, None, st))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _lib.check(lib.mvb_s1_decode(h, len(voices), steps, st))
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("repeats", type=int, nargs="?", default=5)
    ap.add_argument("--steps", type=int, default=64)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    cfg = ModelArgs.from_name("metavoice-1B")
    base = synth.stage1_state_dict(synth.FULL, 0)
    last = [k for k in base if k.startswith(f"transformer.h.{cfg.n_layer - 1}.") or k.startswith("transformer.ln_f.")]
    ft = dict(base)
    for k in last:
        ft[k] = (base[k].float() * 1.01).to(torch.bfloat16)
    e8 = Transformer.from_state_dict(base, cfg, device="cuda:0")
    e8.setup_caches(16, cfg.block_size, max_new=256)
    e8b = Transformer.from_state_dict(base, cfg, device="cuda:0")
    e8b.setup_caches(16, cfg.block_size, max_new=256, tensor_core_path="B")
    e1 = Transformer.from_state_dict(base, cfg, device="cuda:0")
    e1.setup_caches(2, cfg.block_size, max_new=256)
    for _ in range(7):
        e8.add_voice(ft)
    e1.add_voice(ft)
    del base, ft
    arms = {"utts8_one_voice": (e8, [0] * 8), "utts8_one_voice_B": (e8b, [0] * 8), "utts8_eight_voices": (e8, list(range(8))),
            "utts1_voice0": (e1, [0]), "utts1_finetuned": (e1, [1])}
    times = {k: [] for k in arms}
    for m, vs in arms.values():
        timed(m, vs, 4)                               # warm-up: graph capture, first launches
    for _ in range(a.repeats):
        for k, (m, vs) in arms.items():
            times[k].append(timed(m, vs, a.steps))
    med = {k: sorted(ts)[len(ts) // 2] for k, ts in times.items()}
    out = {"workload": f"bf16 weights and KV, {a.steps} decode steps from position {FIRST}, voices overlay 1 block",
           "card": card(), "repeats": a.repeats,
           "ms_per_step": {k: round(v, 4) for k, v in med.items()},
           "ms_all": {k: [round(t, 4) for t in ts] for k, ts in times.items()},
           "eight_voices_over_one_voice_B": round(med["utts8_eight_voices"] / med["utts8_one_voice_B"], 3),
           "eight_voices_over_one_voice": round(med["utts8_eight_voices"] / med["utts8_one_voice"], 3),
           "finetuned_over_voice0_at_1": round(med["utts1_finetuned"] / med["utts1_voice0"], 3),
           "card_after": card()}
    for m in (e8, e8b, e1):
        m.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
