"""Decode throughput of the fp8 engine against the bf16 and int8 engines, one process, CUDA events.

    python tools/fp8_step_time.py [repeats] [--profile OUT_DIR]

The three engines are built from the same synthetic 1.2 B checkpoint.  Workload (tools/int4_step_time.py's): the BASELINE
configs[1] stage-1 decode -- a 48-token prompt, 750 generated tokens, top-p 0.95, guidance 3, temperature 1 (end of audio
disabled so every run decodes all 750) -- prefilled, then decoded by mvb_s1_decode; only the decode is timed.  After one
warm-up run per engine the engines alternate for `repeats` runs each (default 3), at 1 and at 8 utterances.  Prints one JSON
object: ms / token and tokens/s per engine, weight bytes per decode position from the shapes, achieved GB/s over those bytes,
the card name and its power limit.  The weights of an fp8 decode position are read once for all utterances (k_gemv_f8 has
one launch row up to 8 utterances), those of an int8 one once per utterance; the byte count is per position either way.
--profile also writes a torch.profiler kernel table (CUDA time per kernel name) of 64 decode steps at 1 and at 8
utterances for the int8 and fp8 engines, in a separate pass after the timing."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from int4_step_time import N_TOKENS, T_PROMPT, card, run, weight_bytes_per_token  # noqa: E402
from int8_step_time import int8_weight_bytes_per_token  # noqa: E402
from mvb200 import _lib, synth  # noqa: E402
from mvb200.fast_model import ModelArgs, Transformer  # noqa: E402

MODES = ("bf16", "int8", "fp8")


def profile(engines, out_dir):
    from torch.profiler import ProfilerActivity, profile as prof
    os.makedirs(out_dir, exist_ok=True)
    for k in ("int8", "fp8"):
        for n_utts in (1, 8):
            m = engines[k]
            run(m, n_utts, 7)                                       # capture outside the trace
            lib, h, st = m._lib, m.handle, m._stream()
            with prof(activities=[ProfilerActivity.CUDA]) as p:
                _lib.check(lib.mvb_s1_decode(h, n_utts, 64, st))
                torch.cuda.synchronize()
            table = p.key_averages().table(sort_by="cuda_time_total", row_limit=20)
            with open(os.path.join(out_dir, f"fp8_step_time_profile_{k}_u{n_utts}.txt"), "w") as f:
                f.write(table)
            print(f"--- {k}: 64 decode steps at {n_utts} utterance(s)\n{table}", file=sys.stderr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("repeats", type=int, nargs="?", default=3)
    ap.add_argument("--profile", metavar="OUT_DIR")
    a = ap.parse_args()
    repeats, prof_dir = a.repeats, a.profile
    torch.cuda.set_device(0)
    cfg = ModelArgs.from_name("metavoice-1B")
    sd = synth.stage1_state_dict(synth.FULL, 0)
    engines = {}
    for mode in MODES:
        m = Transformer.from_state_dict(sd, cfg, device="cuda:0", quantisation_mode=None if mode == "bf16" else mode)
        m.setup_caches(16, cfg.block_size, kv_dtype="bf16", max_new=N_TOKENS)
        engines[mode] = m
    del sd
    # an fp8 matrix has the int8 matrix's bytes
    bytes_per_step = {"bf16": weight_bytes_per_token(cfg, False), "int8": int8_weight_bytes_per_token(cfg),
                      "fp8": int8_weight_bytes_per_token(cfg)}
    out = {"workload": f"prompt {T_PROMPT}, {N_TOKENS} tokens, top-p 0.95, guidance 3, temperature 1, bf16 KV", "card": card(),
           "repeats": repeats}
    for n_utts in (1, 8):
        for m in engines.values():
            run(m, n_utts, 1)                                       # warm-up (graph capture)
        times = {k: [] for k in engines}
        for r in range(repeats):
            for k, m in engines.items():
                times[k].append(run(m, n_utts, 100 + r))
        res = {}
        for k, ts in times.items():
            ms = sorted(ts)[len(ts) // 2]
            by = bytes_per_step[k]
            res[k] = {"ms_per_step": round(ms, 4), "ms_all": [round(t, 4) for t in ts],
                      "tokens_per_s": round(n_utts * 1e3 / ms, 1), "weight_bytes_per_step": by,
                      "weight_GBps": round(by / ms / 1e6, 1)}
        res["speed_fp8_over_bf16"] = round(res["bf16"]["ms_per_step"] / res["fp8"]["ms_per_step"], 3)
        res["speed_fp8_over_int8"] = round(res["int8"]["ms_per_step"] / res["fp8"]["ms_per_step"], 3)
        out[f"utts_{n_utts}"] = res
    out["card_after"] = card()
    print(json.dumps(out))
    if prof_dir:
        profile(engines, prof_dir)


if __name__ == "__main__":
    main()
