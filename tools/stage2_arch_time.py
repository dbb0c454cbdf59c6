"""Cost of the stage-2 architectures: one mvb_s2_forward (captured-graph replay) on the full-size synthetic stage 2,
production (rmsnorm, swiglu, no bias) against GPTConfig's default (layernorm, gelu, bias), one process, CUDA events.

    python tools/stage2_arch_time.py [repeats] [calls]

S2_FULL (6 layers, E = 384, t = 1024, 6 target hierarchies of 1025) at batch 1 and 8, with a speaker, top-k 200.  Each
(architecture, batch) arm is warmed up (graph capture, first launches), then the arms alternate: `repeats` rounds
(default 5) of `calls` back-to-back forwards each (default 20) between two events; the median ms per forward is
reported.  Prints one JSON object with the times, the card name and its power limit."""
import dataclasses
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from int4_step_time import card  # noqa: E402
from mvb200 import synth  # noqa: E402
from mvb200.second_stage import SecondStage  # noqa: E402

ARCHS = {"production": synth.S2_FULL,
         "gptconfig_default": dataclasses.replace(synth.S2_FULL, norm_type="layernorm", nonlinearity_type="gelu", bias=True)}
BATCHES = (1, 8)


def inputs(m, d, B):
    idx, spk = [], []
    for j in range(B):
        text, cb0, cb1 = synth.synthetic_stage2_input(d, 300 + 40 * j, seed=j)
        idx.append(m.build_input(text, [cb0, cb1]))
        spk.append(synth.synthetic_speaker(seed=100 + j))
    return torch.stack(idx), torch.cat(spk)[:, None]


def run(m, idx, spk, calls):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for s in range(calls):
        m.forward_tokens(idx, spk, 1.0, 200, seed=s)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def main():
    repeats = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    calls = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    if not torch.cuda.is_available():
        raise SystemExit("stage2_arch_time.py needs a CUDA device")
    torch.cuda.set_device(0)
    engines = {a: SecondStage(synth.stage2_checkpoint(d, 1), device="cuda:0", max_batch=max(BATCHES)) for a, d in ARCHS.items()}
    feeds = {(a, B): inputs(engines[a], ARCHS[a], B) for a in ARCHS for B in BATCHES}
    for (a, B), (idx, spk) in feeds.items():                                  # warm-up: graph capture, first launches
        run(engines[a], idx, spk, 3)
    times = {f"{a}_b{B}": [] for a, B in feeds}
    for _ in range(repeats):
        for (a, B), (idx, spk) in feeds.items():
            times[f"{a}_b{B}"].append(run(engines[a], idx, spk, calls))
    res = {"ms_per_forward_median": {k: round(statistics.median(v), 4) for k, v in times.items()},
           "ms_per_forward_all": {k: [round(x, 4) for x in v] for k, v in times.items()},
           "repeats": repeats, "calls": calls, "card": card()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
