"""Decode cost of prompt guidance (guidance_scale = (s, p)) on the full-size synthetic stage 1, one process, CUDA events.

    python tools/prompt_guidance_time.py [repeats]

Workload (tools/int4_step_time.py's, the bench.py stage-1 configuration): 1.2 B bf16 weights, bf16 KV cache, a 48-token
prompt, 750 generated tokens, top-p 0.95, temperature 1, speaker guidance 3 (end of audio disabled so every run decodes all
750).  Four arms: unguided and guided (p = 2) at 1 and at 4 utterances; a guided utterance takes a companion slot, so
guided 4 decodes 8 slots.  Each run admits its utterances (mvb_s1_admit / mvb_s1_admit_guided), then only mvb_s1_decode
over the remaining 749 steps is timed.  After one warm-up run per arm the arms alternate for `repeats` runs each (default
3); the median is reported.  Prints one JSON object with ms per decode step per arm, the card name and its power limit."""
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from int4_step_time import N_TOKENS, T_PROMPT, card  # noqa: E402
from mvb200 import _lib, synth  # noqa: E402
from mvb200.fast_model import ModelArgs, Transformer  # noqa: E402

EOT, P_GUIDANCE = 2561, 2.0
ARMS = [("unguided", 1), ("guided", 1), ("unguided", 4), ("guided", 4)]


def run(m: Transformer, guided: bool, n: int, seed: int) -> float:
    """Admit n utterances (guided: slot u with companion n + u), then time mvb_s1_decode; ms per decode step."""
    lib, h, st = m._lib, m.handle, m._stream()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)                                      # noqa: E731
    for u in range(n):
        prompt = synth.synthetic_prompt(T_PROMPT, seed=seed + u).to(torch.int32).contiguous().numpy()
        spk = synth.synthetic_speaker(seed=seed + 50 + u).reshape(-1).float().contiguous().numpy()
        sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 9999, seed + u)
        if guided:
            _lib.check(lib.mvb_s1_admit_guided(h, u, n + u, vp(prompt), T_PROMPT, vp(spk), C.byref(sp), P_GUIDANCE, EOT, N_TOKENS,
                                               None, st))
        else:
            _lib.check(lib.mvb_s1_admit(h, u, vp(prompt), T_PROMPT, vp(spk), C.byref(sp), N_TOKENS, None, st))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _lib.check(lib.mvb_s1_decode(h, 2 * n if guided else n, N_TOKENS - 1, st))
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (N_TOKENS - 1)


def main():
    repeats = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    torch.cuda.set_device(0)
    cfg = ModelArgs.from_name("metavoice-1B")
    m = Transformer.from_state_dict(synth.stage1_state_dict(synth.FULL, 0), cfg, device="cuda:0")
    m.setup_caches(16, cfg.block_size, kv_dtype="bf16", max_new=N_TOKENS)
    times = {f"{g}_{n}": [] for g, n in ARMS}
    for g, n in ARMS:                                                                # warm-up: graphs, first launches
        run(m, g == "guided", n, 11)
    for r in range(repeats):
        for g, n in ARMS:
            times[f"{g}_{n}"].append(run(m, g == "guided", n, 100 + 10 * r))
    out = {"workload": f"prompt {T_PROMPT}, {N_TOKENS} tokens, top-p 0.95, guidance (3, {P_GUIDANCE}) vs 3, temperature 1, "
                       "bf16 weights and KV", "card": card(), "repeats": repeats, "ms_per_step": {}, "runs_ms": times}
    for k, v in times.items():
        out["ms_per_step"][k] = round(statistics.median(v), 4)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
