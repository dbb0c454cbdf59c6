"""Cost of a non-production stage-1 architecture: decode ms per token at 1 and 8 utterances on the full-size synthetic
stage 1 (metavoice-1B shape: 24 layers, dim 2048, 16 heads; synthetic weights), one process, CUDA events.

    python tools/stage1_arch_time.py [repeats] [steps]

Three arms, alternated: "production" (rmsnorm, swiglu, no bias; the resident decode kernel), "production_no_resident"
(the same model with MVB_S1_NO_RESIDENT: path A at one utterance, the tensor-core rows path at eight -- the paths a
non-production engine takes) and "gptconfig_default" (layernorm, gelu, bias; intermediate 4 x 2048 = 8192).  Each (arm,
batch) admits its prompts, is warmed up (graph capture, first launches), then the arms alternate: `repeats` rounds
(default 5) of one mvb_s1_decode burst of `steps` positions (default 64) from the same positions, between two events;
the median ms per decode step is reported.  Prints one JSON object with the times, the card name and its power limit
(read-only nvidia-smi query)."""
import ctypes as C
import dataclasses
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402

from int4_step_time import card  # noqa: E402
from mvb200 import _lib, synth  # noqa: E402
from mvb200.fast_model import ModelArgs, Transformer  # noqa: E402

T_PROMPT = 48
BATCHES = (1, 8)
GELU = dataclasses.replace(synth.FULL, norm_type="layernorm", nonlinearity_type="gelu", bias=True, intermediate_size=None)
GELU.__post_init__()


def config(d):
    return ModelArgs(block_size=d.block_size, vocab_size=d.vocab_size, n_layer=d.n_layer, n_head=d.n_head, dim=d.dim,
                     intermediate_size=d.intermediate_size, norm_eps=d.norm_eps, norm_type=d.norm_type,
                     nonlinearity_type=d.nonlinearity_type, bias=d.bias)


def admit(m, n_utts):
    lib, h, st = m._lib, m.handle, m._stream()
    for u in range(n_utts):
        prompt = synth.synthetic_prompt(T_PROMPT, seed=10 + u).to(torch.int32).contiguous().numpy()
        spk = synth.synthetic_speaker(seed=60 + u).reshape(-1).float().contiguous().numpy()
        sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 9999, 1 + u)
        _lib.check(lib.mvb_s1_admit(h, u, prompt.ctypes.data_as(C.c_void_p), T_PROMPT, spk.ctypes.data_as(C.c_void_p),
                                    C.byref(sp), m._cfg.max_new, None, st))


def burst(m, n_utts, steps):
    """One decode burst of `steps` positions from position T_PROMPT; ms per step."""
    lib, h, st = m._lib, m.handle, m._stream()
    sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 9999, 7)
    for u in range(n_utts):
        _lib.check(lib.mvb_s1_begin(h, u, 17 + u, T_PROMPT, C.byref(sp), None, None, st))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _lib.check(lib.mvb_s1_decode(h, n_utts, steps, st))
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    repeats = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 64
    if not torch.cuda.is_available():
        raise SystemExit("stage1_arch_time.py needs a CUDA device")
    torch.cuda.set_device(0)
    prod_sd = synth.stage1_state_dict(synth.FULL, 0)
    gelu_sd = synth.stage1_state_dict(GELU, 0, tie_head=True)
    arms = {}
    for B in BATCHES:
        for name, d, sd, tc in (("production", synth.FULL, prod_sd, "BC"), ("production_no_resident", synth.FULL, prod_sd, "B"),
                                ("gptconfig_default", GELU, gelu_sd, "BC")):
            m = Transformer.from_state_dict(sd, config(d), device="cuda:0")
            m.setup_caches(2 * B, d.block_size, kv_dtype="bf16", tensor_core_path=tc, max_new=256)
            admit(m, B)
            burst(m, B, 4)                                          # warm-up: graph capture, first launches
            arms[f"{name}_u{B}"] = (m, B)
        times = {k: [] for k in arms if k.endswith(f"_u{B}")}
        for _ in range(repeats):
            for k in times:
                times[k].append(burst(arms[k][0], B, steps))
        for k, v in times.items():
            arms[k] = (arms[k][0].close(), v)
        torch.cuda.empty_cache()
    res = {"ms_per_token_median": {k: round(statistics.median(v[1]), 4) for k, v in arms.items()},
           "ms_per_token_all": {k: [round(x, 4) for x in v[1]] for k, v in arms.items()},
           "repeats": repeats, "steps": steps, "card": card()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
