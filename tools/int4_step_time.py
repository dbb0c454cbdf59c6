"""Decode throughput of the int4 engine against the bf16 engine, one process, CUDA events.

    python tools/int4_step_time.py [repeats]

Both engines are built from the same synthetic 1.2 B checkpoint.  Workload: the BASELINE configs[1] stage-1 decode -- a
48-token prompt, 750 generated tokens, top-p 0.95, guidance 3, temperature 1 (end of audio disabled so every run decodes
all 750) -- prefilled, then decoded by mvb_s1_decode; only the decode is timed.  After one warm-up run per engine the
engines alternate for `repeats` runs each (default 3).  The same figures at 8 utterances are reported alongside.
Prints one JSON object: ms / token and tokens/s per engine, weight bytes per token from the shapes, achieved GB/s over
those bytes, the card name and its power limit."""
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "metavoice-src_b200"))
import torch  # noqa: E402

from mvb200 import _lib, synth  # noqa: E402
from mvb200.fast_model import ModelArgs, Transformer  # noqa: E402

T_PROMPT, N_TOKENS = 48, 750


def weight_bytes_per_token(c: ModelArgs, int4: bool) -> int:
    """Weights one decode position streams: the layer matrices, the norms, the final norm and lm_head."""
    mats = 4 * c.dim * c.dim + 3 * c.dim * c.intermediate_size
    layer = (mats // 2 + mats // 128 * 4) if int4 else 2 * mats
    return c.n_layer * (layer + 2 * 2 * c.dim) + 2 * (c.vocab_size * c.dim + c.dim)


def run(m: Transformer, n_utts: int, seed: int) -> float:
    """Prefill n_utts prompts, then time mvb_s1_decode over the remaining N_TOKENS - 1 steps; ms per decode step."""
    lib, h, st = m._lib, m.handle, m._stream()
    for u in range(n_utts):
        prompt = synth.synthetic_prompt(T_PROMPT, seed=seed + u)
        spk = synth.synthetic_speaker(seed=seed + 50 + u).reshape(-1).float().contiguous().numpy()
        sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 9999, seed + u)
        lp = prompt.to(torch.int32).contiguous().numpy()
        _lib.check(lib.mvb_s1_admit(h, u, lp.ctypes.data_as(C.c_void_p), T_PROMPT, spk.ctypes.data_as(C.c_void_p),
                                    C.byref(sp), N_TOKENS, None, st))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _lib.check(lib.mvb_s1_decode(h, n_utts, N_TOKENS - 1, st))
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (N_TOKENS - 1)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,power.max_limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        limit, max_limit = (float(v) for v in q.split(","))
    except Exception:   # noqa: BLE001 -- reported as unknown rather than guessed
        limit = max_limit = None
    return {"name": name, "power_limit_W": limit, "power_max_limit_W": max_limit}


def main():
    repeats = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    torch.cuda.set_device(0)
    cfg = ModelArgs.from_name("metavoice-1B")
    sd = synth.stage1_state_dict(synth.FULL, 0)
    engines = {}
    for mode in ("bf16", "int4"):
        m = Transformer.from_state_dict(sd, cfg, device="cuda:0", quantisation_mode=None if mode == "bf16" else mode)
        m.setup_caches(16, cfg.block_size, kv_dtype="bf16", max_new=N_TOKENS)
        engines[mode] = m
    del sd
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
            by = weight_bytes_per_token(cfg, k == "int4")
            res[k] = {"ms_per_step": round(ms, 4), "ms_all": [round(t, 4) for t in ts],
                      "tokens_per_s": round(n_utts * 1e3 / ms, 1), "weight_bytes_per_step": by,
                      "weight_GBps": round(by / ms / 1e6, 1)}
        res["speedup_int4_over_bf16"] = round(res["bf16"]["ms_per_step"] / res["int4"]["ms_per_step"], 3)
        out[f"utts_{n_utts}"] = res
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
