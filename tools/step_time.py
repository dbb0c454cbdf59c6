"""Decode-step time (CUDA events) for several engine configurations in one process.
Usage: python tools/step_time.py "A:1,B:8,C:1,C:1:unfused,C:8" [context_len]
  A = CUDA-core path, B = tensor-core rows path (from 2 utterances up), C = persistent fused kernel; second field =
  utterances; optional third field `unfused`: the persistent kernel leaves the logits to k_sample."""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "metavoice-src_b200"))
import torch  # noqa: E402

import bench  # noqa: E402
from mvb200 import _lib, synth  # noqa: E402
from mvb200.fast_model import ModelArgs, Transformer, pack_arena  # noqa: E402

spec = sys.argv[1] if len(sys.argv) > 1 else "A:1,B:8"
L_mid = int(sys.argv[2]) if len(sys.argv) > 2 else 423
dev = torch.device("cuda:0")
torch.cuda.set_device(dev)
d = synth.FULL
cfg = ModelArgs.from_name("metavoice-1B")
arena, offsets = pack_arena(synth.stage1_state_dict(d, 0), d.n_layer)
arena = arena.to(dev)
peak, _ = bench.measured_peaks()
res = []
for item in spec.split(","):
    parts = item.split(":")
    kind, n = parts[0], int(parts[1])
    if kind not in ("A", "B", "C") or parts[2:] not in ([], ["unfused"]):
        raise SystemExit(f"bad configuration {item!r}: expected A|B|C:<utterances>[:unfused]")
    m = Transformer(cfg, arena, offsets, device=dev)
    m.setup_caches(2 * n, cfg.block_size, kv_dtype="bf16", tensor_core_path={"A": "", "B": "B", "C": "BC"}[kind],
                   unfused_sampler=parts[2:] == ["unfused"])
    lib, h, st = m._lib, m.handle, m._stream()
    for u in range(n):
        sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 9999, 5 + u)
        spk = synth.synthetic_speaker(seed=u).to(dev).reshape(-1).contiguous()
        _lib.check(lib.mvb_s1_set_speaker(h, u, spk.data_ptr(), st))
        _lib.check(lib.mvb_s1_begin(h, u, 100 + u, L_mid - 100, C.byref(sp), None, None, st))
    _lib.check(lib.mvb_s1_decode(h, n, 20, st))   # warm-up + graph capture
    torch.cuda.synchronize()
    reps = 160
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _lib.check(lib.mvb_s1_decode(h, n, reps, st))
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    by = bench.W_BYTES + n * bench.KV_BYTES_PER_POS * (L_mid + 1)
    r = {"cfg": item, "ms_per_step": round(ms, 4), "tok_per_s": round(n / ms * 1e3, 1), "GBps": round(by / ms / 1e6, 1),
         "roofline_frac": round(by / ms / 1e6 / peak, 3)}
    print(json.dumps(r), flush=True)
    res.append(r)
    m.close()
    del m
    torch.cuda.empty_cache()
