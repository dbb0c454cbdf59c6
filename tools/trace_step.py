"""GPU debug: per-phase time breakdown of the persistent decode kernel (clock64 stamps of every CTA), and how long the
producer warp waited for a free ring stage in each phase of its byte schedule.
Writes gpurun_out/trace_<n>.npy and prints medians per event interval."""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "metavoice-src_b200"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from mvb200 import _lib, synth  # noqa: E402
from mvb200.fast_model import ModelArgs, Transformer, pack_arena  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1
L_mid = int(sys.argv[2]) if len(sys.argv) > 2 else 423
dev = torch.device("cuda:0"); torch.cuda.set_device(dev)
d = synth.FULL
cfg = ModelArgs.from_name("metavoice-1B")
arena, offsets = pack_arena(synth.stage1_state_dict(d, 0), d.n_layer)
m = Transformer(cfg, arena.to(dev), offsets, device=dev)
m.setup_caches(2 * n, cfg.block_size, kv_dtype="bf16", trace=True)
lib, h, st = m._lib, m.handle, m._stream()
for u in range(n):
    sp = _lib.Sampling(3.0, 1.0, 0.95, 0, 9999, 5 + u)
    spk = synth.synthetic_speaker(seed=u).to(dev).reshape(-1).contiguous()
    _lib.check(lib.mvb_s1_set_speaker(h, u, spk.data_ptr(), st))
    _lib.check(lib.mvb_s1_begin(h, u, 100 + u, L_mid - 30, C.byref(sp), None, None, st))
N_STEPS, N_STALL = 30, 6
_lib.check(lib.mvb_s1_decode(h, n, N_STEPS, st))
torch.cuda.synchronize()
G = torch.cuda.get_device_properties(dev).multi_processor_count   # one CTA per SM
buf = np.zeros((G, 512), dtype=np.int64)
got = lib.mvb_s1_trace_fetch(h, buf.ctypes.data_as(C.c_void_p), G, st)
stall = buf[:, 512 - N_STALL:]   # the producer stall record: the tail of every CTA's row (saved with the stamps below)
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
np.save(os.path.join(ROOT, "gpurun_out", f"trace_{n}.npy"), buf)
t = buf[:, :2 + 14 * 24 + 4].astype(np.float64)
t = (t - t[:, :1]) / 1.9e3   # ~us at 1.9 GHz
names = ["qkv.wait", "qkv.stage", "qkv.epi", "att.wait", "att.work", "o.wait", "o.stage", "o.epi", "w13.wait", "w13.stage",
         "w13.epi", "w2.wait", "w2.stage", "w2.epi"]
dt = np.diff(t, axis=1)          # interval ending at event i+1
print("total us (median over CTAs):", np.median(t[:, -1]))
per = dt[:, 1:1 + 14 * 24].reshape(G, 24, 14)   # skip start->embed
for j, nm in enumerate(names):
    v = per[:, 2:, j]
    print(f"{nm:10s} median {np.median(v):7.2f}  mean {v.mean():7.2f}  p90 {np.percentile(v, 90):7.2f}  max {v.max():7.2f}")
print("per-layer sum (median CTA):", np.median(per[:, 2:, :].sum(axis=2)))
# producer blocked on a full ring (waiting for b_empty), summed over the launch; per layer and position (all 24 layers)
# for the layer phases, per position for the head
s = stall.astype(np.float64) / 1.9e3
s[:, :5] /= N_STEPS * d.n_layer
s[:, 5] /= N_STEPS
print("producer blocked, us per layer (head: per position):")
for j, nm in enumerate(["qkv", "kv", "wo", "w13", "w2", "head"]):
    v = s[:, j]
    print(f"{'blk.' + nm:10s} median {np.median(v):7.2f}  mean {v.mean():7.2f}  p90 {np.percentile(v, 90):7.2f}  max {v.max():7.2f}")
print("producer blocked per layer (median CTA):", np.median(s[:, :5].sum(axis=1)))
