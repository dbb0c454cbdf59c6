"""EnCodec encode throughput on cuda:0 (EncodecEncodeEngine, csrc/encoder.cu), one process.

    python tools/encode_time.py [repeats] [out.json]

Arms, after a warm-up of each, alternating for `repeats` rounds (default 7), CUDA events around each arm:
  batch8   encode_batch over 8 x 10 s at 24 kHz (one launch set);
  solo8    8 x encode of the same 8 x 10 s;
  solo30   encode of 1 x 30 s.
Reports the median ms and audio-seconds per second of each arm, the fp32 FLOP/s from `flops(L)` (counted from shapes)
as a share of the H100 SXM data-sheet 67 TFLOP/s FP32 figure, and the reference arm: transformers
EncodecModel.encode(bandwidth=6.0) of 1 x 10 s on the host cores (fp32, wall clock, median of 3).  Random EnCodec
weights from synth.encodec_model_and_state_dict.  The card's name and power limit are read in the same call."""
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "metavoice-src_b200"))
import torch  # noqa: E402

from mvb200 import synth  # noqa: E402
from mvb200.vocoder import EncodecEncodeEngine  # noqa: E402

SR, FP32_DATASHEET = 24000, 67e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = (v.strip() for v in q.split(","))
        return name, float(limit)
    except Exception:   # noqa: BLE001 -- reported as unknown rather than guessed
        return torch.cuda.get_device_name(0), None


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    assert torch.cuda.is_available(), "encode_time needs a GPU"
    repeats = int(sys.argv[1]) if len(sys.argv) > 1 else 7
    m, sd = synth.encodec_model_and_state_dict(seed=0)
    eng = EncodecEncodeEngine(sd, device="cuda", max_frames=2250, max_batch=8, max_total_frames=8 * 750)
    ten = [torch.from_numpy(synth.synthetic_waveform(10.0, SR, seed=i)).cuda() for i in range(8)]
    thirty = torch.from_numpy(synth.synthetic_waveform(30.0, SR, seed=9)).cuda()
    arms = {"batch8": (lambda: eng.encode_batch(ten), 80.0, sum(eng.flops(x.numel()) for x in ten)),
            "solo8": (lambda: [eng.encode(x) for x in ten], 80.0, sum(eng.flops(x.numel()) for x in ten)),
            "solo30": (lambda: eng.encode(thirty), 30.0, eng.flops(thirty.numel()))}
    for fn, _, _ in arms.values():
        fn()
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    for _ in range(repeats):
        for k, (fn, _, _) in arms.items():
            ms[k].append(timed(fn))
    name, limit = card()
    out = {"card": name, "power_limit_w": limit, "repeats": repeats, "arms": {}}
    for k, (_, secs, flops) in arms.items():
        med = statistics.median(ms[k])
        out["arms"][k] = {"median_ms": round(med, 3), "min_ms": round(min(ms[k]), 3), "max_ms": round(max(ms[k]), 3),
                          "audio_s_per_s": round(secs / (med / 1e3), 1), "fp32_tflops": round(flops / (med / 1e3) / 1e12, 3),
                          "share_of_fp32_datasheet": round(flops / (med / 1e3) / FP32_DATASHEET, 4)}
    x = ten[0].cpu().view(1, 1, -1)
    host = []
    with torch.no_grad():
        for _ in range(3):
            t0 = time.perf_counter()
            m.encode(x, bandwidth=6.0)
            host.append(time.perf_counter() - t0)
    h = statistics.median(host)
    out["transformers_cpu_10s"] = {"median_ms": round(h * 1e3, 1), "audio_s_per_s": round(10.0 / h, 2),
                                   "threads": torch.get_num_threads()}
    print(json.dumps(out))
    if len(sys.argv) > 2:
        with open(sys.argv[2], "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
