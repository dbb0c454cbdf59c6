"""Speaker-reference front-end time on cuda:0: SpeakerEncoder.embed_files against embed_utterance_from_file, one process.

    python tools/speaker_batch_time.py [repeats] [out.json]

Workload: 8 references of 30 s at 44.1 kHz, PCM16 mono wavs written to a temporary directory (speech-like synthetic
signals with 0.7 s of leading and 1.1 s of trailing silence), random speaker-encoder weights.  Arms, after two warm-up
calls of each, alternating for `repeats` rounds (default 7):
  batch8   embed_files(8 paths): read + mix on the host, device resample / trim / embed;
  host8    8 x embed_utterance_from_file: read, float64 scipy resample and trim on the host, device embed per file;
  batch1 / host1   the same for the first file alone.
Each arm reports the host wall clock of the whole call (ending in a device synchronise) and the CUDA-event time from
its start to its end on the stream; medians over the rounds.  The card's name, power limit and SM clock are read in
the same call."""
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "metavoice-src_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

from mvb200 import synth  # noqa: E402
from mvb200.speaker_encoder import SpeakerEncoder  # noqa: E402
from test_speaker_frontend_gpu import _reference, _write_wav  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit, sm, sm_max = (v.strip() for v in q.split(","))
        return {"card": name, "power_limit_w": float(limit), "sm_clock_mhz": float(sm), "sm_clock_max_mhz": float(sm_max)}
    except Exception:   # noqa: BLE001 -- reported as unknown rather than guessed
        return {"card": torch.cuda.get_device_name(0), "power_limit_w": None}


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    a.record()
    fn()
    b.record()
    b.synchronize()
    return (time.perf_counter() - t0) * 1e3, a.elapsed_time(b)


def main():
    assert torch.cuda.is_available(), "speaker_batch_time needs a GPU"
    repeats = int(sys.argv[1]) if len(sys.argv) > 1 else 7
    enc = SpeakerEncoder(model_state=synth.speaker_encoder_state_dict(3), device="cuda", verbose=False)
    with tempfile.TemporaryDirectory() as d:
        paths = []
        for i in range(8):
            paths.append(os.path.join(d, f"ref{i}.wav"))
            _write_wav(paths[-1], _reference(44100, 30.0, seed=40 + i, stereo=False), 44100)
        arms = {"batch8": lambda: enc.embed_files(paths),
                "host8": lambda: [enc.embed_utterance_from_file(p, numpy=False) for p in paths],
                "batch1": lambda: enc.embed_files(paths[:1]),
                "host1": lambda: enc.embed_utterance_from_file(paths[0], numpy=False)}
        for fn in arms.values():
            fn()
            fn()
        wall = {k: [] for k in arms}
        dev = {k: [] for k in arms}
        for _ in range(repeats):
            for k, fn in arms.items():
                w, e = timed(fn)
                wall[k].append(w)
                dev[k].append(e)
        got = enc.embed_files(paths).cpu()
        want = torch.stack([torch.as_tensor(enc.embed_utterance_from_file(p, numpy=True)) for p in paths])
    out = {**card(), "repeats": repeats, "workload": "8 x 30 s PCM16 mono at 44.1 kHz", "arms": {},
           "max_normwise_batch_vs_host": float(((got - want).norm(dim=1) / want.norm(dim=1)).max())}
    for k in arms:
        out["arms"][k] = {"wall_ms_median": round(statistics.median(wall[k]), 2), "wall_ms_min": round(min(wall[k]), 2),
                          "wall_ms_max": round(max(wall[k]), 2), "event_ms_median": round(statistics.median(dev[k]), 2)}
    enc.close()
    print(json.dumps(out, indent=1))
    if len(sys.argv) > 2:
        with open(sys.argv[2], "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
