"""Batched synthesis against the per-utterance loop, one process, on cuda:0.

    python tools/batch_synth_time.py [repeats]

Three comparisons, 8 utterances each, the two arms alternating for `repeats` rounds (default 5) after a warm-up of both:
  decode  mvb_voc_decode_batch over 8 x 375 frames (5 s at 75 Hz) against 8 x mvb_voc_decode (CUDA events, random
          EnCodec weights from synth.encodec_model_and_state_dict);
  post    mvb_audio_post_batch over 8 x 5 s at 24 kHz against 8 x mvb_audio_post (CUDA events, signal generation excluded);
  synth   TTS.synthesise_batch over 8 texts against 8 x TTS.synthesise (host clock around calls that end in a device
          synchronise), on a synthetic snapshot: the 2-layer stage 1 (synth.TINY) and the full-size stage 2
          (synth.S2_FULL).  Each stage-1 request may generate up to 750 tokens (about 5 s of audio); the tiny random
          model decides where each utterance ends, so the seconds of audio produced are reported alongside.
Prints one JSON object with the median ms of each arm, the speed-ups, the card name and its power limit."""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "metavoice-src_b200"))
import torch  # noqa: E402

from mvb200 import _lib, synth  # noqa: E402

N, FRAMES, SR = 8, 375, 24000


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = (v.strip() for v in q.split(","))
        return name, float(limit)
    except Exception:   # noqa: BLE001 -- reported as unknown rather than guessed
        return torch.cuda.get_device_name(0), None


def events_ms(fn) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def wall_ms(fn) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def alternate(arms: dict, repeats: int, timer) -> dict:
    for f in arms.values():      # warm-up
        f()
    torch.cuda.synchronize()
    ts = {k: [] for k in arms}
    for _ in range(repeats):
        for k, f in arms.items():
            ts[k].append(timer(f))
    return {k: sorted(v)[len(v) // 2] for k, v in ts.items()} | {k + "_all": [round(x, 3) for x in v] for k, v in ts.items()}


def decode_arms():
    from mvb200.vocoder import EncodecDecodeEngine
    _, sd = synth.encodec_model_and_state_dict(0)
    e = EncodecDecodeEngine(sd, device="cuda:0", max_batch=N, max_total_frames=N * FRAMES)
    g = torch.Generator().manual_seed(0)
    codes = [torch.randint(0, 1024, (8, FRAMES), generator=g, dtype=torch.int32).cuda() for _ in range(N)]
    flat = torch.cat([c.reshape(-1) for c in codes])
    T = (C.c_int32 * N)(*[FRAMES] * N)
    out = torch.empty(N * FRAMES * e.upsample, device="cuda:0")
    st = e._st()

    def batched():
        _lib.check(e._lib.mvb_voc_decode_batch(e._h, N, flat.data_ptr(), T, e._bws.data_ptr(), N, N * FRAMES, out.data_ptr(), st))

    def solo():
        for i, c in enumerate(codes):
            _lib.check(e._lib.mvb_voc_decode(e._h, c.data_ptr(), FRAMES, out[i * FRAMES * e.upsample:].data_ptr(), st))

    solo()
    ref = out.clone()
    batched()
    assert torch.equal(out, ref), "decode_batch differs from the solo decodes"
    return {"decode_batch": batched, "decode_solo_x8": solo}, e


def post_arms():
    lib = _lib.load()
    n = 5 * SR
    wavs = torch.cat([torch.from_numpy(synth.synthetic_waveform(5.0, SR, seed=10 + i)) for i in range(N)]).cuda()
    pcm = torch.empty(N * n, dtype=torch.int16, device="cuda:0")
    stats = torch.empty(N, 2, device="cuda:0")
    bws = torch.empty(lib.mvb_audio_post_batch_workspace_bytes(N, N * n), dtype=torch.uint8, device="cuda:0")
    ws = torch.empty(lib.mvb_audio_post_workspace_bytes(n), dtype=torch.uint8, device="cuda:0")
    lens = (C.c_int32 * N)(*[n] * N)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def batched():
        _lib.check(lib.mvb_audio_post_batch(wavs.data_ptr(), N, lens, SR, 14.0, 1, bws.data_ptr(), N, N * n, pcm.data_ptr(), None,
                                            stats.data_ptr(), st))

    def solo():
        for i in range(N):
            _lib.check(lib.mvb_audio_post(wavs[i * n:].data_ptr(), n, SR, 14.0, 1, ws.data_ptr(), pcm[i * n:].data_ptr(), None,
                                          stats[i].data_ptr(), st))

    solo()
    ref = pcm.clone()
    batched()
    assert torch.equal(pcm, ref), "batched post differs from the solo posts"
    return {"post_batch": batched, "post_solo_x8": solo}


def synth_arms(tmp):
    from mvb200.fast_inference import TTS
    snap = os.path.join(tmp, "snapshot")
    os.makedirs(snap)
    torch.save(synth.stage1_checkpoint(synth.TINY, 0), os.path.join(snap, "first_stage.pt"))
    torch.save(synth.stage2_checkpoint(synth.S2_FULL, 1), os.path.join(snap, "second_stage.pt"))
    _, enc = synth.encodec_model_and_state_dict(0)
    spk = os.path.join(snap, "spk.pt")
    torch.save(synth.synthetic_speaker(), spk)
    tts = TTS(snap, output_dir=os.path.join(tmp, "out"), encodec_state_dict=enc, device="cuda:0", max_utts=N)
    tts.model._cfg.max_new = 750
    texts = [f"Utterance number {i}: a sentence of about five seconds for the batch timing." for i in range(N)]
    audio = {}

    def batched():
        ps = tts.synthesise_batch(texts, [spk] * N, seed=7)
        audio["batch"] = sum(os.path.getsize(p) - 44 for p in ps if p) / 2 / SR

    def solo():
        secs = 0.0
        for t in texts:
            try:
                secs += (os.path.getsize(tts.synthesise(t, spk)) - 44) / 2 / SR
            except Exception as e:   # noqa: BLE001 -- an utterance under 400 ms: synthesise raises, the batch returns None
                print(f"synthesise: {e}")
        audio["solo"] = secs

    return {"synthesise_batch": batched, "synthesise_x8": solo}, audio


def main():
    repeats = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    assert torch.cuda.is_available(), "needs a GPU"
    name, limit = card()
    res = {"gpu": name, "power_limit_w": limit, "utterances": N, "repeats": repeats}
    arms, _keep = decode_arms()
    res.update(alternate(arms, repeats, events_ms))
    res.update(alternate(post_arms(), repeats, events_ms))
    with tempfile.TemporaryDirectory() as tmp:
        arms, audio = synth_arms(tmp)
        res.update(alternate(arms, max(2, repeats // 2), wall_ms))
        res["audio_s_batch"], res["audio_s_solo"] = round(audio["batch"], 2), round(audio["solo"], 2)
    for a, b in (("decode_batch", "decode_solo_x8"), ("post_batch", "post_solo_x8"), ("synthesise_batch", "synthesise_x8")):
        res[a.split("_")[0] + "_speedup"] = round(res[b] / res[a], 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
