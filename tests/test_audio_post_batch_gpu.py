"""GPU: the batched on-device audio post (`mvb_audio_post_batch`, through `audio_out.wav_bytes_on_device_batch`) against
`mvb_audio_post` / `wav_bytes_on_device` on each signal alone, which run the same kernels over a group of one signal: no
signal of a batch may change another's result.

One mixed batch: a 60 s signal at 24 kHz, a 0.3 s tone, a signal with a NaN, an all-gated 5 Hz rumble, a signal below the
energy floor and one a sample short of a block, plus ordinary speech-like signals between them.  Every signal's PCM16, LKFS and
gain must be bit-identical to the single-signal call (NaN LKFS compared as NaN) -- so neither the NaN signal nor the silent
one changes any other signal -- and `wav_bytes_on_device_batch` must raise, for the first bad signal, what
`wav_bytes_on_device` raises for it, naming its index.  Invalid arguments return MVB_ERR_ARG (or MVB_ERR_UNSUPPORTED
for a signal over 15,996 blocks) before anything is written."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SR = 24000
DEV = "cuda"


def _signals():
    from mvb200 import synth
    t03 = np.arange(int(0.3 * SR)) / SR
    nan_sig = synth.synthetic_waveform(2.0, SR, seed=3).copy()
    nan_sig[777] = np.nan
    t = np.arange(3 * SR) / SR
    return {
        "speech 60 s": synth.synthetic_waveform(60.0, SR, seed=1),
        "tone 0.3 s": (0.5 * np.sin(2 * math.pi * 440 * t03)).astype(np.float32),
        "speech 2 s": synth.synthetic_waveform(2.0, SR, seed=2),
        "NaN sample": nan_sig,
        "5 Hz rumble": (0.01 * np.sin(2 * math.pi * 5 * t)).astype(np.float32),
        "below the floor": (1e-4 * np.random.default_rng(4).standard_normal(SR)).astype(np.float32),
        "one sample short of a block": synth.synthetic_waveform(1.0, SR, seed=5)[:int(0.4 * SR) - 1] * 3,
        "speech 5 s": synth.synthetic_waveform(5.0, SR, seed=6),
    }


def _solo(lib, L, w):
    n = w.numel()
    ws = torch.empty(lib.mvb_audio_post_workspace_bytes(n), dtype=torch.uint8, device=DEV)
    pcm = torch.empty(n, dtype=torch.int16, device=DEV)
    st = torch.empty(2, dtype=torch.float32, device=DEV)
    L.check(lib.mvb_audio_post(w.data_ptr(), n, SR, 14.0, 1, ws.data_ptr(), pcm.data_ptr(), None, st.data_ptr(),
                               C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return pcm.cpu(), st.cpu()


def _same_float(a, b):
    return (math.isnan(a) and math.isnan(b)) or a == b


def test_batch_bit_identical_to_solo():
    from mvb200 import _lib as L
    lib = L.load()
    sigs = _signals()
    wavs = [torch.from_numpy(v).to(DEV) for v in sigs.values()]
    lens = [w.numel() for w in wavs]
    total = sum(lens)
    ws = torch.empty(lib.mvb_audio_post_batch_workspace_bytes(len(wavs), total), dtype=torch.uint8, device=DEV)
    flat = torch.cat(wavs)
    pcm = torch.full((total,), -12345, dtype=torch.int16, device=DEV)
    stats = torch.full((len(wavs), 2), 7.0, device=DEV)
    L.check(lib.mvb_audio_post_batch(flat.data_ptr(), len(wavs), (C.c_int32 * len(wavs))(*lens), SR, 14.0, 1, ws.data_ptr(),
                                     len(wavs), total, pcm.data_ptr(), None, stats.data_ptr(),
                                     C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    pcm, stats = pcm.cpu(), stats.cpu()
    pos = 0
    for i, (label, w) in enumerate(zip(sigs, wavs)):
        sp, ss = _solo(lib, L, w)
        assert torch.equal(pcm[pos:pos + lens[i]], sp), f"{label}: PCM differs from the single-signal call"
        for k in range(2):
            assert _same_float(float(stats[i, k]), float(ss[k])), (label, k, float(stats[i, k]), float(ss[k]))
        print(f"{label}: LKFS {float(ss[0]):.3f}, gain {float(ss[1]):.4f}: bit-identical")
        pos += lens[i]


def test_wav_bytes_batch_equals_solo_and_raises_like_it():
    from mvb200 import audio_out as A
    sigs = _signals()
    wavs = {k: torch.from_numpy(v).to(DEV) for k, v in sigs.items()}
    solo, errors = {}, {}
    for k, w in wavs.items():
        try:
            solo[k] = A.wav_bytes_on_device(w, SR)
        except Exception as e:           # noqa: BLE001 -- the exception itself is what is compared
            errors[k] = e
    assert set(errors) == {"tone 0.3 s", "NaN sample", "5 Hz rumble", "one sample short of a block"}, errors
    good = [k for k in wavs if k not in errors]
    got = A.wav_bytes_on_device_batch([wavs[k] for k in good], SR)
    assert got == [solo[k] for k in good]
    keys = list(wavs)
    for k, err in errors.items():
        batch = [wavs[g] for g in good[:2]] + [wavs[k]] + [wavs[g] for g in good[2:]]
        with pytest.raises(type(err)) as ei:
            A.wav_bytes_on_device_batch(batch, SR)
        assert str(ei.value) == f"signal 2: {err}", (k, str(ei.value))
    # the whole mixed batch: the first bad signal in input order is reported
    first = next(i for i, k in enumerate(keys) if k in errors)
    with pytest.raises(type(errors[keys[first]]), match=f"^signal {first}: "):
        A.wav_bytes_on_device_batch(list(wavs.values()), SR)


def test_invalid_arguments():
    from mvb200 import _lib as L
    lib = L.load()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    x = torch.zeros(1 << 20, device=DEV)
    pcm = torch.full((1 << 20,), 99, dtype=torch.int16, device=DEV)
    ws = torch.empty(lib.mvb_audio_post_batch_workspace_bytes(4, 1 << 20), dtype=torch.uint8, device=DEV)
    assert lib.mvb_audio_post_batch_workspace_bytes(0, 100) == 0
    cases = [("n = 0", 0, [100], 4, 1 << 20, L.MVB_ERR_ARG), ("n > max_batch", 3, [100] * 3, 2, 1 << 20, L.MVB_ERR_ARG),
             ("empty signal", 2, [100, 0], 4, 1 << 20, L.MVB_ERR_ARG),
             ("sum > max_total_samples", 2, [600, 600], 4, 1000, L.MVB_ERR_ARG),
             ("over 15,996 blocks", 1, [2400 * 16000], 4, 1 << 26, L.MVB_ERR_UNSUPPORTED)]
    for label, n, lens, mb, mt, want in cases:
        rc = lib.mvb_audio_post_batch(x.data_ptr(), n, (C.c_int32 * len(lens))(*lens), SR, 14.0, 1, ws.data_ptr(), mb, mt,
                                      pcm.data_ptr(), None, None, st)
        assert rc == want, (label, rc)
    torch.cuda.synchronize()
    assert (pcm == 99).all(), "an invalid call wrote its output"
