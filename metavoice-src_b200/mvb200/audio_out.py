"""Host-side audio post-processing of the reference's `_save_audio` (fam/llm/decoders.py:40-47): it calls
`audiocraft.data.audio.audio_write(name, wav, 24000, strategy="loudness", loudness_compressor=True)`.

audiocraft==1.2.0 is not in this image, so this restates the published algorithm of
`audiocraft/data/audio_utils.py::normalize_loudness` / `normalize_audio` / `_clip_wav` and
`audiocraft/data/audio.py::audio_write` (parity unpinned: nothing in the reference's tests covers it); the loudness
meter itself is torchaudio's ITU-R BS.1770 implementation -- the very function audiocraft calls -- which IS installed.
SURVEY.md §8 row a18 keeps this step on the host (N2 moves it on device).
"""
from __future__ import annotations

import struct

import numpy as np
import torch

LOUDNESS_HEADROOM_DB = 14.0      # audio_write default `loudness_headroom_db`
ENERGY_FLOOR = 2e-3              # normalize_loudness default `energy_floor`


def normalize_loudness(wav: torch.Tensor, sample_rate: int, loudness_headroom_db: float = LOUDNESS_HEADROOM_DB,
                       loudness_compressor: bool = False, energy_floor: float = ENERGY_FLOOR) -> torch.Tensor:
    """wav [C, T] fp32 -> same shape, integrated loudness moved to -`loudness_headroom_db` LUFS, optional tanh
    compressor.  Signals below the energy floor are returned unchanged (as audiocraft does)."""
    import torchaudio
    energy = wav.pow(2).mean().sqrt().item()
    if energy < energy_floor:
        return wav
    input_loudness_db = torchaudio.functional.loudness(wav, sample_rate).item()
    delta_loudness = -loudness_headroom_db - input_loudness_db
    gain = 10.0 ** (delta_loudness / 20.0)
    output = gain * wav
    if loudness_compressor:
        output = torch.tanh(output)
    assert output.isfinite().all(), (input_loudness_db, energy)
    return output


def audio_write_wav(path_stem: str, wav: torch.Tensor, sample_rate: int, strategy: str = "loudness",
                    loudness_compressor: bool = True) -> str:
    """`audio_write(..., format="wav")`: normalise ([C, T] or [T] fp32 on any device), clip to [-1, 1], write PCM16.
    Returns the path (stem + ".wav")."""
    assert wav.dtype.is_floating_point, "wav is not floating point"
    wav = wav.detach().to("cpu", torch.float32)
    if wav.dim() == 1:
        wav = wav[None]
    elif wav.dim() > 2:
        raise ValueError("Input wav should be at most 2 dimension.")
    assert wav.isfinite().all()
    if strategy == "loudness":
        wav = normalize_loudness(wav, sample_rate, LOUDNESS_HEADROOM_DB, loudness_compressor)
    elif strategy != "clip":
        raise ValueError(f"unsupported normalisation strategy {strategy!r}")
    wav = wav.clamp(-1.0, 1.0)                                              # _clip_wav
    path = path_stem + ".wav"
    # interleaved little-endian PCM16 (torchaudio.save(..., encoding="PCM_S", bits_per_sample=16))
    pcm = (wav.t().contiguous().numpy() * 32767.0).round().astype("<i2").tobytes()
    ch = wav.shape[0]
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 36 + len(pcm)) + b"WAVEfmt "
                + struct.pack("<IHHIIHH", 16, 1, ch, sample_rate, sample_rate * 2 * ch, 2 * ch, 16))
        f.write(b"data" + struct.pack("<I", len(pcm)) + pcm)
    return path


def read_wav_pcm16(path: str):
    """Minimal reader for the files written above (tests)."""
    b = open(path, "rb").read()
    assert b[:4] == b"RIFF" and b[8:12] == b"WAVE"
    ch, sr = struct.unpack("<H", b[22:24])[0], struct.unpack("<I", b[24:28])[0]
    n = struct.unpack("<I", b[40:44])[0]
    x = np.frombuffer(b[44:44 + n], dtype="<i2").reshape(-1, ch).T.astype(np.float32) / 32767.0
    return torch.from_numpy(x.copy()), sr


# ---- on-device variant (SURVEY.md row N2): loudness meter, gain, compressor and PCM16 conversion in libmvb200 -----------
def wav_bytes_on_device(wav: torch.Tensor, sample_rate: int, loudness_headroom_db: float = LOUDNESS_HEADROOM_DB,
                        loudness_compressor: bool = True, return_stats: bool = False):
    """Device fp32 mono waveform [T] (or [1, T]) -> the bytes of the wav FILE `_save_audio` would have written
    (decoders.py:40-47): only 2 bytes per sample cross the PCIe bus, no temp file (serving.py:96-97 re-reads the file it
    just wrote; a server can return these bytes directly)."""
    assert wav.is_cuda, "wav_bytes_on_device expects a device tensor (use audio_write_wav for host tensors)"
    (blob,), (lk,), (gain,) = _post_batch([wav], sample_rate, loudness_headroom_db, loudness_compressor)
    if isinstance(blob, Exception):
        raise blob
    return (blob, lk, gain) if return_stats else blob


def _undefined_meter_error(w: torch.Tensor, sample_rate: int) -> Exception:
    """The meter is undefined (NaN): what audio_write_wav raises for the same input.  The device only reports NaN for
    non-finite samples, signals above the floor shorter than one 400 ms block (torchaudio's `loudness` raises
    RuntimeError), and signals whose blocks are all gated (NaN loudness: the finiteness assert)."""
    n = w.numel()
    if not bool(w.isfinite().all()):
        return AssertionError("wav contains non-finite samples")
    if n < round(0.4 * sample_rate):
        return RuntimeError(f"loudness: {n} samples are shorter than one 400 ms gating block at {sample_rate} Hz")
    return AssertionError(f"loudness is undefined: every 400 ms block of the {n}-sample signal is below -70 LKFS")


def _wav_header(n_bytes: int, sample_rate: int) -> bytes:
    return (b"RIFF" + struct.pack("<I", 36 + n_bytes) + b"WAVEfmt " +
            struct.pack("<IHHIIHH", 16, 1, 1, sample_rate, sample_rate * 2, 2, 16) + b"data" + struct.pack("<I", n_bytes))


_POST_BATCH_WS = {}


def _post_batch(wavs, sample_rate: int, loudness_headroom_db: float, loudness_compressor: bool):
    """The batched on-device post of every signal: ([wav file bytes, or the exception wav_bytes_on_device raises for that
    signal], LKFS [n], gain [n])."""
    import ctypes as C
    from . import _lib
    from ._engine import current_stream
    lib = _lib.load()
    ws_ = [w.detach().reshape(-1).to(torch.float32) for w in wavs]
    dev = ws_[0].device
    assert all(w.is_cuda and w.device == dev for w in ws_), "wav_bytes_on_device_batch expects device tensors on one device"
    lens = [w.numel() for w in ws_]
    n, total = len(ws_), sum(lens)
    cap = _POST_BATCH_WS.get(dev)
    if cap is None or cap[0] < n or cap[1] < total:
        nb, ns = max(n, 32, cap[0] if cap else 0), max(total, 1 << 20, cap[1] if cap else 0)
        cap = (nb, ns, torch.empty(lib.mvb_audio_post_batch_workspace_bytes(nb, ns), dtype=torch.uint8, device=dev))
        _POST_BATCH_WS[dev] = cap
    flat = torch.cat(ws_) if n > 1 else ws_[0].contiguous()   # one signal (wav_bytes_on_device): no device copy
    pcm = torch.empty(total, dtype=torch.int16, device=dev)
    stats = torch.empty(n, 2, dtype=torch.float32, device=dev)
    _lib.check(lib.mvb_audio_post_batch(flat.data_ptr(), n, (C.c_int32 * n)(*lens), int(sample_rate), float(loudness_headroom_db),
                                        int(bool(loudness_compressor)), cap[2].data_ptr(), cap[0], cap[1], pcm.data_ptr(), None,
                                        stats.data_ptr(), current_stream(dev)))
    stats = stats.cpu().tolist()
    pcm = pcm.cpu().numpy().astype("<i2", copy=False)
    out, pos = [], 0
    for (lk, _), w, k in zip(stats, ws_, lens):
        if lk != lk:
            out.append(_undefined_meter_error(w, sample_rate))
        else:
            body = pcm[pos:pos + k].tobytes()
            out.append(_wav_header(len(body), sample_rate) + body)
        pos += k
    return out, [s[0] for s in stats], [s[1] for s in stats]


def wav_bytes_on_device_batch(wavs, sample_rate: int, loudness_headroom_db: float = LOUDNESS_HEADROOM_DB,
                              loudness_compressor: bool = True):
    """``[wav_bytes_on_device(w, sample_rate) for w in wavs]`` with one launch set for the whole list (the signals are
    concatenated on the device).  Signal i's bytes equal ``wav_bytes_on_device(wavs[i], sample_rate)``; for a signal
    whose loudness is undefined, this raises what ``wav_bytes_on_device`` raises for it, naming the signal's index (the
    first such signal)."""
    if not wavs:
        return []
    out, _, _ = _post_batch(wavs, sample_rate, loudness_headroom_db, loudness_compressor)
    for i, r in enumerate(out):
        if isinstance(r, Exception):
            raise type(r)(f"signal {i}: {r}")
    return out
