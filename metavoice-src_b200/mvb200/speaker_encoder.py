"""Host-side mirror of ``fam/quantiser/audio/speaker_encoder/model.py::SpeakerEncoder`` over libmvb200 (SURVEY.md row N3).

Same constructor keywords, ``embed_utterance`` / ``embed_utterance_from_file`` / ``compute_partial_slices`` contract and
``speaker_encoder.pt`` layout (``{"model_state": {lstm.*, linear.*}}``, model.py:45-46).  The mel front-end, the 3-layer
LSTM, the projection and the partial-window averaging run on the device (csrc/speaker.cu); reading / resampling /
trimming the reference file stays on the host in ``embed_utterance_from_file`` (the reference uses librosa for those:
librosa.load at 16 kHz + librosa.effects.trim(top_db=20), model.py:112-113 -- restated here with scipy's polyphase
resampler, not pinned).  ``embed_files`` runs the whole front-end for a batch of files on the device: the same polyphase
filter in fp32 (``mvb_resample_batch``), the same trim (``mvb_spk_trim_batch``) and one embedding launch set
(``mvb_spk_embed_batch``).
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import struct
from math import gcd
from typing import Dict, List, Optional, Sequence, Union

import numpy as np
import torch

from . import _lib
from ._engine import Engine, pack_arena_bytes, split_runs

mel_window_length = 25
mel_window_step = 10
mel_n_channels = 40
sampling_rate = 16000
partials_n_frames = 160
model_hidden_size = 256
model_embedding_size = 256
model_num_layers = 3


def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    lin, log0, step = 200.0 / 3, 1000.0, np.log(6.4) / 27.0
    return np.where(f >= log0, log0 / lin + np.log(np.maximum(f, 1e-10) / log0) / step, f / lin)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    lin, log0, step = 200.0 / 3, 1000.0, np.log(6.4) / 27.0
    return np.where(m >= log0 / lin, log0 * np.exp(step * (m - log0 / lin)), lin * m)


def slaney_mel_filterbank(sr: int, n_fft: int, n_mels: int) -> np.ndarray:
    """Triangular filters on the Slaney mel scale with area normalisation ([n_mels, n_fft/2 + 1], fp32): what
    librosa.filters.mel(sr, n_fft, n_mels) returns with its defaults (fmin 0, fmax sr/2, htk False, norm "slaney")."""
    freqs = np.linspace(0, sr / 2, 1 + n_fft // 2)
    edges = _mel_to_hz(np.linspace(_hz_to_mel(0.0), _hz_to_mel(sr / 2), n_mels + 2))
    width = np.diff(edges)
    fb = np.zeros((n_mels, freqs.size))
    for i in range(n_mels):
        up = (freqs - edges[i]) / width[i]
        down = (edges[i + 2] - freqs) / width[i + 1]
        fb[i] = np.clip(np.minimum(up, down), 0, None) * (2.0 / (edges[i + 2] - edges[i]))
    return fb.astype(np.float32)


def read_wav(path: str, mono: bool = True):
    """PCM16 / PCM32 / float32 RIFF wav -> (float32 mono [-1, 1], sample_rate); with ``mono=False`` the channels are kept,
    [channels, n].  Other containers (mp3, flac) need a decoder that is not part of this engine."""
    with open(path, "rb") as f:
        data = f.read()
    if data[:4] != b"RIFF" or data[8:12] != b"WAVE":
        raise NotImplementedError(f"{path}: only RIFF/WAVE speaker references are decoded here (mp3/flac need ffmpeg or librosa)")
    pos, fmt, pcm = 12, None, None
    while pos + 8 <= len(data):
        cid, size = data[pos:pos + 4], struct.unpack("<I", data[pos + 4:pos + 8])[0]
        body = data[pos + 8:pos + 8 + size]
        if cid == b"fmt ":
            fmt = struct.unpack("<HHIIHH", body[:16])
        elif cid == b"data":
            pcm = body
        pos += 8 + size + (size & 1)
    if fmt is None or pcm is None:
        raise ValueError(f"{path}: malformed wav")
    tag, ch, sr, _, _, bits = fmt
    if tag == 1 and bits == 16:
        x = np.frombuffer(pcm, dtype="<i2").astype(np.float32) / 32768.0
    elif tag == 1 and bits == 32:
        x = np.frombuffer(pcm, dtype="<i4").astype(np.float32) / 2147483648.0
    elif tag == 3 and bits == 32:
        x = np.frombuffer(pcm, dtype="<f4").astype(np.float32)
    else:
        raise NotImplementedError(f"{path}: wav format tag {tag} / {bits} bit")
    if not mono:
        return np.ascontiguousarray(x.reshape(-1, ch).T), sr
    if ch > 1:
        x = x.reshape(-1, ch).mean(axis=1)          # librosa.load(mono=True)
    return x, sr


def resample(x: np.ndarray, sr_in: int, sr_out: int) -> np.ndarray:
    if sr_in == sr_out:
        return x.astype(np.float32)
    from math import gcd
    from scipy.signal import resample_poly
    g = gcd(sr_in, sr_out)
    return resample_poly(x.astype(np.float64), sr_out // g, sr_in // g).astype(np.float32)


def resample_ratio(sr_in: int, sr_out: int):
    """(up, down) = (sr_out, sr_in) reduced by their gcd, as resample_poly reduces them."""
    g = gcd(sr_in, sr_out)
    return sr_out // g, sr_in // g


def resample_taps(up: int, down: int) -> np.ndarray:
    """float64 filter of scipy.signal.resample_poly(x, up, down) with its defaults: a Kaiser(5) windowed sinc of
    20 max(up, down) + 1 taps at cutoff 1 / max(up, down), times up."""
    from scipy.signal import firwin
    m = max(up, down)
    return firwin(20 * m + 1, 1.0 / m, window=("kaiser", 5.0)) * up


def polyphase(h: np.ndarray, up: int) -> np.ndarray:
    """h -> [up, ceil(len(h) / up)] with row r = h[r], h[r + up], ... (zero past the end): mvb_resample_batch's order."""
    P = -(-h.size // up)
    return np.concatenate([h, np.zeros(up * P - h.size, h.dtype)]).reshape(P, up).T.copy()


def resampled_length(n: int, up: int, down: int) -> int:
    return -(-n * up // down)


def trim_silence(y: np.ndarray, top_db: float = 20.0, frame_length: int = 2048, hop_length: int = 512) -> np.ndarray:
    """librosa.effects.trim(y, top_db): keep the span between the first and last frame whose RMS is within top_db of the
    loudest frame (centered frames, zero padded)."""
    if y.size == 0:
        return y
    pad = np.pad(y.astype(np.float64), frame_length // 2)
    n = 1 + (pad.size - frame_length) // hop_length
    idx = np.arange(frame_length)[None, :] + hop_length * np.arange(n)[:, None]
    rms = np.sqrt(np.mean(pad[idx] ** 2, axis=1))
    ref = rms.max()
    if ref <= 0:
        return y[:0]
    db = 20.0 * np.log10(np.maximum(rms, 1e-10) / ref)
    keep = np.nonzero(db > -top_db)[0]
    if keep.size == 0:
        return y[:0]
    return y[keep[0] * hop_length:min(y.size, (keep[-1] + 1) * hop_length)]


class SpeakerEncoder(Engine):
    """model.py:21-117 with the arithmetic in libmvb200."""

    def __init__(self, weights_fpath: Optional[str] = None, device: Optional[Union[str, torch.device]] = None, verbose: bool = True,
                 eval: bool = False, model_state: Optional[Dict[str, torch.Tensor]] = None, max_seconds: float = 180.0):
        if device is None:
            device = "cuda"
        if model_state is None:
            model_state = torch.load(weights_fpath, map_location="cpu", weights_only=False)["model_state"]
        g = lambda k: model_state[k].detach().float().contiguous()
        tensors = []
        for l in range(model_num_layers):
            tensors += [g(f"lstm.weight_ih_l{l}"), g(f"lstm.weight_hh_l{l}"), g(f"lstm.bias_ih_l{l}") + g(f"lstm.bias_hh_l{l}")]
        n_fft = int(sampling_rate * mel_window_length / 1000)
        hop = int(sampling_rate * mel_window_step / 1000)
        i = np.arange(n_fft)
        tensors += [g("linear.weight"), g("linear.bias"),
                    torch.from_numpy(slaney_mel_filterbank(sampling_rate, n_fft, mel_n_channels)),
                    torch.from_numpy((0.5 - 0.5 * np.cos(2 * np.pi * i / n_fft)).astype(np.float32)),     # periodic Hann
                    torch.from_numpy(np.cos(2 * np.pi * i / n_fft).astype(np.float32)),
                    torch.from_numpy((-np.sin(2 * np.pi * i / n_fft)).astype(np.float32))]
        super().__init__(device, *pack_arena_bytes(tensors))
        # embed_utterance pads the waveform to the end of its last partial window, up to one window past the input: the
        # workspace holds max_seconds of input plus that window
        self.max_input_samples = int(max_seconds * sampling_rate)
        cfg = _lib.SpkConfig(mel_n_channels, model_hidden_size, model_num_layers, model_embedding_size, n_fft, hop,
                             partials_n_frames, self.max_input_samples + partials_n_frames * hop)
        self.cfg = cfg
        self._create(self._lib.mvb_spk_create, self._lib.mvb_spk_destroy, cfg, self._lib.mvb_spk_workspace_bytes)
        # batch front-end: filters per (up, down) on the device, and a workspace for MVB_SPK_MAX_BATCH utterances of up
        # to twice the longest single one, allocated on first use
        self._taps: Dict[tuple, torch.Tensor] = {}
        self.batch_max, self.batch_samples = _lib.SPK_MAX_BATCH, 2 * cfg.max_samples
        self._batch_ws: Optional[torch.Tensor] = None
        if verbose:
            print(f"Loaded the speaker embedding model on {self.device.type}.")

    @staticmethod
    def compute_partial_slices(n_samples: int, rate, min_coverage):
        """model.py:55-79: windows of 160 mel frames every round(16000 / rate / 160) frames; the last one is dropped when
        it covers less than ``min_coverage`` of real audio."""
        spf = int(sampling_rate * mel_window_step / 1000)
        n_frames = int(np.ceil((n_samples + 1) / spf))
        step = int(np.round((sampling_rate / rate) / spf))
        starts = list(range(0, max(1, n_frames - partials_n_frames + step + 1), step))
        mel_slices = [slice(i, i + partials_n_frames) for i in starts]
        wav_slices = [slice(i * spf, (i + partials_n_frames) * spf) for i in starts]
        last = wav_slices[-1]
        if (n_samples - last.start) / (last.stop - last.start) < min_coverage and len(mel_slices) > 1:
            mel_slices, wav_slices = mel_slices[:-1], wav_slices[:-1]
        return wav_slices, mel_slices

    @torch.no_grad()
    def wav_to_mel_spectrogram(self, wav: np.ndarray) -> torch.Tensor:
        """audio.py:10-22 on the device: fp32 [n_frames, 40]."""
        w = torch.from_numpy(np.ascontiguousarray(wav, dtype=np.float32)).to(self.device)
        mel = torch.empty((1 + w.numel() // self.cfg.hop, mel_n_channels), dtype=torch.float32, device=self.device)
        _lib.check(self._lib.mvb_spk_mel(self._h, w.data_ptr(), w.numel(), mel.data_ptr(), self._st()))
        return mel

    @torch.no_grad()
    def embed_utterance(self, wav: np.ndarray, return_partials=False, rate=1.3, min_coverage=0.75, numpy: bool = True):
        if len(wav) > self.max_input_samples:
            raise ValueError(f"speaker reference longer than {self.max_input_samples / sampling_rate:g} s")
        wav_slices, mel_slices = self.compute_partial_slices(len(wav), rate, min_coverage)
        max_wave_length = wav_slices[-1].stop
        if max_wave_length >= len(wav):
            wav = np.pad(wav, (0, max_wave_length - len(wav)), "constant")
        w = torch.from_numpy(np.ascontiguousarray(wav, dtype=np.float32)).to(self.device)
        starts = np.asarray([s.start for s in mel_slices], dtype=np.int32)
        embed = torch.empty(model_embedding_size, dtype=torch.float32, device=self.device)
        partials = torch.empty((len(starts), model_embedding_size), dtype=torch.float32, device=self.device)
        _lib.check(self._lib.mvb_spk_embed(self._h, w.data_ptr(), w.numel(), starts.ctypes.data_as(C.c_void_p), len(starts),
                                           embed.data_ptr(), partials.data_ptr(), self._st()))
        if numpy:
            embed_o, partials_o = embed.cpu().numpy(), partials.cpu().numpy()
        else:
            embed_o, partials_o = embed, partials
        if return_partials:
            return embed_o, partials_o, wav_slices
        return embed_o

    def _batch_workspace(self) -> torch.Tensor:
        if self._batch_ws is None:
            self._batch_ws = self._batch_workspace_of(
                self._lib.mvb_spk_batch_workspace_bytes(C.byref(self.cfg), self.batch_max, self.batch_samples), zeroed=False)
        return self._batch_ws

    def _groups(self, lengths: Sequence[int]) -> List[range]:
        """Consecutive runs of indices that fit one batch call: at most batch_max of them, batch_samples in all."""
        return split_runs(lengths, self.batch_max, self.batch_samples)

    def _embed_device(self, buf: torch.Tensor, offs: Sequence[int], lens: Sequence[int], rate, min_coverage):
        """Utterance i = the lens[i] 16 kHz samples of the device buffer buf at offs[i] -> embeddings [n, 256] and
        partials [sum windows, 256] on the device, and each utterance's wav slices."""
        for n in lens:
            if n > self.max_input_samples:
                raise ValueError(f"speaker reference longer than {self.max_input_samples / sampling_rate:g} s")
        plans = [self.compute_partial_slices(n, rate, min_coverage) for n in lens]
        padded = [max(n, ws[-1].stop) for n, (ws, _) in zip(lens, plans)]
        n_win = [len(ms) for _, ms in plans]
        first_win = np.concatenate([[0], np.cumsum(n_win)]).astype(np.int64)
        embeds = torch.empty((len(lens), model_embedding_size), dtype=torch.float32, device=self.device)
        partials = torch.empty((int(first_win[-1]), model_embedding_size), dtype=torch.float32, device=self.device)
        ws = self._batch_workspace()
        for g in self._groups(padded):
            starts = np.ascontiguousarray(np.concatenate([[s.start for s in plans[i][1]] for i in g]), dtype=np.int32)
            off = np.ascontiguousarray([offs[i] for i in g], dtype=np.int64)
            nw = np.ascontiguousarray([lens[i] for i in g], dtype=np.int32)
            npart = np.ascontiguousarray([n_win[i] for i in g], dtype=np.int32)
            ptr = lambda a: a.ctypes.data_as(C.c_void_p)
            _lib.check(self._lib.mvb_spk_embed_batch(
                self._h, len(g), buf.data_ptr(), ptr(off), ptr(nw), ptr(starts), ptr(npart), ws.data_ptr(), self.batch_max,
                self.batch_samples, embeds[g[0]].data_ptr(), partials[int(first_win[g[0]])].data_ptr(), self._st()))
        return embeds, partials, first_win, [ws_ for ws_, _ in plans]

    @torch.no_grad()
    def embed_utterance_batch(self, wavs: Sequence[np.ndarray], rate=1.3, min_coverage=0.75, return_partials=False):
        """embed_utterance over a list of 16 kHz waveforms: fp32 [n, 256], row i bit-identical to embed_utterance(wavs[i]);
        with return_partials also each utterance's partial embeddings and wav slices."""
        lens = [len(w) for w in wavs]
        host = np.concatenate([np.asarray(w, dtype=np.float32).reshape(-1) for w in wavs] + [np.zeros(1, np.float32)])
        buf = torch.from_numpy(host).to(self.device)
        offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).tolist()
        embeds, partials, first, slices = self._embed_device(buf, offs, lens, rate, min_coverage)
        embeds = embeds.cpu().numpy()
        if not return_partials:
            return embeds
        partials = partials.cpu().numpy()
        return embeds, [partials[first[i]:first[i + 1]] for i in range(len(lens))], slices

    def _resample_filter(self, up: int, down: int) -> torch.Tensor:
        if (up, down) not in self._taps:
            self._taps[(up, down)] = torch.from_numpy(polyphase(resample_taps(up, down), up).astype(np.float32)).to(self.device)
        return self._taps[(up, down)]

    @torch.no_grad()
    def embed_files(self, paths: Sequence[str], min_seconds: float = 30.0) -> torch.Tensor:
        """embed_utterance_from_file for a list of RIFF/WAVE files with the front-end on the device: each file is read and
        mixed to mono on the host, resampled to 16 kHz (one launch per input rate and 32 files), trimmed and embedded in
        batches.  Returns fp32 [n, 256] on the device in input order.  A file shorter than ``min_seconds`` (the 30 s of
        check_audio_file), at a rate whose resampling filter exceeds MVB_RESAMPLE_MAX_TAPS, or longer than max_seconds
        once resampled (before trimming) raises an error that names it, before anything runs on the device."""
        sigs = []
        for p in paths:
            x, sr = read_wav(p)
            if x.size / sr < min_seconds:
                raise Exception(f"{p}: The audio file is too short. Please provide an audio file that is at least "
                                f"{min_seconds} seconds long to proceed.")
            up, down = resample_ratio(sr, sampling_rate)
            if up != down and 20 * max(up, down) + 1 > _lib.RESAMPLE_MAX_TAPS:
                raise ValueError(f"{p}: resampling {sr} Hz to {sampling_rate} Hz ({up}/{down}) needs a filter longer than "
                                 f"{_lib.RESAMPLE_MAX_TAPS} taps")
            n16 = resampled_length(x.size, up, down)
            if n16 > self.max_input_samples:
                raise ValueError(f"{p}: speaker reference longer than {self.max_input_samples / sampling_rate:g} s")
            sigs.append((x, up, down, n16))
        if not sigs:
            return torch.empty((0, model_embedding_size), dtype=torch.float32, device=self.device)
        # the 16 kHz buffer holds the files grouped by rate, so that each rate's outputs are packed
        order = sorted(range(len(sigs)), key=lambda i: (sigs[i][1], sigs[i][2]))
        lens = [sigs[i][3] for i in order]
        offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64).tolist()
        buf = torch.empty(sum(lens), dtype=torch.float32, device=self.device)
        k = 0
        while k < len(order):
            _, up, down, _ = sigs[order[k]]
            e = k
            while e < len(order) and sigs[order[e]][1:3] == (up, down):
                e += 1
            host = np.concatenate([sigs[i][0] for i in order[k:e]])
            if up == down:
                buf[offs[k]:offs[k] + host.size].copy_(torch.from_numpy(host))
            else:
                x = torch.from_numpy(host).to(self.device)
                taps = self._resample_filter(up, down)
                n_in = [sigs[i][0].size for i in order[k:e]]
                x_off = np.concatenate([[0], np.cumsum(n_in)]).astype(np.int64)
                for c in range(0, e - k, self.batch_max):
                    chunk = np.ascontiguousarray(n_in[c:c + self.batch_max], dtype=np.int32)
                    _lib.check(self._lib.mvb_resample_batch(
                        len(chunk), x[int(x_off[c]):].data_ptr(), chunk.ctypes.data_as(C.c_void_p), up, down, taps.data_ptr(),
                        20 * max(up, down) + 1, buf[offs[k + c]:].data_ptr(), self._st()))
            k = e
        spans = torch.empty((len(lens), 2), dtype=torch.int32, device=self.device)
        ws = self._batch_workspace()
        for g in self._groups(lens):
            n = np.ascontiguousarray([lens[i] for i in g], dtype=np.int32)
            _lib.check(self._lib.mvb_spk_trim_batch(self._h, len(g), buf[offs[g[0]]:].data_ptr(), n.ctypes.data_as(C.c_void_p),
                                                    20.0, ws.data_ptr(), self.batch_max, self.batch_samples,
                                                    spans[g[0]].data_ptr(), self._st()))
        spans = spans.cpu().numpy()                           # one copy: compute_partial_slices needs the trimmed lengths
        embeds, _, _, _ = self._embed_device(buf, [o + int(b) for o, (b, _) in zip(offs, spans)],
                                             [int(e - b) for b, e in spans], 1.3, 0.75)
        out = torch.empty_like(embeds)
        out[torch.as_tensor(order, device=self.device)] = embeds
        return out

    def embed_utterance_from_file(self, fpath: str, numpy: bool) -> torch.Tensor:
        wav, sr = read_wav(fpath)                             # librosa.load(fpath, sr=16000)
        wav = trim_silence(resample(wav, sr, sampling_rate), top_db=20)
        return self.embed_utterance(wav, numpy=numpy)


def check_audio_file(path: str, threshold_s: float = 30.0):
    """fam/llm/utils.py:55-70: the speaker reference must hold at least 30 s of audio."""
    wav, sr = read_wav(path)
    if wav.size / sr < threshold_s:
        raise Exception(f"The audio file is too short. Please provide an audio file that is at least {threshold_s} seconds long to proceed.")


def _embedding_cache_path(local_file_path: str) -> str:
    name = "embedding_" + hashlib.md5(local_file_path.encode("utf-8")).hexdigest() + ".pt"
    os.makedirs(os.path.expanduser("~/.cache/fam/"), exist_ok=True)
    return os.path.expanduser(f"~/.cache/fam/{name}")


def get_cached_embedding(local_file_path: str, spkemb_model: SpeakerEncoder) -> torch.Tensor:
    """fam/llm/inference.py:419-435: disk cache ~/.cache/fam/embedding_<md5(path)>.pt keyed by the path string."""
    if not os.path.exists(local_file_path):
        raise FileNotFoundError(f"File {local_file_path} not found!")
    cache_path = _embedding_cache_path(local_file_path)
    if not os.path.exists(cache_path):
        spk_emb = spkemb_model.embed_utterance_from_file(local_file_path, numpy=False).unsqueeze(0).cpu()
        torch.save(spk_emb, cache_path)
    else:
        spk_emb = torch.load(cache_path, map_location="cpu")
    return spk_emb


def get_cached_embeddings(paths: Sequence[str], spkemb_model: SpeakerEncoder) -> torch.Tensor:
    """get_cached_embedding for a list of files -> fp32 [n, 256] on the CPU in input order, with the same cache files:
    hits are read from disk, and every miss is embedded in one SpeakerEncoder.embed_files call and written back."""
    for p in paths:
        if not os.path.exists(p):
            raise FileNotFoundError(f"File {p} not found!")
    out: Dict[str, torch.Tensor] = {}
    misses = []
    for p in paths:
        if p in out or p in misses:
            continue
        cache_path = _embedding_cache_path(p)
        if os.path.exists(cache_path):
            out[p] = torch.load(cache_path, map_location="cpu").reshape(1, -1)
        else:
            misses.append(p)
    if misses:
        embeds = spkemb_model.embed_files(misses).cpu()
        for p, e in zip(misses, embeds):
            out[p] = e.unsqueeze(0).clone()
            torch.save(out[p], _embedding_cache_path(p))
    return torch.cat([out[p] for p in paths]).float() if paths else torch.empty((0, model_embedding_size))
