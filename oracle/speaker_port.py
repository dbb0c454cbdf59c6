"""ORACLE (test infrastructure, never the product path): CPU restatement of the speaker-encoder path (SURVEY.md row N3)

    fam/quantiser/audio/speaker_encoder/audio.py:10-22      wav_to_mel_spectrogram  (librosa.feature.melspectrogram)
    fam/quantiser/audio/speaker_encoder/model.py:50-53      forward: 3-layer LSTM -> linear -> ReLU -> L2 norm
    fam/quantiser/audio/speaker_encoder/model.py:55-79      compute_partial_slices
    fam/quantiser/audio/speaker_encoder/model.py:81-103     embed_utterance: partial windows, mean, L2 norm

Pinning: the network, the slicing and the averaging are pinned against the reference's own ``SpeakerEncoder`` class
(oracle/make_golden_speaker.py -> tests/golden/speaker.npz).  The mel front-end lives in third-party ``librosa``
(requirements.txt pins 0.10.1), absent from the image: ``mel_spectrogram`` below restates its published algorithm
(centered STFT with zero padding, periodic Hann window, power spectrum, Slaney mel filterbank with Slaney
normalisation) -- PARITY UNPINNED for that function only.
"""
from __future__ import annotations

import numpy as np
import torch

SR, N_FFT, HOP, N_MELS, PARTIAL_FRAMES = 16000, 400, 160, 40, 160


def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-10) / min_log_hz) / logstep, f / f_sp)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_filterbank(sr=SR, n_fft=N_FFT, n_mels=N_MELS) -> np.ndarray:
    """librosa.filters.mel(sr, n_fft, n_mels, fmin=0, fmax=sr/2, htk=False, norm='slaney') -> [n_mels, 1 + n_fft/2] fp32."""
    fftfreqs = np.linspace(0, sr / 2, 1 + n_fft // 2)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(0.0), _hz_to_mel(sr / 2), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    w = np.zeros((n_mels, 1 + n_fft // 2))
    for i in range(n_mels):
        lower, upper = -ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]
        w[i] = np.maximum(0, np.minimum(lower, upper))
    w *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return w.astype(np.float32)


def hann_periodic(n=N_FFT) -> np.ndarray:
    return (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n) / n)).astype(np.float32)


def mel_spectrogram(wav: np.ndarray, dtype=np.float32) -> np.ndarray:
    """audio.py:10-22: power mel spectrogram (NOT log), [n_frames, 40], n_frames = 1 + len(wav) // 160.  float32: the
    window and the windowed frames in fp32, as librosa computes them; float64: the float64 periodic Hann window, no
    rounding before the filterbank (whose fp32 values are librosa's)."""
    y = np.pad(np.asarray(wav, dtype=np.float32), N_FFT // 2)          # center=True, pad_mode="constant" (librosa 0.10)
    n_frames = 1 + (len(y) - N_FFT) // HOP
    idx = np.arange(N_FFT)[None, :] + HOP * np.arange(n_frames)[:, None]
    if dtype == np.float64:
        frames = y[idx].astype(np.float64) * (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N_FFT) / N_FFT))[None, :]
    else:
        frames = y[idx] * hann_periodic()[None, :]
    spec = np.abs(np.fft.rfft(frames.astype(np.float64), axis=1)) ** 2
    return (spec @ mel_filterbank().astype(np.float64).T).astype(dtype)


def compute_partial_slices(n_samples: int, rate: float = 1.3, min_coverage: float = 0.75):
    """model.py:55-79 (same arithmetic; returns (wav_slices, mel_slices) as lists of (start, stop))."""
    spf = int(SR * 10 / 1000)
    n_frames = int(np.ceil((n_samples + 1) / spf))
    frame_step = int(np.round((SR / rate) / spf))
    wav_s, mel_s = [], []
    steps = max(1, n_frames - PARTIAL_FRAMES + frame_step + 1)
    for i in range(0, steps, frame_step):
        mel_s.append((i, i + PARTIAL_FRAMES))
        wav_s.append((i * spf, (i + PARTIAL_FRAMES) * spf))
    last = wav_s[-1]
    coverage = (n_samples - last[0]) / (last[1] - last[0])
    if coverage < min_coverage and len(mel_s) > 1:
        mel_s, wav_s = mel_s[:-1], wav_s[:-1]
    return wav_s, mel_s


class SpeakerOracle:
    """dtype: the arithmetic of the network, the average and (float64) the mel front-end; the weights are the
    checkpoint's fp32 values either way."""

    def __init__(self, model_state: dict, dtype: torch.dtype = torch.float32):
        self.dtype = dtype
        g = lambda k: model_state[k].float().to(dtype)
        self.layers = [dict(w_ih=g(f"lstm.weight_ih_l{l}"), w_hh=g(f"lstm.weight_hh_l{l}"), b=g(f"lstm.bias_ih_l{l}") + g(f"lstm.bias_hh_l{l}"))
                       for l in range(3)]
        self.lw, self.lb = g("linear.weight"), g("linear.bias")

    @torch.no_grad()
    def forward(self, mels: torch.Tensor) -> torch.Tensor:
        """mels [P, T, 40] -> L2-normalised embeddings [P, 256] (model.py:50-53; torch.nn.LSTM gate order i, f, g, o)."""
        x = mels.to(self.dtype)
        for L in self.layers:
            P, T, _ = x.shape
            H = L["w_hh"].shape[1]
            h, c = torch.zeros(P, H, dtype=self.dtype), torch.zeros(P, H, dtype=self.dtype)
            ys = []
            for t in range(T):
                gts = x[:, t] @ L["w_ih"].t() + h @ L["w_hh"].t() + L["b"]
                i, f, g, o = gts.chunk(4, dim=-1)
                c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
                h = torch.sigmoid(o) * torch.tanh(c)
                ys.append(h)
            x = torch.stack(ys, dim=1)
        e = torch.relu(x[:, -1] @ self.lw.t() + self.lb)
        return e / torch.norm(e, dim=1, keepdim=True)

    def embed_utterance(self, wav: np.ndarray, rate: float = 1.3, min_coverage: float = 0.75, mel_fn=None):
        wav_s, mel_s = compute_partial_slices(len(wav), rate, min_coverage)
        if wav_s[-1][1] >= len(wav):
            wav = np.pad(wav, (0, wav_s[-1][1] - len(wav)), "constant")
        mel = mel_fn(wav) if mel_fn is not None else mel_spectrogram(wav, np.float64 if self.dtype == torch.float64 else np.float32)
        mels = torch.from_numpy(np.array([mel[a:b] for a, b in mel_s]))
        pe = self.forward(mels)
        raw = pe.mean(dim=0)
        return (raw / torch.linalg.norm(raw, 2)).numpy(), pe.numpy()
