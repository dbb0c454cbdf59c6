"""CPU: the host side of the batched speaker front-end (SpeakerEncoder.embed_files).

The resampling filter is designed once on the host in float64 (speaker_encoder.resample_taps) and the device only
applies it, so the host design must be scipy's own: resample_poly with these taps passed as its window gives bit for
bit what resample_poly designs itself.  `poly_reference` restates the device's output formula (mvb_resample_batch in
include/mvb200.h) in float64; it matches scipy to rounding here and is the reference the GPU tests compare against.
The polyphase reordering must round-trip, and the batch workspace size must follow its documented layout at the
capacity limits and refuse values outside them."""
import ctypes as C

import numpy as np
import pytest
from scipy.signal import resample_poly

from mvb200.speaker_encoder import polyphase, resample_ratio, resample_taps, resampled_length

RATES = [(8000, 16000), (11025, 16000), (16000, 16000), (22050, 16000), (24000, 16000), (44100, 16000), (48000, 16000),
         (96000, 16000), (16000, 24000), (44100, 24000), (48000, 24000)]


def poly_reference(x, up, down, taps=None, delay=True, with_abs=False):
    """float64 y[j] = sum_q h[r + q up] x[m - q], t = j down + (len(h) - 1) / 2, r = t mod up, m = t div up (zero outside
    the signal); delay=False drops the (len(h) - 1) / 2.  With with_abs also sum_q |h| |x| per output."""
    h = resample_taps(up, down) if taps is None else np.asarray(taps, np.float64)
    x = np.asarray(x, np.float64)
    hp = polyphase(h, up)
    P = hp.shape[1]
    t = np.arange(resampled_length(x.size, up, down), dtype=np.int64) * down + ((h.size - 1) // 2 if delay else 0)
    r, m = t % up, t // up
    y, a = np.zeros(t.size), np.zeros(t.size)
    for q in range(P):
        idx = m - q
        ok = (idx >= 0) & (idx < x.size)
        v = hp[r[ok], q] * x[idx[ok]]
        y[ok] += v
        a[ok] += np.abs(v)
    return (y, a) if with_abs else y


@pytest.mark.parametrize("sr_in,sr_out", RATES)
def test_host_taps_are_scipys_filter(sr_in, sr_out):
    up, down = resample_ratio(sr_in, sr_out)
    x = np.random.default_rng(sr_in).standard_normal(3 * down + 7)
    want = resample_poly(x, up, down)
    if up == down:
        assert np.array_equal(want, x)
        return
    h = resample_taps(up, down)
    assert h.size == 20 * max(up, down) + 1
    assert np.array_equal(resample_poly(x, up, down, window=h / up), want)
    ref = poly_reference(x, up, down)
    assert ref.shape == want.shape
    assert np.abs(ref - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


def test_taps_at_the_standard_rates():
    """11.025 / 22.05 / 44.1 kHz -> 16 kHz need 12,801 / 8,821 / 8,821 taps, all inside MVB_RESAMPLE_MAX_TAPS."""
    from mvb200 import _lib
    for sr, n in ((11025, 12801), (22050, 8821), (44100, 8821)):
        assert resample_taps(*resample_ratio(sr, 16000)).size == n <= _lib.RESAMPLE_MAX_TAPS
    for sr in (8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000):
        up, down = resample_ratio(sr, 16000)
        assert up == down or 20 * max(up, down) + 1 <= _lib.RESAMPLE_MAX_TAPS, sr


@pytest.mark.parametrize("up,down", [(2, 1), (640, 441), (160, 441), (1, 6), (3, 2), (7, 5)])
def test_polyphase_round_trips(up, down):
    h = resample_taps(up, down)
    hp = polyphase(h, up)
    P = -(-h.size // up)
    assert hp.shape == (up, P)
    for r in range(up):
        for q in range(P):
            assert hp[r, q] == (h[r + q * up] if r + q * up < h.size else 0.0)
    assert np.array_equal(hp.T.reshape(-1)[:h.size], h)
    assert not hp.T.reshape(-1)[h.size:].any()


def _cfg(max_samples=180 * 16000 + 160 * 160):
    from mvb200 import _lib
    return _lib.SpkConfig(40, 256, 3, 256, 400, 160, 160, max_samples)


def _layout_bytes(max_batch, max_total, n_mels=40, hop=160):
    a = lambda b: (b + 255) // 256 * 256
    frames = max_batch + max_total // hop
    return a(frames * n_mels * 4) + a(frames * 4) + a(frames * 256 * 4) + a((max_batch + max_total // 512) * 4)


def test_batch_workspace_bytes_at_the_limits():
    from mvb200 import _lib
    lib = _lib.load()
    cfg = _cfg()
    for mb, mt in ((1, 1), (32, 1), (1, 2 ** 31 - 1), (32, 2 ** 31 - 1), (8, 8 * 30 * 16000), (32, 2 * cfg.max_samples)):
        assert lib.mvb_spk_batch_workspace_bytes(C.byref(cfg), mb, mt) == _layout_bytes(mb, mt), (mb, mt)
    for mb, mt in ((0, 16000), (33, 16000), (-1, 16000), (1, 0), (1, -1), (1, 2 ** 31), (32, 2 ** 40)):
        assert lib.mvb_spk_batch_workspace_bytes(C.byref(cfg), mb, mt) == 0, (mb, mt)
        assert b"speaker batch" in lib.mvb_last_error()
    bad = _cfg()
    bad.hidden = 128
    assert lib.mvb_spk_batch_workspace_bytes(C.byref(bad), 1, 16000) == 0


def test_resample_rejects_before_touching_the_device():
    """Argument errors need no GPU: they are returned before any launch, with null device pointers never dereferenced."""
    from mvb200 import _lib
    lib = _lib.load()
    n = (C.c_int32 * 1)(100)
    dummy = C.c_void_p(16)
    assert lib.mvb_resample_batch(1, dummy, n, 640, 441, dummy, 12800, dummy, None) == _lib.MVB_ERR_ARG
    assert lib.mvb_resample_batch(1, dummy, n, 820, 1, dummy, 16401, dummy, None) == _lib.MVB_ERR_UNSUPPORTED
    assert b"16384" in lib.mvb_last_error()
    assert lib.mvb_resample_batch(0, dummy, n, 2, 1, dummy, 41, dummy, None) == _lib.MVB_ERR_ARG
    assert lib.mvb_resample_batch(33, dummy, n, 2, 1, dummy, 41, dummy, None) == _lib.MVB_ERR_ARG
    assert lib.mvb_resample_batch(1, dummy, n, 0, 1, dummy, 41, dummy, None) == _lib.MVB_ERR_ARG
    assert lib.mvb_resample_batch(1, None, n, 2, 1, dummy, 41, dummy, None) == _lib.MVB_ERR_ARG
    zero = (C.c_int32 * 1)(0)
    assert lib.mvb_resample_batch(1, dummy, zero, 2, 1, dummy, 41, dummy, None) == _lib.MVB_ERR_ARG
