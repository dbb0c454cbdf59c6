"""GPU: the batched speaker front-end through its C entry points: k_resample_poly (mvb_resample_batch), k_trim_rms +
k_trim_span (mvb_spk_trim_batch) and the segmented mel / LSTM / mean launches of mvb_spk_embed_batch.  u = 2^-23.

k_resample_poly  y[j] = sum_q h[r][q] x[m - q], a chain of at most P = ceil(n_taps / up) fmaf from 0 over fp32 taps
                 rounded once from the float64 design (x is fp32 and exact in both).  Against float64
                 scipy.signal.resample_poly on the same x:
                   |dy| <= (P + 1) u sum_q |h| |x|          (P roundings of the chain, one of the taps),
                 the gamma_P bound for the polyphase tap count; every check also asserts ||dy|| / ||y|| < 1e-6.
k_trim_*         rms = sqrtf(sum / 2048) with the 2048 squares summed by 64-term per-lane fmaf chains and a 5-step
                 butterfly (69 roundings on non-negative terms) and one sqrtf: |drms| / rms <= (69 / 2 + 1) u.  The
                 ratio to the loudest frame doubles that and adds one rounding (72 u), and the kernel compares it with
                 10^(-top_db / 20) rounded to fp32 (u more), which in dB is 20 / ln 10 = 8.69 dB per unit of relative
                 error: |d dB| <= 8.69 * 73 u = 634 u = 7.6e-5 dB.  Frames whose float64 dB lies
                 within TIE_DB = 1e-4 dB of -top_db may fall on either side; the device span must lie between the spans
                 the float64 host gives with those frames dropped and kept, and the number of such frames is printed.
mvb_spk_embed_batch  utterance i is bit-identical to mvb_spk_embed (SpeakerEncoder.embed_utterance) on it alone, partials
                 included; one ragged batch is compared with the float64 oracle at the E2E bound of
                 test_speaker_ops_gpu.

Sensitivity: the resampler without delay compensation and with a Hann window instead of Kaiser(5) puts elements over
the bound; the trim with >= instead of > disagrees with the device on an exact tie; concatenating the solo results
with two utterances of different length swapped differs from the batch."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
from scipy.signal import firwin, resample_poly

from test_speaker_frontend_cpu import RATES, poly_reference

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
SR = 16000
DEV = "cuda"
GUARD = 1024
TIE_DB = 1e-4
E2E = 5e-6


def _lib():
    from mvb200 import _lib as L
    return L, L.load()


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _i32(xs):
    return np.ascontiguousarray(np.asarray(xs, dtype=np.int32))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _guarded(n, dtype=torch.float32):
    fill = float("nan") if dtype == torch.float32 else -7
    buf = torch.full((2 * GUARD + n,), fill, dtype=dtype, device=DEV)
    return buf, buf[GUARD:GUARD + n]


def _check_guards(buf, n):
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + n:]).all(), "write outside the output"
    assert not torch.isnan(buf[GUARD:GUARD + n]).any(), "output not fully written"


def _resample_dev(xs, up, down, taps=None):
    """mvb_resample_batch over the list xs (fp32) -> (guarded buffer, packed output, output lengths)."""
    from mvb200.speaker_encoder import polyphase, resample_taps, resampled_length
    L, lib = _lib()
    if up == down:                                        # a copy: no filter
        h, d_taps = np.zeros(0), torch.zeros(1, device=DEV)
    else:
        h = resample_taps(up, down) if taps is None else taps
        d_taps = torch.from_numpy(polyphase(h, up).astype(np.float32)).to(DEV)
    x = torch.from_numpy(np.concatenate(xs).astype(np.float32)).to(DEV)
    n_out = [resampled_length(v.size, up, down) for v in xs]
    buf, out = _guarded(sum(n_out))
    L.check(lib.mvb_resample_batch(len(xs), x.data_ptr(), _p(_i32([v.size for v in xs])), up, down, d_taps.data_ptr(), h.size,
                                   out.data_ptr(), _st()))
    torch.cuda.synchronize()
    return buf, out, n_out


def _signal(n, seed):
    return (0.3 * np.random.default_rng(seed).standard_normal(n)).astype(np.float32)


def _lengths(up, down):
    return sorted({1, 2, max(1, down - 1), down, down + 1, max(1, up - 1), up + 1})


@pytest.mark.parametrize("sr_in,sr_out", RATES)
def test_resample_vs_float64_scipy(sr_in, sr_out):
    from mvb200.speaker_encoder import resample_ratio
    up, down = resample_ratio(sr_in, sr_out)
    P = -(-(20 * max(up, down) + 1) // up)
    worst = 0.0
    for n in _lengths(up, down) + [180 * sr_in]:
        x = _signal(n, n + sr_in)
        buf, out, (n_out,) = _resample_dev([x], up, down)
        _check_guards(buf, n_out)
        got = out.double().cpu().numpy()
        want = resample_poly(x.astype(np.float64), up, down)
        assert got.shape == want.shape
        if up == down:
            assert np.array_equal(got, want)
            continue
        _, a = poly_reference(x, up, down, with_abs=True)
        bound = (P + 1) * U * a
        err = np.abs(got - want)
        assert (err <= bound).all(), (n, int((err > bound).sum()), int(np.argmax(err - bound)))
        nw = np.linalg.norm(err) / max(np.linalg.norm(want), 1e-300)
        assert nw < 1e-6 or np.linalg.norm(want) == 0, (n, nw)
        worst = max(worst, float((err / np.maximum(bound, 1e-300)).max()))
    print(f"resample {sr_in} -> {sr_out} ({up}/{down}, {P} taps per phase): worst |err|/bound {worst:.2e}")


def test_resample_sensitivity():
    """No delay compensation, or a Hann window instead of Kaiser(5), must each put elements over the bound."""
    up, down = 160, 441
    P = -(-(20 * 441 + 1) // up)
    x = _signal(3 * 44100, 1)
    _, out, _ = _resample_dev([x], up, down)
    got = out.double().cpu().numpy()
    _, a = poly_reference(x, up, down, with_abs=True)
    bound = (P + 1) * U * a
    no_delay = poly_reference(x, up, down, delay=False)
    hann = poly_reference(x, up, down, taps=firwin(20 * 441 + 1, 1 / 441, window="hann") * up)
    for label, ref in (("no delay", no_delay), ("hann", hann)):
        over = int((np.abs(got - ref) > bound).sum())
        print(f"resample sensitivity {label}: {over} of {got.size} over the bound")
        assert over > 0, label


def test_resample_ragged_batch_is_bit_identical_to_solo():
    up, down = 160, 441
    rng = np.random.default_rng(7)
    lens = [1, 2, 440, 441, 442] + list(rng.integers(1, 3 * 44100, 26)) + [30 * 44100]
    xs = [_signal(int(n), i) for i, n in enumerate(lens)]
    buf, out, n_out = _resample_dev(xs, up, down)
    _check_guards(buf, sum(n_out))
    off = 0
    for x, n in zip(xs, n_out):
        sbuf, solo, _ = _resample_dev([x], up, down)
        _check_guards(sbuf, n)
        assert torch.equal(out[off:off + n], solo)
        off += n


# ---- trim ---------------------------------------------------------------------------------------------------------------
def _trim_dev(enc, xs, top_db=20.0):
    L, lib = _lib()
    x = torch.from_numpy(np.concatenate(xs).astype(np.float32)).to(DEV)
    spans = torch.full((len(xs), 2), -7, dtype=torch.int32, device=DEV)
    L.check(lib.mvb_spk_trim_batch(enc._h, len(xs), x.data_ptr(), _p(_i32([v.size for v in xs])), top_db,
                                   enc._batch_workspace().data_ptr(), enc.batch_max, enc.batch_samples, spans.data_ptr(), _st()))
    return spans.cpu().numpy()


def _host_span(y, top_db, shift):
    """trim_silence's span with the threshold moved by `shift` dB, or (0, 0)."""
    pad = np.pad(y.astype(np.float64), 1024)
    n = 1 + (pad.size - 2048) // 512
    idx = np.arange(2048)[None, :] + 512 * np.arange(n)[:, None]
    rms = np.sqrt(np.mean(pad[idx] ** 2, axis=1))
    ref = rms.max()
    if ref <= 0:
        return (0, 0), (0, 0), 0
    db = 20.0 * np.log10(np.maximum(rms, 1e-10) / ref)
    sure, maybe = np.nonzero(db > -top_db + shift)[0], np.nonzero(db > -top_db - shift)[0]
    span = lambda k: (int(k[0]) * 512, min(y.size, (int(k[-1]) + 1) * 512))
    return span(sure), span(maybe), int(((db > -top_db - shift) & (db <= -top_db + shift)).sum())


def _tone(n, lead, tail, seed):
    x = np.zeros(n, np.float32)
    t = np.arange(n - lead - tail)
    x[lead:n - tail] = (0.5 * np.sin(2 * np.pi * 220 * t / SR) * (1 + 0.3 * np.sin(t / 977.0))).astype(np.float32)
    return x + (1e-4 * np.random.default_rng(seed).standard_normal(n)).astype(np.float32) * (np.arange(n) % 3 == 0)


@pytest.fixture(scope="module")
def enc():
    from mvb200 import synth
    from mvb200.speaker_encoder import SpeakerEncoder
    e = SpeakerEncoder(model_state=synth.speaker_encoder_state_dict(3), device=DEV, verbose=False)
    yield e
    e.close()


def test_trim_vs_float64_host(enc):
    from mvb200 import synth
    from mvb200.speaker_encoder import trim_silence
    xs = [_tone(5 * SR, 20000, 15000, 1), _tone(3 * SR, 0, 0, 2), np.zeros(40000, np.float32), _tone(300, 50, 50, 3),
          _tone(511, 0, 100, 4), _tone(2048, 700, 0, 5), _tone(2049, 0, 0, 6), _signal(1, 7),
          synth.synthetic_waveform(180, SR, seed=9), _tone(10 * SR, 3 * SR, 4 * SR, 8)]
    got = _trim_dev(enc, xs)
    ties = 0
    for i, x in enumerate(xs):
        sure, maybe, t = _host_span(x, 20.0, TIE_DB)
        ties += t
        b, e = (int(v) for v in got[i])
        if sure == (0, 0):
            assert (b, e) == (0, 0), i
            assert trim_silence(x).size == 0
            continue
        assert maybe[0] <= b <= sure[0] and sure[1] <= e <= maybe[1], (i, (b, e), sure, maybe)
        if sure == maybe:
            assert np.array_equal(x[b:e], trim_silence(x)), i
    print(f"trim: {len(xs)} signals, {ties} frames within {TIE_DB} dB of the threshold")


def test_trim_strict_threshold_on_an_exact_tie(enc):
    """A quiet stretch at exactly 0.1 of the loud one's RMS sits at -20 dB exactly in float64, and its fp32 ratio equals
    the fp32 threshold 0.1f: `>` drops it (the device, the host), `>=` would keep it."""
    n_loud, n_quiet = 20 * 512, 20 * 512
    x = np.zeros(n_loud + n_quiet + 8 * 512, np.float32)
    x[:n_loud] = 0.625 * np.where(np.arange(n_loud) % 2, 1, -1)
    x[n_loud:n_loud + n_quiet] = 0.0625 * np.where(np.arange(n_quiet) % 2, 1, -1)
    from mvb200.speaker_encoder import trim_silence
    (b, e), = _trim_dev(enc, [x])
    host = trim_silence(x)
    assert (b, e) == (0, host.size)
    pad = np.pad(x.astype(np.float64), 1024)
    idx = np.arange(2048)[None, :] + 512 * np.arange(1 + x.size // 512)[:, None]
    rms = np.sqrt(np.mean(pad[idx] ** 2, axis=1))
    db = 20 * np.log10(np.maximum(rms, 1e-10) / rms.max())
    assert (db == -20.0).any()
    keep_ge = np.nonzero(db >= -20.0)[0]
    assert min(x.size, (keep_ge[-1] + 1) * 512) != e, "trim with >= agrees with the device"


# ---- batched embedding ----------------------------------------------------------------------------------------------------
def _speech(n, seed=9):
    from mvb200 import synth
    if n == 0:
        return np.zeros(0, np.float32)
    return synth.synthetic_waveform(n / SR + 1, SR, seed=seed)[:n]


def _ragged(n, seed):
    rng = np.random.default_rng(seed)
    lens = [1, 180 * SR, 25599, 25600, 25601][:n]
    lens += [int(v) for v in rng.integers(2, 2 * 30 * SR // max(n, 1), max(0, n - len(lens)))]
    return lens


@pytest.mark.parametrize("n", [1, 3, 8, 32])
def test_embed_batch_bit_identical_to_solo(enc, n):
    lens = _ragged(n, n)
    wavs = [_speech(m, seed=i) for i, m in enumerate(lens)]
    solo = [enc.embed_utterance(w, return_partials=True) for w in wavs]
    for order in (list(range(n)), list(range(n))[::-1]):
        batch = [wavs[i] for i in order]
        padded = [max(len(w), enc.compute_partial_slices(len(w), 1.3, 0.75)[0][-1].stop) for w in batch]
        assert len(enc._groups(padded)) == 1, "the batch must go through one call"
        e, p, _ = enc.embed_utterance_batch(batch, return_partials=True)
        for k, i in enumerate(order):
            assert np.array_equal(e[k], solo[i][0]), (n, k, lens[i])
            assert np.array_equal(p[k], solo[i][1]), (n, k, lens[i])
    if n >= 3:
        a, b = 0, 2                                       # lengths 1 and 25599: different window counts
        swapped = [solo[i][0] for i in range(n)]
        swapped[a], swapped[b] = swapped[b], swapped[a]
        e = enc.embed_utterance_batch(wavs)
        assert not np.array_equal(np.stack(swapped), e)


def test_embed_batch_vs_float64_oracle(enc):
    from mvb200 import synth
    from oracle import speaker_port as P
    o = P.SpeakerOracle(synth.speaker_encoder_state_dict(3), dtype=torch.float64)
    lens = [25600, int(6.4 * SR), 1, 30 * SR]
    wavs = [_speech(m, seed=i) for i, m in enumerate(lens)]
    e, p, _ = enc.embed_utterance_batch(wavs, return_partials=True)
    for i, w in enumerate(wavs):
        re, rp = o.embed_utterance(w)
        nw_e = float(np.linalg.norm(e[i] - re) / np.linalg.norm(re))
        nw_p = float(np.linalg.norm(p[i] - rp) / np.linalg.norm(rp))
        print(f"embed batch n={lens[i]}: normwise {nw_p:.2e} (partials), {nw_e:.2e} (embedding)")
        assert nw_e < E2E and nw_p < E2E


# ---- argument checks ------------------------------------------------------------------------------------------------------
def test_invalid_arguments_leave_outputs_untouched(enc):
    L, lib = _lib()
    ws = enc._batch_workspace()
    mb, mt = enc.batch_max, enc.batch_samples
    x = torch.from_numpy(_speech(40000)).to(DEV)
    from mvb200.speaker_encoder import polyphase, resample_taps
    taps = torch.from_numpy(polyphase(resample_taps(160, 441), 160).astype(np.float32)).to(DEV)
    out = torch.full((40000,), float("nan"), device=DEV)
    n1 = _i32([40000])
    for args, code in (((0, 160, 441, 8821), L.MVB_ERR_ARG), ((33, 160, 441, 8821), L.MVB_ERR_ARG),
                       ((1, 160, 441, 8820), L.MVB_ERR_ARG), ((1, 0, 441, 8821), L.MVB_ERR_ARG),
                       ((1, 1000, 1, 20001), L.MVB_ERR_UNSUPPORTED)):
        n, up, down, nt = args
        assert lib.mvb_resample_batch(n, x.data_ptr(), _p(n1), up, down, taps.data_ptr(), nt, out.data_ptr(), _st()) == code, args
    assert lib.mvb_resample_batch(1, x.data_ptr(), _p(_i32([0])), 160, 441, taps.data_ptr(), 8821, out.data_ptr(), _st()) == L.MVB_ERR_ARG
    spans = torch.full((2, 2), -7, dtype=torch.int32, device=DEV)
    for n, lens, db, cap in ((0, [1], 20.0, mb), (2, [1, 1], 20.0, 1), (1, [0], 20.0, mb), (1, [1], 0.0, mb),
                             (1, [1], float("nan"), mb), (1, [1], float("inf"), mb), (1, [mt + 1], 20.0, mb)):
        assert lib.mvb_spk_trim_batch(enc._h, n, x.data_ptr(), _p(_i32(lens)), db, ws.data_ptr(), cap, mt, spans.data_ptr(),
                                      _st()) == L.MVB_ERR_ARG, (n, lens, db, cap)
    assert lib.mvb_spk_trim_batch(enc._h, 1, x.data_ptr(), _p(_i32([10])), 20.0, ws.data_ptr(), 33, mt, spans.data_ptr(), _st()) == L.MVB_ERR_ARG
    assert lib.mvb_spk_trim_batch(enc._h, 1, x.data_ptr(), _p(_i32([10])), 20.0, None, mb, mt, spans.data_ptr(), _st()) == L.MVB_ERR_ARG
    emb = torch.full((2, 256), float("nan"), device=DEV)
    part = torch.full((4, 256), float("nan"), device=DEV)
    max_start = (enc.cfg.max_samples // 160) - 160
    cases = [
        (1, [0], [100], [0], [1], mb, mt),                  # fine (checked below)
        (0, [0], [100], [0], [1], mb, mt),                  # n < 1
        (2, [0, 0], [100, 100], [0, 0], [1, 1], 1, mt),     # n > max_batch
        (1, [-1], [100], [0], [1], mb, mt),                 # negative offset
        (1, [0], [-1], [0], [1], mb, mt),                   # negative length
        (1, [0], [100], [-1], [1], mb, mt),                 # negative start
        (1, [0], [100], [0], [0], mb, mt),                  # no window
        (1, [0], [enc.cfg.max_samples + 1], [0], [1], mb, mt),   # longer than max_samples
        (1, [0], [100], [max_start + 1], [1], mb, mt),      # padding past max_samples
        (1, [0], [100], [0], [1], mb, 1000),                # padded length past max_total_samples
        (1, [0], [100], [0], [1], 0, mt),                   # bad capacity
    ]
    for k, (n, off, nw, st, npart, cap, tot) in enumerate(cases):
        rc = lib.mvb_spk_embed_batch(enc._h, n, x.data_ptr(), _p(np.ascontiguousarray(off, np.int64)), _p(_i32(nw)), _p(_i32(st)),
                                     _p(_i32(npart)), ws.data_ptr(), cap, tot, emb.data_ptr(), part.data_ptr(), _st())
        assert rc == (L.MVB_OK if k == 0 else L.MVB_ERR_ARG), (k, rc)
        if k == 0:
            torch.cuda.synchronize()
            assert not torch.isnan(emb[0]).any() and torch.isnan(emb[1]).all() and torch.isnan(part[1:]).all()
            emb.fill_(float("nan"))
            part.fill_(float("nan"))
    assert lib.mvb_spk_embed_batch(enc._h, 1, x.data_ptr(), _p(np.zeros(1, np.int64)), _p(_i32([100])), _p(_i32([0])), _p(_i32([1])),
                                   None, mb, mt, emb.data_ptr(), None, _st()) == L.MVB_ERR_ARG
    torch.cuda.synchronize()
    assert torch.isnan(out).all() and (spans == -7).all() and torch.isnan(emb).all() and torch.isnan(part).all()
