"""GPU: the whole EnCodec encoder (`EncodecEncodeEngine`, `mvb_enc_encode` / `mvb_enc_encode_batch`, `get_tokens`).

* Embeddings against the float64 oracle (test_encodec_encoder_cpu.EncodecEncodeOracle, pinned there to transformers):
  normwise 1e-4 and elementwise 1e-3 of the largest reference magnitude, at lengths from one sample (every level
  zero-extended) to 30 s.  (The CPU fp32 transformers encoder is within 5.0e-7 of float64 normwise.)
* Codes against transformers EncodecModel.encode(x, bandwidth=6.0) in fp32: identical, except (codebook, frame) choices
  where the float64 oracle's own best and second-best scores are within 1e-4 relative (the embedding tolerance): from
  such a choice on, the frame is not compared further; the number of these frames is reported.
* encode_batch at B = 1, 3, 8 and 32 with ragged L_i (1 sample, lengths off the 320-sample grid, 1 s) in two orders:
  bit-identical to encode of each alone; the raw call on NaN-filled, guarded outputs writes every segment and nothing
  else; a batch over capacity is split; every invalid argument returns MVB_ERR_ARG with the outputs untouched.
* get_tokens on written 24 kHz PCM16 mono and stereo files equals encode of the same samples (stereo: the first channel).
* Codes from encode_batch go to EncodecDecodeEngine.decode_batch unchanged and give F_i 320 samples each."""
import ctypes as C
import os
import struct

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
LENS = (1, 319, 321, 641, 7, 24000, 4001, 1917)
MAX_TOTAL = 1024
GUARD = 1024


@pytest.fixture(scope="module")
def setup():
    from mvb200 import synth
    from mvb200.vocoder import EncodecEncodeEngine
    m, sd = synth.encodec_model_and_state_dict(seed=0)
    e = EncodecEncodeEngine(sd, device=DEV, max_frames=2250, max_batch=32, max_total_frames=MAX_TOTAL)
    yield e, m, sd
    e.close()


def _wav(L, seed):
    from mvb200 import synth
    return torch.from_numpy(synth.synthetic_waveform(L / 24000 + 0.01, 24000, seed=seed)[:L].copy())


def test_embeddings_vs_float64_oracle(setup):
    from test_encodec_encoder_cpu import EncodecEncodeOracle
    e, _, sd = setup
    o = EncodecEncodeOracle(sd, n_q=8, device=DEV)
    for L in (1, 2, 7, 40, 319, 320, 321, 1920, 1921, 24000, 720000):
        x = _wav(L, seed=L % 97)
        got = e.embed(x).double()
        ref = o.embed(x.double().to(DEV).view(1, 1, L))[0]
        assert got.shape == ref.shape == (128, -(-L // 320))
        err = (got - ref).abs()
        nw = float(err.norm() / ref.norm())
        el = float(err.max() / ref.abs().max())
        print(f"embed L={L}: normwise {nw:.2e}, max |err| / max |ref| {el:.2e}")
        assert nw < 1e-4 and el < 1e-3


def test_codes_vs_transformers_fp32(setup):
    from test_encodec_encoder_cpu import EncodecEncodeOracle
    e, m, sd = setup
    o = EncodecEncodeOracle(sd, n_q=8, device=DEV)
    m = m.float()
    for L in (1, 321, 1917, 24000, 120000):
        x = _wav(L, seed=3 + L % 11)
        got = e.encode(x).long().cpu()
        with torch.no_grad():
            ref = m.encode(x.view(1, 1, L), bandwidth=6.0).audio_codes[0, 0]
        steps = o.quantize(o.embed(x.double().to(DEV).view(1, 1, L))[0])
        live = torch.ones(got.shape[1], dtype=torch.bool)
        near = 0
        for q, (_, top2) in enumerate(steps):
            rel = ((top2[:, 1] - top2[:, 0]) / top2[:, 0].abs().clamp_min(1e-30)).cpu()
            close = live & (rel < 1e-4)
            differ = live & ~close & (got[q] != ref[q])
            assert not differ.any(), f"L={L} q={q}: {int(differ.sum())} codes differ at a clear float64 decision"
            near += int(close.sum())
            live &= ~close
        print(f"codes L={L}: identical to transformers fp32 outside {near} near-tie frames of {got.shape[1]}")


def _lens(B, reverse):
    seq = LENS[::-1] if reverse else LENS
    return [seq[i % len(seq)] for i in range(B)]


def _raw(e, wavs, n=None, lens=None, max_batch=32, max_total=MAX_TOTAL, emb=True):
    """The C batch entry point on NaN-filled (codes: -1) guarded outputs: (rc, codes buffer, embedding buffer, sizes)."""
    lens = lens or [int(w.numel()) for w in wavs]
    n = len(lens) if n is None else n
    Fs = [-(-L // 320) for L in lens]
    nc, ne = 8 * sum(Fs), 128 * sum(Fs)
    cbuf = torch.full((2 * GUARD + nc,), -1, dtype=torch.int32, device=DEV)
    ebuf = torch.full((2 * GUARD + ne,), float("nan"), device=DEV)
    flat = torch.cat([w.reshape(-1) for w in wavs]).to(DEV) if wavs else torch.zeros(1, device=DEV)
    Lc = (C.c_int32 * max(len(lens), 1))(*lens)
    rc = e._lib.mvb_enc_encode_batch(e._h, n, flat.data_ptr(), Lc, e._bws.data_ptr(), max_batch, max_total,
                                     cbuf[GUARD:].data_ptr(), ebuf[GUARD:].data_ptr() if emb else None, e._st())
    torch.cuda.synchronize()
    return rc, cbuf, ebuf, nc, ne, Fs


@pytest.mark.parametrize("B", [1, 3, 8, 32])
@pytest.mark.parametrize("reverse", [False, True])
def test_batch_bit_identical_to_solo(setup, B, reverse):
    from mvb200 import _lib as L
    e, _, _ = setup
    lens = _lens(B, reverse)
    wavs = [_wav(n, seed=B * 7 + i) for i, n in enumerate(lens)]
    rc, cbuf, ebuf, nc, ne, Fs = _raw(e, wavs)
    assert rc == L.MVB_OK, L.load().mvb_last_error()
    assert (cbuf[:GUARD] == -1).all() and (cbuf[GUARD + nc:] == -1).all(), "codes written outside the output"
    assert torch.isnan(ebuf[:GUARD]).all() and torch.isnan(ebuf[GUARD + ne:]).all(), "embeddings written outside the output"
    codes, embs = cbuf[GUARD:GUARD + nc], ebuf[GUARD:GUARD + ne]
    assert (codes >= 0).all() and (codes < 1024).all() and not torch.isnan(embs).any(), "a segment was not fully written"
    want_c = [e.encode(w) for w in wavs]
    want_e = [e.embed(w) for w in wavs]
    assert torch.equal(codes, torch.cat([c.reshape(-1) for c in want_c])), f"codes B={B} lens={lens[:8]}"
    assert torch.equal(embs, torch.cat([x.reshape(-1) for x in want_e])), f"embeddings B={B}"
    got = e.encode_batch(wavs)
    assert len(got) == B and all(torch.equal(g, w) for g, w in zip(got, want_c)), "python wrapper"
    print(f"encode_batch B={B} lens={lens[:8]}: bit-identical to solo")


def test_python_wrapper_splits_oversized_batches(setup):
    e, _, _ = setup
    wavs = [_wav(n, seed=n) for n in [240000, 240000, 321, 1]]          # 750 + 750 + 2 + 1 frames > MAX_TOTAL
    got = e.encode_batch(wavs)
    assert all(torch.equal(g, e.encode(w)) for g, w in zip(got, wavs))


def test_invalid_arguments_leave_outputs_untouched(setup):
    from mvb200 import _lib as L
    e, _, _ = setup
    lib = L.load()
    assert lib.mvb_enc_batch_workspace_bytes(C.byref(e.cfg), 33, 1024) == 0
    assert lib.mvb_enc_batch_workspace_bytes(C.byref(e.cfg), 0, 1024) == 0
    ok = [_wav(n, 1) for n in (1, 320, 700)]
    cases = {
        "n = 0": dict(wavs=ok, n=0),
        "n > max_batch": dict(wavs=ok, n=3, max_batch=2),
        "max_batch > 32": dict(wavs=[_wav(8, 2)] * 33, max_batch=33),
        "L_i < 1": dict(wavs=ok, lens=[1, 0, 700]),
        "L_i > 320 max_frames": dict(wavs=[_wav(320 * 2250 + 1, 3)]),
        "sum F_i > max_total_frames": dict(wavs=[_wav(320 * 1000, 4), _wav(320 * 25, 5)]),
    }
    for label, kw in cases.items():
        rc, cbuf, ebuf, _, _, _ = _raw(e, kw["wavs"], n=kw.get("n"), lens=kw.get("lens"), max_batch=kw.get("max_batch", 32))
        assert rc == L.MVB_ERR_ARG, (label, rc)
        assert (cbuf == -1).all() and torch.isnan(ebuf).all(), f"{label}: outputs written"
    x = _wav(10, 6).to(DEV)
    codes = torch.full((8, 1), -1, dtype=torch.int32, device=DEV)
    for L_bad in (0, 320 * 2250 + 1):
        assert lib.mvb_enc_encode(e._h, x.data_ptr(), L_bad, codes.data_ptr(), None, e._st()) == L.MVB_ERR_ARG
    assert (codes == -1).all()


def _write_wav(path, pcm):                  # int16 [n, ch] at 24 kHz
    ch = pcm.shape[1]
    data = pcm.astype("<i2").tobytes()
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 36 + len(data)) + b"WAVEfmt " +
                struct.pack("<IHHIIHH", 16, 1, ch, 24000, 24000 * 2 * ch, 2 * ch, 16) + b"data" + struct.pack("<I", len(data)) + data)


def test_get_tokens_mono_and_stereo(setup, tmp_path):
    from mvb200.vocoder import get_tokens
    e, _, _ = setup
    a = (_wav(9000, 1).numpy() * 32767).astype(np.int16)
    b = (_wav(9000, 2).numpy() * 32767).astype(np.int16)
    mono, stereo = os.path.join(tmp_path, "m.wav"), os.path.join(tmp_path, "s.wav")
    _write_wav(mono, a[:, None])
    _write_wav(stereo, np.stack([a, b], axis=1))
    want = e.encode(torch.from_numpy(a.astype(np.float32) / 32768.0)).tolist()
    assert get_tokens(e, mono) == want
    assert get_tokens(e, stereo) == want
    assert len(want) == 8 and len(want[0]) == -(-9000 // 320)


def test_codes_feed_the_batched_decoder(setup):
    from mvb200.vocoder import EncodecDecodeEngine
    e, _, sd = setup
    wavs = [_wav(n, seed=n) for n in (2560, 24000, 4001)]
    codes = e.encode_batch(wavs)
    d = EncodecDecodeEngine(sd, device=DEV, max_frames=2048, max_batch=4, max_total_frames=256)
    try:
        out = d.decode_batch(codes)
        assert [o.numel() for o in out] == [c.shape[1] * 320 for c in codes]
        assert all(torch.isfinite(o).all() for o in out)
    finally:
        d.close()
