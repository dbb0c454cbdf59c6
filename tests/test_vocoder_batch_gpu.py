"""GPU: the batched EnCodec decode (`mvb_voc_decode_batch` / `mvb_voc_decode_latent_batch`, through
`EncodecDecodeEngine.decode_batch` / `decode_latent_batch`) against the single-utterance calls.

The single-utterance calls launch the same kernels with one segment, and every kernel computes a segment's tiles without
reading another's (the LSTM sums each gate row in the same order whether it runs one sequence or four per pass), so
utterance i of a batch must be bit-identical to `mvb_voc_decode` / `mvb_voc_decode_latent` on it alone, for B = 1, 3, 8
and 32 ragged utterances of T_i in {8, 9, 31, 257, 375, 2048 = max_frames} in two orders, with code values 0
and 1023 present.  The output buffer is NaN-filled with NaN guards on both sides: the call must write every segment and
nothing else.  One ragged batch is compared with the float64 oracle port at the whole-decode bound of
test_vocoder_ops_gpu.py.  Sensitivity: the solo results concatenated with two utterances of different length swapped must
differ from the batch.  Every invalid argument returns MVB_ERR_ARG before anything is launched (outputs untouched)."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
LENS = (8, 9, 31, 257, 375, 2048)
MAX_TOTAL = 16384
GUARD = 1024
NORMWISE = 1e-4


@pytest.fixture(scope="module")
def eng():
    from mvb200 import synth
    from mvb200.vocoder import EncodecDecodeEngine
    _, sd = synth.encodec_model_and_state_dict(seed=0)
    e = EncodecDecodeEngine(sd, device=DEV, max_frames=2048, max_batch=32, max_total_frames=MAX_TOTAL)
    yield e, sd
    e.close()


def _lens(B, reverse):
    seq = LENS[::-1] if reverse else LENS
    return [seq[i % len(seq)] for i in range(B)]


def _codes(lens, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for T in lens:
        c = torch.randint(0, 1024, (8, T), generator=g, dtype=torch.int32)
        c[:, 0] = 0
        c[:, -1] = 1023
        out.append(c)
    return out


def _raw(e, fn, codes, rows, per_frame, n=None, lens=None, max_batch=32):
    """The C entry point on a NaN-filled, guarded output: (rc, guarded buffer, body)."""
    from mvb200 import _lib as L
    lens = lens or [c.shape[1] for c in codes]
    n = len(lens) if n is None else n
    total = rows * sum(c.shape[1] for c in codes) * per_frame
    buf = torch.full((2 * GUARD + total,), float("nan"), device=DEV)
    flat = torch.cat([c.reshape(-1) for c in codes]).to(DEV, torch.int32) if codes else torch.zeros(1, dtype=torch.int32, device=DEV)
    T = (C.c_int32 * max(len(lens), 1))(*lens)
    rc = getattr(e._lib, fn)(e._h, n, flat.data_ptr(), T, e._bws.data_ptr(), max_batch, MAX_TOTAL, buf[GUARD:].data_ptr(),
                             e._st())
    torch.cuda.synchronize()
    return rc, buf, buf[GUARD:GUARD + total], L


@pytest.mark.parametrize("B", [1, 3, 8, 32])
@pytest.mark.parametrize("reverse", [False, True])
def test_batch_bit_identical_to_solo(eng, B, reverse):
    e, _ = eng
    lens = _lens(B, reverse)
    codes = _codes(lens, seed=B * 2 + reverse)
    for fn, rows, pf, solo, api in (("mvb_voc_decode_batch", 1, e.upsample, e.decode, e.decode_batch),
                                    ("mvb_voc_decode_latent_batch", e.cfg.hidden, 1, e.decode_latent, e.decode_latent_batch)):
        rc, buf, body, L = _raw(e, fn, codes, rows, pf)
        assert rc == L.MVB_OK, L.load().mvb_last_error()
        assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + body.numel():]).all(), f"{fn}: write outside the output"
        assert not torch.isnan(body).any(), f"{fn}: a segment was not fully written"
        want = [solo(c) for c in codes]
        assert torch.equal(body, torch.cat([w.reshape(-1) for w in want])), f"{fn} B={B} lens={lens}"
        got = api(codes)
        assert len(got) == B and all(torch.equal(g, w) for g, w in zip(got, want)), f"{fn}: python wrapper"
        if B >= 3 and fn == "mvb_voc_decode_batch":
            # sensitivity: the solo results with two utterances of different length swapped are not the batch
            sw = list(want)
            sw[1], sw[2] = sw[2], sw[1]
            assert lens[1] != lens[2] and not torch.equal(body, torch.cat([w.reshape(-1) for w in sw]))
        print(f"{fn} B={B} lens={lens[:6]}...: bit-identical to solo")


def test_python_wrapper_splits_oversized_batches(eng):
    e, _ = eng
    lens = [2048] * 9 + [8]                 # 18440 frames > MAX_TOTAL: two launch sets
    codes = _codes(lens, seed=77)
    got = e.decode_batch(codes)
    assert all(torch.equal(g, e.decode(c)) for g, c in zip(got, codes))


def test_ragged_batch_vs_float64_oracle(eng):
    from test_vocoder_ops_gpu import _oracle_f64
    e, sd = eng
    lens = [375, 8, 257, 31]
    codes = _codes(lens, seed=5)
    got = e.decode_batch(codes)
    o = _oracle_f64(sd)
    prev = torch.get_default_dtype()
    for c, w in zip(codes, got):
        torch.set_default_dtype(torch.float64)
        try:
            with torch.device(DEV):
                ref = o.decode(c.long()[None].to(DEV))[0, 0]
        finally:
            torch.set_default_dtype(prev)
        nw = float((w.double() - ref).norm() / ref.norm())
        print(f"decode_batch T={c.shape[1]}: normwise {nw:.2e} vs the float64 oracle")
        assert w.shape == ref.shape and nw < NORMWISE


def test_invalid_arguments_leave_outputs_untouched(eng):
    from mvb200 import _lib as L
    e, _ = eng
    lib = L.load()
    assert lib.mvb_voc_batch_workspace_bytes(C.byref(e.cfg), 33, 1024) == 0
    assert lib.mvb_voc_batch_workspace_bytes(C.byref(e.cfg), 0, 1024) == 0
    ok = _codes([8, 9, 31], seed=1)
    cases = {
        "n = 0": dict(codes=ok, n=0),
        "n > max_batch": dict(codes=ok, n=3, max_batch=2),
        "max_batch > 32": dict(codes=_codes([8] * 33, seed=2), max_batch=33),
        "T_i < 8": dict(codes=_codes([8, 7, 31], seed=3)),
        "T_i > max_frames": dict(codes=_codes([8, 2049], seed=4)),
        "sum T_i > max_total_frames": dict(codes=_codes([2048] * 8 + [9], seed=5)),
    }
    for label, kw in cases.items():
        for fn, rows, pf in (("mvb_voc_decode_batch", 1, e.upsample), ("mvb_voc_decode_latent_batch", e.cfg.hidden, 1)):
            rc, buf, _, _ = _raw(e, fn, kw["codes"], rows, pf, n=kw.get("n"), max_batch=kw.get("max_batch", 32))
            assert rc == L.MVB_ERR_ARG, (label, fn, rc)
            assert torch.isnan(buf).all(), f"{label}: {fn} wrote its output"
