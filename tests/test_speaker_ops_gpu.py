"""GPU: the speaker-encoder kernels of csrc/speaker.cu one at a time against float64 references of the same operations on
the kernels' own fp32 inputs, then the whole of SpeakerEncoder.embed_utterance against the float64 oracle.  `k_spk_mel`
runs through mvb_spk_mel, `k_spk_lstm` and `k_spk_mean` through the hook mvb_spk_op_test, which uses mvb_spk_embed's
launch helper.  Handles are built here on arenas packed in the header's order with the filterbank, window and tables
SpeakerEncoder.__init__ builds, so that other front-end configurations and mel band counts can be run.  u = 2^-23.

k_spk_mel    frame v[n] = fl(wav[s] window[n]) (zero outside the signal; one rounding), then for bin k
               re = sum_n v[n] cosT[k n mod n_fft],  im likewise with sinT,
             each an n_fft-term fmaf chain from 0, so with the frame rounding
               |dre| <= (n_fft + 1) u sum_n |v| |cosT|,   |dim| likewise;
             power p = re^2 + im^2 (possibly contracted):
               |dp| <= 2 |re| dre + dre^2 + 2 |im| dim + dim^2 + 2u p;
             mel = an n_bins-term fmaf chain of the non-negative fb p from 0:
               |dmel| <= n_bins u sum_k fb p + sum_k fb |dp|.
             The reference uses the fp32 tables the kernel reads; a second, normwise-only comparison uses true float64
             trigonometry and the float64 periodic Hann window.
k_spk_lstm   teacher-forced: each step of the float64 reference starts from the kernel's own traced state (h of layer
             l - 1 at step t, h and c of layer l at step t - 1).  The pre-activation is a per-lane fmaf chain of
             ceil(K / 32) input terms and 8 recurrent terms, the 5-step warp_sum butterfly, and the bias add:
               |da| <= (ceil(K / 32) + 8 + 6) u (sum |w_ih| |x| + sum |w_hh| |h| + |b|).
             sigma(a) = 1 / (1 + expf(-a)) (expf 2 ulp, one add, one IEEE division; sigma' <= 1/4):
               |dsigma| <= |da| / 4 + 5u sigma;   tanhf (2 ulp, tanh' <= 1): |dtanh| <= |da| + 2u |tanh|.
             Cell, against the kernel's own c_{t-1} (no drift term):
               |dc| <= |df| |c_{t-1}| + |di| |g| + i |dg| + |di| |dg| + 2u (|f c_{t-1}| + |i g|);
             h = o tanhf(c) against the kernel's own c_t:  |dh| <= |do| |tanh c| + 2u o |tanh c| + u |h|.
             With saturated gates c and h reach the subnormal range (1e-43 at inputs of 1e3), where a rounding is off
             by up to half a subnormal step eta = 2^-149 and a 2-ulp function by 2 eta, whatever the relative terms say:
             the gate bounds carry 3 eta (2 for tanh g), c 2 eta and h 3 eta more.
             Head, from the traced final h of layer 3: e = relu(b + sum_k W[j, k] h[k]), a 256-term serial fmaf chain
             from the bias, |de| <= 256 u (|b| + sum |W| |h|) (ReLU is 1-Lipschitz, so an element whose pre-activation lies
             within its bound of 0 may land on either side and still meet it); y = e / ||e|| with ||e||^2 summed by
             warp_sum and 8 serial adds (14 roundings), sqrtf and a division:
               |dy_j| <= |de_j| / ||e|| + |y_j| (||de|| / ||e|| + 16u).
k_spk_mean   m = (sum_p x_p) / P by P serial adds from 0 (P - 1 roundings) and a division:
               |dm| <= (P - 1) u sum_p |x_p| / P + u |m|,  y = m / ||m|| as for the head.
Every output has NaN guards on both sides (a write outside it or an element left unwritten fails), and every check
also asserts ||err|| / ||ref|| < 1e-4 and prints the worst |err| / bound.

End to end, SpeakerEncoder.embed_utterance is compared normwise with oracle/speaker_port.SpeakerOracle in float64
(float64 mel front-end, LSTM and average).  That comparison is free-running over 160 steps x 3 layers, so it has no
elementwise bound: its threshold E2E sits more than 10x above the worst error measured on an H100 (see E2E).

Sensitivity: reflect instead of zero centre padding (librosa < 0.10), frames shifted by one sample, a symmetric Hann
window, the f and g gates swapped, bias_ih without bias_hh, the head without its ReLU and the mean of the un-normalised
partials must each put elements over the bound."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
NORMWISE = 1e-4
# End-to-end normwise threshold (partials and embedding vs the float64 oracle), free-running.  Worst measured on an H100
# over the lengths of test_embed_utterance_vs_float64_oracle: 4.0e-7 (partials, 30 s), 4.0e-7 (embedding, 25,599
# samples); E2E is 12.5x that.
E2E = 5e-6
ETA = 2.0 ** -149                       # one subnormal step: the absolute part of an fp32 rounding near zero
GUARD = 1024
DEV = "cuda"
H = 256
SR = 16000
PROD = dict(n_mels=40, n_fft=400, hop=160, T=160)
MAX_180 = 180 * SR + 160 * 160          # what SpeakerEncoder(max_seconds=180) asks the workspace for
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    from mvb200 import _lib as L
    return L, L.load()


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _guarded(n):
    buf = torch.full((2 * GUARD + n,), float("nan"), device=DEV)
    return buf, buf[GUARD:GUARD + n]


def _check_guards(buf, n):
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + n:]).all(), "write outside the output"
    assert not torch.isnan(buf[GUARD:GUARD + n]).any(), "output not fully written"


def _report(label, got, ref, bound):
    err = (got - ref).abs()
    ratio, nw = float((err / bound).max()), float(err.norm() / ref.norm().clamp_min(1e-300))
    print(f"{label}: max |err|/bound {ratio:.2e}, normwise {nw:.2e}")
    bad = (err > bound).nonzero()
    assert bad.numel() == 0, f"{label}: {bad.shape[0]} elements over the bound, first at {bad[0].tolist()}"
    assert nw < NORMWISE, f"{label}: normwise {nw:.2e}"
    return ratio


def _over(got, ref, bound):
    return int(((got - ref).abs() > bound).sum())


def _i32(xs):
    return np.ascontiguousarray(np.asarray(xs, dtype=np.int32))


def _state(n_mels, seed=3):
    """synth.speaker_encoder_state_dict with a layer-0 input width of n_mels (the same U(-1/16, 1/16) init)."""
    from mvb200 import synth
    sd = synth.speaker_encoder_state_dict(seed)
    if n_mels != 40:
        g = torch.Generator().manual_seed(seed + n_mels)
        sd["lstm.weight_ih_l0"] = (torch.rand(4 * H, n_mels, generator=g) * 2 - 1) / 16
    return sd


class Spk:
    """An mvb_spk handle over an arena packed here: per layer {w_ih, w_hh, b_ih + b_hh}, linear w and b, the Slaney
    filterbank, the periodic Hann window, cos and -sin tables (include/mvb200.h, SpeakerEncoder.__init__)."""

    def __init__(self, n_mels=40, n_fft=400, hop=160, T=160, max_samples=30 * SR, sd=None, random_fb=False):
        from mvb200.speaker_encoder import slaney_mel_filterbank
        L, lib = _lib()
        self.n_mels, self.n_fft, self.hop, self.T, self.max_samples = n_mels, n_fft, hop, T, max_samples
        self.sd = sd = _state(n_mels) if sd is None else sd
        i = np.arange(n_fft)
        fb = slaney_mel_filterbank(SR, n_fft, n_mels)
        if random_fb:
            fb = np.random.default_rng(n_fft).uniform(0, 1e-2, fb.shape).astype(np.float32)
        tensors = []
        for l in range(3):
            tensors += [sd[f"lstm.weight_ih_l{l}"].float(), sd[f"lstm.weight_hh_l{l}"].float(),
                        sd[f"lstm.bias_ih_l{l}"].float() + sd[f"lstm.bias_hh_l{l}"].float()]
        tensors += [sd["linear.weight"].float(), sd["linear.bias"].float(),
                    torch.from_numpy(fb),
                    torch.from_numpy((0.5 - 0.5 * np.cos(2 * np.pi * i / n_fft)).astype(np.float32)),
                    torch.from_numpy(np.cos(2 * np.pi * i / n_fft).astype(np.float32)),
                    torch.from_numpy((-np.sin(2 * np.pi * i / n_fft)).astype(np.float32))]
        offs, total = [], 0
        for t in tensors:
            offs.append(total)
            total = (total + t.numel() * 4 + 255) // 256 * 256
        arena = torch.zeros(total, dtype=torch.uint8)
        for t, o in zip(tensors, offs):
            arena[o:o + t.numel() * 4] = t.contiguous().reshape(-1).view(torch.uint8)
        self.arena_host = arena
        self.arena = arena.to(DEV)
        self.cfg = L.SpkConfig(n_mels, H, 3, H, n_fft, hop, T, max_samples)
        self.ws = torch.zeros(lib.mvb_spk_workspace_bytes(C.byref(self.cfg)), dtype=torch.uint8, device=DEV)
        h = C.c_void_p()
        L.check(lib.mvb_spk_create(C.byref(self.cfg), self.arena.data_ptr(), self.arena.numel(), (C.c_uint64 * len(offs))(*offs),
                                   self.ws.data_ptr(), C.byref(h)))
        self.h = h
        d = lambda t: t.to(DEV, torch.float64)    # noqa: E731
        self.layers = [tuple(d(t) for t in tensors[3 * l:3 * l + 3]) for l in range(3)]
        self.lw, self.lb, self.fb, self.win, self.cos, self.sin = (d(t) for t in tensors[9:])

    def close(self):
        if self.h is not None:
            _lib()[1].mvb_spk_destroy(self.h)
            self.h = None

    def frames(self, n):
        return 1 + n // self.hop

    def mel(self, wav):
        """k_spk_mel of fp32 wav (device) -> fp32 [n_frames, n_mels] (device)."""
        L, lib = _lib()
        F, n = self.frames(wav.numel()), self.n_mels
        buf, out = _guarded(F * n)
        L.check(lib.mvb_spk_mel(self.h, wav.data_ptr(), wav.numel(), out.data_ptr(), _st()))
        torch.cuda.synchronize()
        _check_guards(buf, F * n)
        return out.view(F, n)

    def lstm(self, mel, starts, trace=True):
        """op 0: fp32 partials [P, 256] and (trace=True) the state trace [P, T, 3, 2, 256] (device)."""
        L, lib = _lib()
        st = _i32(starts)
        P = st.size
        bp, part = _guarded(P * H)
        nt = P * self.T * 3 * 2 * H
        bt, tr = _guarded(nt) if trace else (None, None)
        L.check(lib.mvb_spk_op_test(self.h, 0, mel.data_ptr(), mel.shape[0], st.ctypes.data_as(C.c_void_p), P, part.data_ptr(),
                                    None if tr is None else tr.data_ptr(), _st()))
        _check_guards(bp, P * H)
        if not trace:
            return part.view(P, H), None
        _check_guards(bt, nt)
        return part.view(P, H), tr.view(P, self.T, 3, 2, H)

    def mean(self, partials):
        """op 1: fp32 [256] (device)."""
        L, lib = _lib()
        buf, out = _guarded(H)
        L.check(lib.mvb_spk_op_test(self.h, 1, partials.data_ptr(), 0, None, partials.shape[0], out.data_ptr(), None, _st()))
        _check_guards(buf, H)
        return out

    def embed(self, wav, starts, n_partials=None, embed_out=None, partials_out=None):
        """mvb_spk_embed -> its status (no check)."""
        _, lib = _lib()
        st = _i32(starts)
        ptr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
        rc = lib.mvb_spk_embed(self.h, ptr(wav), 0 if wav is None else wav.numel(), st.ctypes.data_as(C.c_void_p),
                               st.size if n_partials is None else n_partials, ptr(embed_out), ptr(partials_out), _st())
        torch.cuda.synchronize()
        return rc


_ENGINES = {}


def _engine(**kw):
    key = tuple(sorted(kw.items()))
    if key not in _ENGINES:
        _ENGINES[key] = Spk(**kw)
    return _ENGINES[key]


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for e in _ENGINES.values():
        e.close()
    _ENGINES.clear()


_WAV = {}


def _speech(n):
    """n samples of the speech-like synthetic signal (a prefix of one 180 s + window draw)."""
    if "w" not in _WAV:
        from mvb200 import synth
        _WAV["w"] = synth.synthetic_waveform(MAX_180 / SR + 1, SR, seed=9)
    assert n <= _WAV["w"].size
    return _WAV["w"][:n]


def test_arena_matches_speaker_encoder():
    """The arena packed here is byte for byte the one SpeakerEncoder builds, so the handles of this module are the
    product's."""
    from mvb200.speaker_encoder import SpeakerEncoder
    sd = _state(40)
    enc = SpeakerEncoder(model_state=sd, device=DEV, verbose=False)
    try:
        spk = _engine(**PROD, max_samples=MAX_180)
        assert torch.equal(enc._arena.cpu(), spk.arena_host)
        assert enc.cfg.max_samples == MAX_180 and enc.max_input_samples == 180 * SR
    finally:
        enc.close()


# ---- k_spk_mel ----------------------------------------------------------------------------------------------------------
def mel_model(spk, wav, shift=0, pad="zero", window=None):
    """(ref, bound) of k_spk_mel in float64 on the kernel's fp32 tables; shift / pad / window alter the reference."""
    n_fft, hop = spk.n_fft, spk.hop
    x = torch.from_numpy(np.asarray(wav)).to(DEV, torch.float64)
    n = x.numel()
    F = spk.frames(n)
    s = torch.arange(F, device=DEV)[:, None] * hop - n_fft // 2 + shift + torch.arange(n_fft, device=DEV)[None, :]
    if pad == "reflect":
        s = torch.where(s < 0, -s, s)
        s = torch.where(s >= n, 2 * (n - 1) - s, s)
    inside = (s >= 0) & (s < n)
    win = spk.win if window is None else window
    V = torch.where(inside, x[s.clamp(0, n - 1)], torch.zeros((), dtype=torch.float64, device=DEV)) * win[None, :]
    k = torch.arange(n_fft // 2 + 1, device=DEV)
    ph = (k[:, None] * torch.arange(n_fft, device=DEV)[None, :]) % n_fft
    Cm, Sm = spk.cos[ph], spk.sin[ph]
    re, im = V @ Cm.t(), V @ Sm.t()
    Va = V.abs()
    dre, dim = (n_fft + 1) * U * (Va @ Cm.abs().t()), (n_fft + 1) * U * (Va @ Sm.abs().t())
    p = re * re + im * im
    dp = 2 * re.abs() * dre + dre * dre + 2 * im.abs() * dim + dim * dim + 2 * U * p
    ref = p @ spk.fb.t()
    bound = (n_fft // 2 + 1) * U * ref + dp @ spk.fb.t() + 1e-300
    return ref, bound


def mel_true(spk, wav):
    """float64 power mel with true trigonometry and the float64 periodic Hann window (centred, zero padded)."""
    n_fft, hop = spk.n_fft, spk.hop
    x = torch.from_numpy(np.asarray(wav)).to(DEV, torch.float64)
    n = x.numel()
    s = torch.arange(spk.frames(n), device=DEV)[:, None] * hop - n_fft // 2 + torch.arange(n_fft, device=DEV)[None, :]
    inside = (s >= 0) & (s < n)
    i = torch.arange(n_fft, device=DEV, dtype=torch.float64)
    V = torch.where(inside, x[s.clamp(0, n - 1)], torch.zeros((), dtype=torch.float64, device=DEV)) * (0.5 - 0.5 * torch.cos(2 * math.pi * i / n_fft))
    return (torch.fft.rfft(V, dim=1).abs() ** 2) @ spk.fb.t()


MEL_CONFIGS = {
    "production": dict(**PROD, max_samples=MAX_180),
    "maxima": dict(n_mels=64, n_fft=2048, hop=512, T=160, max_samples=30 * SR),
    "odd_nfft": dict(n_mels=40, n_fft=401, hop=160, T=160, max_samples=30 * SR),
    # both bins of a 2-point frame sit on filter edges, where every Slaney filter is 0: a random filterbank instead
    "nfft2_hop1": dict(n_mels=40, n_fft=2, hop=1, T=160, max_samples=30 * SR, random_fb=True),
}


def _mel_lengths(c):
    n_fft, hop, mx = c["n_fft"], c["hop"], c["max_samples"]
    ls = [1, 2, n_fft // 2 - 1, n_fft // 2, n_fft // 2 + 1, hop - 1, hop, hop + 1, n_fft, 25600, int(6.4 * SR), 30 * SR, mx]
    if mx >= 180 * SR:
        ls.append(180 * SR)                 # 18,001 frames: the 180 s input before SpeakerEncoder's extra window
    return sorted({n for n in ls if 1 <= n <= mx})


@pytest.mark.parametrize("name", list(MEL_CONFIGS))
def test_mel_vs_float64(name):
    c = MEL_CONFIGS[name]
    spk = _engine(**c)
    worst = 0.0
    for n in _mel_lengths(c):
        wav = _speech(n)
        got = spk.mel(torch.from_numpy(wav).to(DEV)).double()
        ref, bound = mel_model(spk, wav)
        assert got.shape == ref.shape == (spk.frames(n), c["n_mels"])
        worst = max(worst, _report(f"k_spk_mel {name} n={n} ({got.shape[0]} frames)", got, ref, bound))
        true = mel_true(spk, wav)
        nw = float((got - true).norm() / true.norm().clamp_min(1e-300))
        print(f"k_spk_mel {name} n={n}: normwise {nw:.2e} vs true float64 trigonometry")
        assert nw < NORMWISE
    print(f"k_spk_mel {name}: worst |err|/bound {worst:.2e}")


def test_mel_sensitivity():
    """Reflect padding on the edge frames, frames one sample late and a symmetric Hann window each break the bound."""
    spk = _engine(**PROD, max_samples=MAX_180)
    wav = _speech(int(6.4 * SR))
    got = spk.mel(torch.from_numpy(wav).to(DEV)).double()
    _, bound = mel_model(spk, wav)
    i = torch.arange(spk.n_fft, device=DEV, dtype=torch.float64)
    sym = (0.5 - 0.5 * torch.cos(2 * math.pi * i / (spk.n_fft - 1))).float().double()
    n = {"reflect padding": _over(got, mel_model(spk, wav, pad="reflect")[0], bound),
         "shifted by one sample": _over(got, mel_model(spk, wav, shift=1)[0], bound),
         "symmetric Hann": _over(got, mel_model(spk, wav, window=sym)[0], bound)}
    print(f"k_spk_mel altered references, elements over the bound: {n}")
    assert all(v > 0 for v in n.values()), n


# ---- k_spk_lstm ---------------------------------------------------------------------------------------------------------
def lstm_model(spk, mel, starts, trace, swap_fg=False, bias=None):
    """Teacher-forced float64 steps from the kernel's own trace -> (h, c, bound_h, bound_c), each [P, T, 3, 256].
    bias: per-layer float64 biases replacing b_ih + b_hh (sensitivity)."""
    P, T = trace.shape[:2]
    tr = trace.double()
    hk, ck = tr[:, :, :, 0], tr[:, :, :, 1]
    st = torch.as_tensor(np.asarray(starts), device=DEV).long()
    x0 = mel.double()[st[:, None] + torch.arange(T, device=DEV)[None, :]]
    zero = torch.zeros(P, 1, H, dtype=torch.float64, device=DEV)
    hs, cs, bhs, bcs = [], [], [], []
    for l in range(3):
        w_ih, w_hh, b = spk.layers[l]
        if bias is not None:
            b = bias[l]
        x = x0 if l == 0 else hk[:, :, l - 1]
        hp = torch.cat([zero, hk[:, :-1, l]], 1)
        cp = torch.cat([zero, ck[:, :-1, l]], 1)
        K = x.shape[-1]
        a = x @ w_ih.t() + hp @ w_hh.t() + b
        da = (math.ceil(K / 32) + 8 + 6) * U * (x.abs() @ w_ih.abs().t() + hp.abs() @ w_hh.abs().t() + b.abs())
        ai, af, ag, ao = a.split(H, -1)
        di, df, dg, do = da.split(H, -1)
        if swap_fg:
            af, ag = ag, af
        i, f, g, o = torch.sigmoid(ai), torch.sigmoid(af), torch.tanh(ag), torch.sigmoid(ao)
        di, df, do = di / 4 + 5 * U * i + 3 * ETA, df / 4 + 5 * U * f + 3 * ETA, do / 4 + 5 * U * o + 3 * ETA
        dg = dg + 2 * U * g.abs() + 2 * ETA
        c = f * cp + i * g
        bc = df * cp.abs() + di * g.abs() + i * dg + di * dg + 2 * U * ((f * cp).abs() + (i * g).abs()) + 2 * ETA
        tck = torch.tanh(ck[:, :, l])
        h = o * tck
        bh = do * tck.abs() + 2 * U * o * tck.abs() + U * h.abs() + 3 * ETA
        hs.append(h), cs.append(c), bhs.append(bh), bcs.append(bc)
    return torch.stack(hs, 2), torch.stack(cs, 2), torch.stack(bhs, 2), torch.stack(bcs, 2)


def head_model(spk, h_last, relu=True):
    """(y, bound) of linear + ReLU + L2 norm from the final h of layer 3 [P, 256]."""
    h = h_last.double()
    e = h @ spk.lw.t() + spk.lb
    de = 256 * U * (h.abs() @ spk.lw.abs().t() + spk.lb.abs())
    if relu:
        e = e.clamp_min(0)
    N = e.norm(dim=1, keepdim=True)
    y = e / N
    return y, de / N + y.abs() * (de.norm(dim=1, keepdim=True) / N + 16 * U) + 1e-300


def mean_model(x, unnormalised_from=None):
    """(y, bound) of k_spk_mean on fp32 partials x [P, 256]; unnormalised_from: raw head outputs averaged instead."""
    xd = x.double()
    P = xd.shape[0]
    m = xd.mean(0) if unnormalised_from is None else unnormalised_from.mean(0)
    dm = (P - 1) * U * xd.abs().sum(0) / P + U * xd.mean(0).abs()
    N = m.norm()
    y = m / N
    return y, dm / N + y.abs() * (dm.norm() / N + 16 * U) + 1e-300


def _starts(F, T, P):
    """P windows over F frames: overlapping when T is, the last ending exactly on the last frame."""
    if P == 1:
        return [F - T]
    step = max(1, min(77, (F - T) // (P - 1)))
    st = [min(i * step, F - T) for i in range(P - 1)] + [F - T]
    return st


def _lstm_inputs(spk, scale, F=3001):
    if scale == "mel":
        return spk.mel(torch.from_numpy(_speech(30 * SR)).to(DEV))
    g = torch.Generator(device=DEV).manual_seed(F + spk.n_mels)
    return torch.randn(F, spk.n_mels, generator=g, device=DEV) * float(scale)


def _check_lstm(spk, mel, starts, label):
    part, trace = spk.lstm(mel, starts)
    h, c, bh, bc = lstm_model(spk, mel, starts, trace)
    r1 = _report(f"k_spk_lstm {label} h", trace[:, :, :, 0].double(), h, bh)
    r2 = _report(f"k_spk_lstm {label} c", trace[:, :, :, 1].double(), c, bc)
    y, by = head_model(spk, trace[:, -1, 2, 0])
    r3 = _report(f"k_spk_lstm {label} head", part.double(), y, by)
    return max(r1, r2), r3, (part, trace)


@pytest.mark.parametrize("T", [1, 2, 160])
@pytest.mark.parametrize("n_mels", [1, 40, 64])
def test_lstm_teacher_forced(n_mels, T):
    spk = _engine(n_mels=n_mels, n_fft=400, hop=160, T=T, max_samples=30 * SR)
    worst_cell, worst_head = 0.0, 0.0
    for scale in ("mel", "1e-3", "1e3"):
        mel = _lstm_inputs(spk, scale)
        for P in (1, 3, 37, 233):
            st = _starts(mel.shape[0], T, P)
            a, b, _ = _check_lstm(spk, mel, st, f"n_mels={n_mels} T={T} P={P} input={scale}")
            worst_cell, worst_head = max(worst_cell, a), max(worst_head, b)
    print(f"k_spk_lstm n_mels={n_mels} T={T}: worst |err|/bound {worst_cell:.2e} (h, c), {worst_head:.2e} (head)")


def test_lstm_sensitivity():
    """f and g swapped, bias_ih without bias_hh, and the head without ReLU each break the bound."""
    spk = _engine(**PROD, max_samples=MAX_180)
    mel = _lstm_inputs(spk, "mel")
    st = _starts(mel.shape[0], 160, 37)
    _, _, (part, trace) = _check_lstm(spk, mel, st, "sensitivity")
    got_h, got_c = trace[:, :, :, 0].double(), trace[:, :, :, 1].double()
    _, _, bh, bc = lstm_model(spk, mel, st, trace)

    def over(ref):            # h depends on the gates only through o (it is checked on the kernel's c): count c too
        return _over(got_h, ref[0], bh) + _over(got_c, ref[1], bc)

    swapped = lstm_model(spk, mel, st, trace, swap_fg=True)
    b_ih = [spk.sd[f"lstm.bias_ih_l{l}"].to(DEV, torch.float64) for l in range(3)]
    no_hh = lstm_model(spk, mel, st, trace, bias=b_ih)
    _, by = head_model(spk, trace[:, -1, 2, 0])
    no_relu = head_model(spk, trace[:, -1, 2, 0], relu=False)[0]
    n = {"f/g swapped": over(swapped), "bias_ih only": over(no_hh), "head without ReLU": _over(part.double(), no_relu, by)}
    print(f"k_spk_lstm altered references, elements over the bound: {n}")
    assert all(v > 0 for v in n.values()), n


# ---- k_spk_mean ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [1, 2, 233, 1024])
def test_mean_vs_float64(P):
    spk = _engine(**PROD, max_samples=MAX_180)
    g = torch.Generator(device=DEV).manual_seed(P)
    signed = torch.randn(P, H, generator=g, device=DEV)
    mel = _lstm_inputs(spk, "mel")
    prod, _ = spk.lstm(mel, [(2 * i) % (mel.shape[0] - 159) for i in range(P)], trace=False)
    worst = 0.0
    for label, x in (("signed random", signed), ("production partials", prod)):
        y, by = mean_model(x)
        worst = max(worst, _report(f"k_spk_mean P={P} {label}", spk.mean(x.contiguous()).double(), y, by))
    print(f"k_spk_mean P={P}: worst |err|/bound {worst:.2e}")


def test_mean_sensitivity():
    """The mean of the un-normalised partials (raw head outputs) breaks the bound."""
    spk = _engine(**PROD, max_samples=MAX_180)
    mel = _lstm_inputs(spk, "mel")
    part, trace = spk.lstm(mel, _starts(mel.shape[0], 160, 37))
    got = spk.mean(part).double()
    y, by = mean_model(part)
    _report("k_spk_mean P=37", got, y, by)
    raw = (trace[:, -1, 2, 0].double() @ spk.lw.t() + spk.lb).clamp_min(0)
    n = _over(got, mean_model(part, unnormalised_from=raw)[0], by)
    print(f"k_spk_mean of un-normalised partials: {n} elements over the bound")
    assert n > 0


# ---- structure and determinism ------------------------------------------------------------------------------------------
def test_hook_matches_embed_and_windows_are_independent():
    """mvb_spk_embed == op 0 on mvb_spk_mel's output, then op 1 (bit for bit); the trace changes nothing; a window's
    partial does not depend on the other windows of the call; two identical calls agree bit for bit; 1024 windows are
    accepted and 1025 refused."""
    L, _ = _lib()
    spk = _engine(**PROD, max_samples=MAX_180)
    wav = torch.from_numpy(_speech(30 * SR)).to(DEV)
    mel = spk.mel(wav)
    F = mel.shape[0]
    st = _starts(F, 160, 37)
    emb, part = torch.empty(H, device=DEV), torch.empty(37, H, device=DEV)
    assert spk.embed(wav, st, embed_out=emb, partials_out=part) == L.MVB_OK
    p0, _ = spk.lstm(mel, st)
    p1, _ = spk.lstm(mel, st, trace=False)
    assert torch.equal(part, p0) and torch.equal(p0, p1)
    assert torch.equal(emb, spk.mean(p0))
    emb2, part2 = torch.empty(H, device=DEV), torch.empty(37, H, device=DEV)
    assert spk.embed(wav, st, embed_out=emb2, partials_out=part2) == L.MVB_OK
    assert torch.equal(emb, emb2) and torch.equal(part, part2)
    sub = [st[5], st[-1], st[0]]
    ps, _ = spk.lstm(mel, sub, trace=False)
    assert torch.equal(ps, p0[[5, 36, 0]])
    alone, _ = spk.lstm(mel, [st[20]], trace=False)
    assert torch.equal(alone[0], p0[20])
    many = [(2 * i) % (F - 159) for i in range(1025)]
    e = torch.empty(H, device=DEV)
    assert spk.embed(wav, many[:1024], embed_out=e) == L.MVB_OK and torch.isfinite(e).all()
    e.fill_(7.0)
    assert spk.embed(wav, many, embed_out=e) == L.MVB_ERR_ARG and (e == 7.0).all()


def test_bit_identical_to_recorded_library():
    """With no trace, SpeakerEncoder's partials and embedding equal bit for bit what the library produced before
    k_spk_lstm gained its trace (tests/golden/speaker_device_bits.npz, oracle/make_golden_speaker_bits.py)."""
    from mvb200 import synth
    from mvb200.speaker_encoder import SpeakerEncoder
    from oracle import make_golden_speaker_bits as B
    g = np.load(os.path.join(ROOT, "tests", "golden", "speaker_device_bits.npz"))
    enc = SpeakerEncoder(model_state=synth.speaker_encoder_state_dict(3), device=DEV, verbose=False)
    try:
        for name, wav in B.waveforms().items():
            e, p, _ = enc.embed_utterance(wav, return_partials=True)
            assert np.array_equal(e.view(np.uint32), g[f"{name}_embed"].view(np.uint32)), name
            assert np.array_equal(p.view(np.uint32), g[f"{name}_partials"].view(np.uint32)), name
    finally:
        enc.close()


# ---- invalid arguments --------------------------------------------------------------------------------------------------
def test_invalid_arguments_leave_outputs_untouched():
    """Null pointers, n_samples 0 / max + 1, n_partials 0 / 1025, a start of -1 and a window one frame past the end all
    return MVB_ERR_ARG before anything is launched: the output and the whole workspace keep their sentinels."""
    L, lib = _lib()
    spk = Spk(**PROD, max_samples=4 * SR)
    try:
        n = 3 * SR
        wav = torch.from_numpy(_speech(spk.max_samples + 1)).to(DEV)
        F = spk.frames(n)
        out = torch.full((H,), 7.0, device=DEV)
        parts = torch.full((4, H), 7.0, device=DEV)
        spk.ws.fill_(0xA5)
        w = wav[:n]
        cases = {
            "null handle": lambda: lib.mvb_spk_embed(None, w.data_ptr(), n, _i32([0]).ctypes.data_as(C.c_void_p), 1, out.data_ptr(),
                                                     None, _st()),
            "null wav": lambda: lib.mvb_spk_embed(spk.h, None, n, _i32([0]).ctypes.data_as(C.c_void_p), 1, out.data_ptr(), None, _st()),
            "null starts": lambda: lib.mvb_spk_embed(spk.h, w.data_ptr(), n, None, 1, out.data_ptr(), None, _st()),
            "null embed": lambda: spk.embed(w, [0]),
            "n_samples 0": lambda: lib.mvb_spk_embed(spk.h, w.data_ptr(), 0, _i32([0]).ctypes.data_as(C.c_void_p), 1, out.data_ptr(),
                                                     None, _st()),
            "n_samples max + 1": lambda: spk.embed(wav, [0], embed_out=out),
            "n_partials 0": lambda: spk.embed(w, [0], n_partials=0, embed_out=out),
            "n_partials 1025": lambda: spk.embed(w, [0] * 1025, embed_out=out),
            "start -1": lambda: spk.embed(w, [0, -1], embed_out=out, partials_out=parts),
            "window past the end": lambda: spk.embed(w, [0, F - 160 + 1], embed_out=out, partials_out=parts),
        }
        for label, call in cases.items():
            rc = call()
            torch.cuda.synchronize()
            print(f"{label}: rc {rc} ({lib.mvb_last_error().decode()})")
            assert rc == L.MVB_ERR_ARG, label
            assert (out == 7.0).all() and (parts == 7.0).all(), f"{label}: output written"
            assert (spk.ws == 0xA5).all(), f"{label}: workspace written"
        assert spk.embed(w, [0, F - 160], embed_out=out, partials_out=parts[:2]) == L.MVB_OK   # the last valid window
        mel = spk.mel(w)
        ok = torch.full((H,), 7.0, device=DEV)
        for label, args in {"op 0 start -1": (0, mel, [-1]), "op 0 past the end": (0, mel, [F - 159]), "op 2": (2, mel, [0])}.items():
            st = _i32(args[2])
            rc = lib.mvb_spk_op_test(spk.h, args[0], args[1].data_ptr(), F, st.ctypes.data_as(C.c_void_p), 1, ok.data_ptr(), None, _st())
            assert rc == L.MVB_ERR_ARG and (ok == 7.0).all(), label
    finally:
        spk.close()


# ---- end to end ---------------------------------------------------------------------------------------------------------
def _coverage_lengths():
    """Around the first two lengths past one window at which the 0.75 coverage rule keeps one more window: the length
    that still drops it and the one that keeps it."""
    from mvb200.speaker_encoder import SpeakerEncoder as S
    out, prev = [], len(S.compute_partial_slices(25600, 1.3, 0.75)[1])
    for n in range(25601, 60000):
        k = len(S.compute_partial_slices(n, 1.3, 0.75)[1])
        if k > prev:
            assert len(S.compute_partial_slices(n - 1, 1.3, 0.0)[1]) == k    # n - 1 forms the window and drops it
            out += [n - 1, n]
        prev = k
        if len(out) == 4:
            return out
    raise AssertionError("no coverage transitions found")


def test_embed_utterance_vs_float64_oracle():
    from mvb200 import synth
    from mvb200.speaker_encoder import SpeakerEncoder
    from oracle import speaker_port as P
    sd = synth.speaker_encoder_state_dict(3)
    enc = SpeakerEncoder(model_state=sd, device=DEV, verbose=False)
    o = P.SpeakerOracle(sd, dtype=torch.float64)
    lengths = [1, 25599, 25600, 25601] + _coverage_lengths() + [int(6.4 * SR), 30 * SR, int(179.9 * SR), 180 * SR]
    worst_p = worst_e = 0.0
    try:
        for n in lengths:
            wav = _speech(n)
            e, p, _ = enc.embed_utterance(wav, return_partials=True)
            re, rp = o.embed_utterance(wav)
            assert p.shape == rp.shape, (n, p.shape, rp.shape)
            nw_p = float(np.linalg.norm(p - rp) / np.linalg.norm(rp))
            nw_e = float(np.linalg.norm(e - re) / np.linalg.norm(re))
            print(f"embed_utterance n={n} ({p.shape[0]} windows): normwise {nw_p:.2e} (partials), {nw_e:.2e} (embedding)")
            worst_p, worst_e = max(worst_p, nw_p), max(worst_e, nw_e)
            assert nw_p < E2E and nw_e < E2E, n
        print(f"embed_utterance vs float64 oracle: worst normwise {worst_p:.2e} (partials), {worst_e:.2e} (embedding); "
              f"threshold {E2E:.0e}")
        with pytest.raises(ValueError, match="longer than 180 s"):
            enc.embed_utterance(_speech(180 * SR + 1))
    finally:
        enc.close()
