"""GPU: the multi-band-diffusion vocoder as `TTS` builds it (fast_inference.py: MultiBandDiffusionEngine(max_seconds=30.0)
with the default MBDSettings: 4 band models, the full 20-call schedule, UNet widths 48 / 192 / 768 / 3072, tensor-core
convolutions, one stream per band model), at F = 12, 375 (5 s), 750 (10 s) and 2250 frames (30 s: 2250 x 320 = 720 000
samples, the workspace capacity), for n_samples = 320 F and 320 F - 7 (right padding to the stride and the final crop).
The checkpoint is synth.mbd_checkpoint of the default MBDConfig with bf16-representable convolution taps.

REFERENCE.  The restatement's own unet_forward, split_bands and re_eq (oracle/mbd_port.py) run on the device in float64
over the same data widened from fp32: the weights, mbd._lowpass_bank's fp32 taps (swapped in for the restatement's bank
by a wrapper), the fp32 schedule table the engine packs, and the supplied noise.

CHAIN IDENTITY.  One band model's sampler driven from Python through the hooks alone (mvb_mbd_unet_test, then
mvb_mbd_op_test op 7; op 10 for the initial sample, 8 for Philox draws, 2 / 4 for the processor, 9 or an accumulating
op 4 for the model sum, 2 / 3 / 4 for re-EQ) is bitwise equal to tokens_to_wav on the four-stream and the
MVB_MBD_ONE_STREAM engines.  So a UNet pass checked through the hook below is the pass tokens_to_wav runs.

TEACHER-FORCED PASSES.  Every call i of every band model m at every length: the engine's own fp32 cur_i goes to the
hook and to the float64 UNet.
Normwise bound of one pass, as a first-order sum over its stages of the bounds the op-level modules state and check:
  * each of the 25 convolutions (4 strided, 4 x 2 ResBlock convs in the encoders, conv_codec, 4 x 2 in the decoders,
    4 transposed) is within NORMWISE = 1e-4 of the float64 convolution of its own input, normwise
    (tests/test_mbd_conv_ops_gpu.py: the gamma-over-K_eff bound with the hi / lo split and the GroupNorm prologue
    elementwise, and 1e-4 normwise, at every width of this configuration);
  * each of the 24 GroupNorm statistics is within 2 u of float64 (u = 2^-24, tests/test_mbd_ops_gpu.py), which moves
    the normalised value by at most 4 u relative; the 4 materialised relu(GroupNorm) add 6 u; the interpolated
    condition and the 4 skip sums add one rounding (u) each;
  * GroupNorm renormalises every layer input and the residual sums add like-sized terms, so to first order a relative
    error entering one stage leaves the pass unamplified: the pass bound is the sum
        RHO = 25 NORMWISE + (24 * 4 + 4 * 6 + 5) u  =  2.5e-3 + 7.5e-6.
  The printed worst ratio per length is the check on that first-order model.
Elementwise, the last transposed convolution (48 -> 1, k8 s4) conditioned on its float64 input f = relu(p), p the
float64 decoder GroupNorm output: its own bound from test_mbd_conv_ops_gpu.py (gamma = 18 * 2 * 2 * 64 / 16 * 2^-23 over
conv(|f|, |W|), 2^-16 |f| for the hi / lo split of a perturbed f, 6 u (|p| + |gb|) for the prologue) plus the rest of the
pass carried in as an input error of RHO_up = RHO - NORMWISE relative to the prologue's magnitude,
|df| <= RHO_up (|p| + |gb| + |gw|), through conv(., |W|); plus 2^-23 |est| for the output rounding.

FREE-RUNNING.  The full 4-model, 20-call sampler plus the processors and re-EQ at F = 375 against the float64 chain
under the same noise; the tolerance is 10x the error measured on an H100.  tokens_to_wav(seed=s) at F = 2250 equals
tokens_to_wav(noise=) the Philox rows of streams m 1024 + r drawn by the randn hook, and those rows match the
host-recomputed Philox stream within the bound of tests/test_mbd_ops_gpu.py.

BOUNDARIES.  n_samples = max_samples + 1, n_frames = max_samples / 320 + 9 (past the condition buffer) and n_frames =
2 Tl + 1 (past the bottleneck rule) at 12 frames: MVB_ERR_ARG naming the value from tokens_to_wav and the hook (output
NaN-filled and untouched), ValueError from the Python wrapper; the limits themselves are accepted; the next valid call
on the same handle is bitwise equal to a fresh handle's.

SENSITIVITY.  References with the step embedding of the neighbouring schedule row, the condition shifted by one frame,
the ResBlock at dilation 2 (the default UNet has one ResBlock per level, at dilation 1), the right padding to the
stride moved to the left (without it the restatement's decoder cannot form the skip sums at 320 F - 7), and the
condition interpolated by rounding to the nearest frame instead of the floor of F.interpolate's nearest mode must each
put passes over the bound.

LONG OP-LEVEL CASES.  The op-level modules' cases at 30 s lengths with their bounds unchanged: level-0 k3 ResBlock conv
(C = 48, dilation 1 / 2 / 4), strided 48 -> 192 and transposed 48 -> 1 at Tin = 180 000 on the tensor cores, the CUDA-core
1 -> 48 encoder conv at Tin = 720 000, GroupNorm statistics at C = 48, T = 180 000, and k_fir_bank / k_band_std /
k_band_mix (both forms) at T = 720 000 for 4, 8 and 32 bands.

COST.  On an H100 80GB HBM3 at its 700 W limit the module runs in about 70 s (about 12 s of it building the checkpoint and
the engines) with 21.3 GiB peak device memory: the arena and the 30 s workspace of each engine (mvb_mbd_workspace_bytes:
3.85 GB with four activation blocks, 1.93 GB with one; both include the packed bf16 taps of the four band models), a
third engine for the boundary test, and the float64 weights of the reference (5 GB).  The float64 UNet pass at 30 s
(about 1.1 TFLOP) takes about 0.15 s there."""
import contextlib
import time

import pytest
import torch
import torch.nn.functional as F

import test_mbd_conv_ops_gpu as cv
import test_mbd_ops_gpu as ops
from mvb200 import synth
from oracle import mbd_port as M

pytestmark = pytest.mark.gpu

U24 = 2.0 ** -24
U23 = 2.0 ** -23
NORMWISE = cv.NORMWISE
N_CONV, N_GN, N_GN_RELU, N_ADD = 25, 24, 4, 5
RHO = N_CONV * NORMWISE + (N_GN * 4 + N_GN_RELU * 6 + N_ADD) * U24
RHO_UP = RHO - NORMWISE
FRAMES = [12, 375, 750, 2250]
SR = 24000
# Free-running float64 chain at F = 375 (test_free_running).  Measured on an H100 80GB HBM3 at its 700 W limit: normwise
# 6.2e-6, max-relative 7.5e-6; the thresholds are about 10x that.
FREE_NORMWISE, FREE_MAXREL = 7e-5, 8e-5


def _round_conv_weights_to_bf16(ck):
    for sd in ck["models"]:
        for k in list(sd):
            if sd[k].ndim == 3:
                sd[k] = sd[k].to(torch.bfloat16).to(torch.float32)
    return ck


class Prod:
    """The production engines over one checkpoint, the float64 reference data and the hooks."""

    def __init__(self):
        from mvb200 import _lib
        from mvb200.mbd import MBDSettings, MultiBandDiffusionEngine, _lowpass_bank, _schedule_table
        torch.cuda.reset_peak_memory_stats()
        self.t0 = time.perf_counter()
        self.L, self.lib = _lib, _lib.load()
        self.s = MBDSettings()
        self.ocfg = M.MBDConfig()
        self.ck = _round_conv_weights_to_bf16(synth.mbd_checkpoint(self.ocfg, 11))
        self.make = lambda **kw: MultiBandDiffusionEngine(self.ck, self.s, device="cuda:0", max_seconds=30.0, **kw)  # noqa: E731
        self.eng4 = self.make()
        self.eng1 = self.make(band_streams=False)
        assert self.eng4.cfg.options == 0 and self.eng4.cfg.max_samples == 720000
        self.rows = _schedule_table(self.s.schedule, self.s.steps())          # fp32 [20, 4]: a, b, sigma, step
        self.n_calls = self.rows.shape[0]
        self.ns, self.clip = float(self.s.schedule.noise_scale), float(self.s.schedule.clip)
        self.bank = {n: _lowpass_bank(n, SR).cuda().contiguous() for n in (self.s.proc_bands, self.s.eq_bands)}
        self.bank64 = {n: b.double() for n, b in self.bank.items()}
        self.proc = [(((pr["std"] / pr["target_std"]) ** self.s.power_std).float().cuda().contiguous(), pr["mean"].float().cuda().contiguous())
                     for pr in self.ck["proc"]]
        self.sd64 = [{k: v.double().cuda() for k, v in sd.items()} for sd in self.ck["models"]]

    # ---- hooks ----
    def unet(self, eng, m, call, cur, cond, n_frames=None, est=None):
        T = cur.numel()
        est = torch.empty(T, device="cuda") if est is None else est
        rc = self.lib.mvb_mbd_unet_test(eng._h, m, call, cur.data_ptr(), T, cond.data_ptr(),
                                        cond.shape[1] if n_frames is None else n_frames, est.data_ptr(), eng._st())
        return rc, est

    def sampler(self, eng, m, cond, noise_m, on_call=None):
        """Band model m's 20 calls through the hooks; on_call(i, cur_i, est_i) sees every call's input and estimate."""
        T = noise_m.shape[1]
        cur = torch.empty(T, device="cuda")
        ops._op(10, cur, a=noise_m[0], i1=T, f=(self.ns, 0, 0, 0, 0))
        for i, (a, b, sigma, _) in enumerate(self.rows.tolist()):
            rc, est = self.unet(eng, m, i, cur, cond)
            self.L.check(rc)
            if on_call is not None:
                on_call(i, cur, est)
            ops._op(7, cur, a=est, b=noise_m[i + 1] if sigma > 0 else None, i1=T, f=(a, b, sigma, self.ns, self.clip))
        return cur

    def processor(self, m, x, out, accumulate):
        nb, T = self.s.proc_bands, x.numel()
        low = torch.empty(nb - 1, T, device="cuda")
        ops._op(2, low, a=x, b=self.bank[nb], i0=nb - 1, i1=T, i2=self.bank[nb].shape[1])
        scale, mean = self.proc[m]
        ops._op(4, out, a=low, b=x, c=scale, e=mean, i0=nb, i1=T, i2=accumulate)

    def re_eq(self, wav, wav_e):
        nb, T = self.s.eq_bands, wav.numel()
        bank = self.bank[nb]
        lw, lr = torch.empty(nb - 1, T, device="cuda"), torch.empty(nb - 1, T, device="cuda")
        ops._op(2, lw, a=wav, b=bank, i0=nb - 1, i1=T, i2=bank.shape[1])
        ops._op(2, lr, a=wav_e, b=bank, i0=nb - 1, i1=T, i2=bank.shape[1])
        sw, sr = torch.empty(nb, device="cuda"), torch.empty(nb, device="cuda")
        ops._op(3, sw, a=lw, b=wav, i0=nb, i1=T)
        ops._op(3, sr, a=lr, b=wav_e, i0=nb, i1=T)
        out = torch.empty(T, device="cuda")
        ops._op(4, out, a=lw, b=wav, c=sr, d=sw, i0=nb, i1=T, i2=0)
        return out

    def hook_chain(self, eng, cond, wav_e, noise, four_blocks):
        T = wav_e.numel()
        nm = self.s.n_models
        if four_blocks:        # per-model outputs summed in model order by k_sum_blocks
            stride = T + 64
            blocks = torch.empty(nm * stride, device="cuda")
            for m in range(nm):
                x = self.sampler(eng, m, cond, noise[m])
                self.processor(m, x, blocks[m * stride:m * stride + T], 0)
            want = blocks[:T].clone()
            for m in range(1, nm):
                want = want + blocks[m * stride:m * stride + T]
            ops._op(9, blocks, i0=nm, i1=T, i2=stride)
            assert torch.equal(blocks[:T], want), "k_sum_blocks differs from the fp32 sum in model order"
            wav = blocks[:T]
        else:                  # accumulated in place by the processor's band mix
            wav = torch.zeros(T, device="cuda")
            for m in range(nm):
                self.processor(m, self.sampler(eng, m, cond, noise[m]), wav, 1)
        return self.re_eq(wav.contiguous(), wav_e)


@pytest.fixture(scope="module")
def P():
    p = Prod()
    yield p
    print(f"production MBD module: {time.perf_counter() - p.t0:.1f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    p.eng4.close()
    p.eng1.close()


def _inputs(F_, T, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    cond = torch.randn(128, F_, generator=g, device="cuda")
    noise = torch.randn(4, 20, T, generator=g, device="cuda")
    wav_e = torch.from_numpy(synth.synthetic_waveform(F_ * 320 / SR, SR, seed=seed))[:T].float().cuda().contiguous()
    return cond, noise, wav_e


# ---- the float64 restatement, with wrappers -------------------------------------------------------------------------
class _FProxy:
    """torch.nn.functional for oracle/mbd_port.py with some functions replaced (variants and recording)."""

    def __init__(self, **over):
        self._over = over

    def __getattr__(self, k):
        return self._over[k] if k in self._over else getattr(F, k)


@contextlib.contextmanager
def _patched(**attrs):
    old = {k: getattr(M, k) for k in attrs}
    for k, v in attrs.items():
        setattr(M, k, v)
    try:
        yield
    finally:
        for k, v in old.items():
            setattr(M, k, v)


def unet64(P, m, call, cur, cond, variant=None):
    """(est [T], p) float64: the restatement's unet_forward; p is the input of the last decoder GroupNorm's relu (the
    last transposed convolution's prologue output)."""
    step = int(P.rows[call, 3])
    rec = {}

    def gn(x, *a, **k):
        y = F.group_norm(x, *a, **k)
        rec["p"] = y
        return y

    over = dict(group_norm=gn)
    res = orig_res = M._res_block
    c64 = cond.double()[None]
    if variant == "neighbour_step":
        step = int(P.rows[call + 1 if call + 1 < P.n_calls else call - 1, 3])
    elif variant == "cond_shift":
        c64 = torch.cat([c64[..., :1], c64[..., :-1]], -1)
    elif variant == "dilation":
        res = lambda sd, p, x, g, d: orig_res(sd, p, x, g, 2 * d)  # noqa: E731
    elif variant == "left_pad":
        over["pad"] = lambda x, p, *a, **k: F.pad(x, (p[1], p[0]), *a, **k) if not a and not k else F.pad(x, p, *a, **k)
    elif variant == "round_interp":
        def interp(x, size):
            tf = x.shape[-1]
            src = torch.round(torch.arange(size, dtype=torch.float64, device=x.device) * (tf / size)).long().clamp(max=tf - 1)
            return x[..., src]
        over["interpolate"] = interp
    with _patched(F=_FProxy(**over), _res_block=res):
        est = M.unet_forward(P.sd64[m], P.ocfg.unet, cur.double().view(1, 1, -1), step, c64)
    return est.view(-1), rec["p"][0]


def last_layer_bound(P, m, p, est_ref):
    """Elementwise bound of the module docstring for the last transposed convolution, conditioned on its float64 input."""
    sd = P.sd64[m]
    key = f"decoders.{P.ocfg.unet.depth - 1}."
    gw, gb, W = sd[key + "norm.weight"][:, None], sd[key + "norm.bias"][:, None], sd[key + "convtr.weight"]
    f = torch.relu(p)
    k, s = P.ocfg.unet.kernel, P.ocfg.unet.stride
    pad = (k - s) // 2
    A = cv._conv(2, f.abs(), W.abs(), s, 1, pad)
    ef = RHO_UP * (p.abs() + gb.abs() + gw.abs()) + 6 * U24 * (p.abs() + gb.abs()) + 2.0 ** -16 * f.abs()
    gam = cv._gamma(2, p.shape[0], k, True)
    bound = gam * A + cv._conv(2, ef, W.abs(), s, 1, pad)
    T = est_ref.numel()
    return bound[0, :T] + U23 * est_ref.abs() + 1e-30


def check_pass(P, m, call, cur, est, cond, variant=None):
    """(normwise / RHO, elementwise |err| / bound max, elements over) of one pass."""
    ref, p = unet64(P, m, call, cur, cond, variant)
    got = est.double()
    err = (got - ref).abs()
    bound = last_layer_bound(P, m, p, ref)
    return float(err.norm() / ref.norm()) / RHO, float((err / bound).max()), int((err > bound).sum())


# ---- chain identity ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F_,T", [(375, 375 * 320 - 7), (2250, 2250 * 320)])
def test_hook_chain_equals_tokens_to_wav(P, F_, T):
    cond, noise, wav_e = _inputs(F_, T, 1000 + F_)
    for name, eng, four in (("four streams", P.eng4, True), ("one stream", P.eng1, False)):
        want = eng.tokens_to_wav(cond, wav_e, noise=noise)
        got = P.hook_chain(eng, cond, wav_e, noise, four)
        print(f"hook chain vs tokens_to_wav, {name}, F={F_} T={T}: {int((got != want).sum())} of {T} samples differ")
        assert torch.isfinite(want).all() and torch.equal(got, want)


# ---- teacher-forced UNet passes ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("F_", FRAMES)
def test_teacher_forced_passes(P, F_):
    t0 = time.perf_counter()
    for T in (320 * F_, 320 * F_ - 7):
        cond, noise, _ = _inputs(F_, T, 2000 + T)
        worst = [0.0, 0.0]
        fails = []

        def on_call(i, cur, est, m):
            nw, el, n_over = check_pass(P, m, i, cur, est, cond)
            worst[0], worst[1] = max(worst[0], nw), max(worst[1], el)
            if nw >= 1 or n_over:
                fails.append((m, i, nw, el, n_over))

        for m in range(P.s.n_models):
            P.sampler(P.eng4, m, cond, noise[m], lambda i, cur, est: on_call(i, cur, est, m))
        print(f"teacher-forced F={F_} T={T}: {P.s.n_models} models x {P.n_calls} calls: worst normwise / RHO {worst[0]:.3e} "
              f"(RHO {RHO:.3e}), worst last-layer |err| / bound {worst[1]:.3e}")
        assert not fails, f"passes over the bound (model, call, normwise / RHO, elementwise ratio, elements over): {fails[:5]}"
    print(f"teacher-forced F={F_}: {time.perf_counter() - t0:.1f} s")


# ---- sensitivity ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["neighbour_step", "cond_shift", "dilation", "left_pad", "round_interp"])
def test_altered_references_violate(P, variant):
    for F_ in (12, 375):
        T = 320 * F_ - 7
        cond, noise, _ = _inputs(F_, T, 3000 + F_)
        seen = []

        def on_call(i, cur, est):
            if i in (1, 10):
                seen.append((i,) + check_pass(P, 0, i, cur, est, cond, variant))

        P.sampler(P.eng4, 0, cond, noise[0], on_call)
        print(f"altered reference {variant} F={F_}: " + ", ".join(f"call {i}: normwise / RHO {nw:.2e}, {n} elements over"
                                                                  for i, nw, _, n in seen))
        assert all(nw > 1 or n > 0 for _, nw, _, n in seen), f"{variant}: a pass within the bound at F={F_}"


# ---- free-running chain -----------------------------------------------------------------------------------------------
def free_running64(P, cond, wav_e, noise):
    sr = P.ocfg.sample_rate
    banks = lambda n, _sr: P.bank64[n]  # noqa: E731
    wav = torch.zeros(wav_e.numel(), dtype=torch.float64, device="cuda")
    c64 = cond.double()
    with _patched(lowpass_bank=banks):
        for m in range(P.s.n_models):
            cur = noise[m, 0].double() * P.ns
            for i, (a, b, sigma, _) in enumerate(P.rows.double().tolist()):
                est, _ = unet64(P, m, i, cur, c64)
                cur = (cur - a * est * P.ns) * b
                if sigma > 0:
                    cur = cur + sigma * noise[m, i + 1].double() * P.ns
                cur = cur.clamp(-P.clip, P.clip)
            scale, mean = P.proc[m]
            bands = M.split_bands(cur, P.s.proc_bands, sr)
            wav = wav + (bands * scale.double()[:, None] + mean.double()[:, None]).sum(0)
        return M.re_eq(wav, wav_e.double(), P.s.eq_bands, sr)


def test_free_running(P):
    F_ = 375
    T = 320 * F_ - 7
    t0 = time.perf_counter()
    cond, noise, wav_e = _inputs(F_, T, 4000)
    got = P.eng4.tokens_to_wav(cond, wav_e, noise=noise).double()
    ref = free_running64(P, cond, wav_e, noise)
    nw = float((got - ref).norm() / ref.norm())
    mr = float((got - ref).abs().max() / ref.abs().max())
    print(f"free-running 4 models x 20 calls + re-EQ, F={F_} T={T}: normwise {nw:.3e} (tolerance {FREE_NORMWISE:.1e}), "
          f"max-relative {mr:.3e} (tolerance {FREE_MAXREL:.1e}); {time.perf_counter() - t0:.1f} s")
    assert nw < FREE_NORMWISE and mr < FREE_MAXREL


def test_seeded_noise_at_capacity(P):
    """tokens_to_wav(seed=) at 30 s equals tokens_to_wav(noise=) with the randn hook's rows of streams m 1024 + r; rows 0
    and 19 of every band model also against the host-recomputed Philox stream."""
    F_, seed = 2250, 2 ** 33 + 17
    T = 320 * F_
    cond, _, wav_e = _inputs(F_, T, 5000)
    noise = torch.empty(4, P.n_calls, T, device="cuda")
    for m in range(4):
        for r in range(P.n_calls):
            ops._op(8, noise[m, r], i1=T, i2=m * 1024 + r, seed=seed)
            if r in (0, P.n_calls - 1):
                ref, rad = ops._randn_reference(T, seed, m * 1024 + r)
                ops._check(f"randn T={T} stream {m * 1024 + r}", noise[m, r].cpu(), ref, 5 * U24 * ref.abs() + 1e-15 * rad + 1e-30)
    a = P.eng4.tokens_to_wav(cond, wav_e, seed=seed)
    b = P.eng4.tokens_to_wav(cond, wav_e, noise=noise)
    assert torch.isfinite(a).all() and torch.equal(a, b)


# ---- boundaries (after the up-front checks) ---------------------------------------------------------------------------
def test_rejected_shapes(P):
    eng, lib = P.eng4, P.lib
    cap = eng.cfg.max_samples
    tl = lambda n: -(-n // 4 ** 4)  # noqa: E731
    short = 12 * 320 - 7
    cases = [(12, cap + 1, str(cap + 1)), (cap // 320 + 9, cap, str(cap // 320 + 9)), (2 * tl(short) + 1, short, str(2 * tl(short) + 1))]
    for nf, ns, name in cases:
        cond = torch.randn(128, nf, device="cuda")
        wav_e = torch.zeros(ns, device="cuda")
        out = torch.full((ns,), float("nan"), device="cuda")
        rc = lib.mvb_mbd_tokens_to_wav(eng._h, cond.data_ptr(), nf, wav_e.data_ptr(), ns, None, 7, out.data_ptr(), eng._st())
        msg = lib.mvb_last_error().decode()
        torch.cuda.synchronize()
        print(f"tokens_to_wav(n_frames={nf}, n_samples={ns}): rc {rc}, {msg!r}")
        assert rc == P.L.MVB_ERR_ARG and name in msg and torch.isnan(out).all()
        rc, est = P.unet(eng, 0, 0, wav_e, cond, est=out)
        msg = lib.mvb_last_error().decode()
        print(f"mvb_mbd_unet_test(n_frames={nf}, n_samples={ns}): rc {rc}, {msg!r}")
        assert rc == P.L.MVB_ERR_ARG and name in msg and torch.isnan(est).all()
        with pytest.raises(ValueError, match=name):
            eng.tokens_to_wav(cond.cpu(), wav_e.cpu())
    # the limits themselves are accepted
    for nf, ns in ((cap // 320 + 8, cap), (2 * tl(short), short)):
        rc, est = P.unet(eng, 0, 0, torch.randn(ns, device="cuda"), torch.randn(128, nf, device="cuda"))
        assert rc == P.L.MVB_OK and torch.isfinite(est).all(), (nf, ns, rc)
    for m, c in ((4, 0), (-1, 0), (0, 20), (0, -1)):
        rc, _ = P.unet(eng, m, c, torch.zeros(short, device="cuda"), torch.zeros(128, 12, device="cuda"))
        assert rc == P.L.MVB_ERR_ARG, (m, c)
    # the next valid call on the same handle equals the same call on a fresh handle
    cond, noise, wav_e = _inputs(12, short, 6000)
    a = eng.tokens_to_wav(cond, wav_e, noise=noise)
    fresh = P.make()
    b = fresh.tokens_to_wav(cond, wav_e, noise=noise)
    fresh.close()
    assert torch.isfinite(a).all() and torch.equal(a, b)


# ---- long op-level cases ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dil", [1, 2, 4])
def test_level0_resblock_conv_30s(dil):
    cv._case(f"resblock k3 C=48 T=180000 dil={dil}", 0, 48, 48, 3, 1, dil, dil, 180000, bias=True, emb=True, resid=True, seed=70 + dil)


def test_level0_strided_and_transposed_30s():
    cv._case("strided 48->192 Tin=180000", 1, 48, 192, 8, 4, 1, 2, 180000, gn=False, seed=74)
    cv._case("transposed 48->1 Tin=180000", 2, 48, 1, 8, 4, 1, 2, 180000, seed=75)
    cv._case("strided 1->48 Tin=720000", 1, 1, 48, 8, 4, 1, 2, 720000, gn=False, use_tc=False, seed=76)
    cv._case("strided 1->48 Tin=719993", 1, 1, 48, 8, 4, 1, 2, 719993, gn=False, use_tc=False, seed=77)


def test_gn_stats_30s():
    x = ops._rand((48, 180000), 78, 1.0, 0.2)
    ops._gn_case("gn C=48 T=180000", x, 4, strict=True)


@pytest.mark.parametrize("n_bands", [4, 8, 32])
def test_band_kernels_30s(n_bands):
    T = 720000
    ops.test_fir_bank(n_bands, T)
    for dc in (0.0, 100.0):
        ops.test_band_std(n_bands, T, dc)
    for form in ("processor", "re_eq"):
        for acc in (0, 1):
            ops.test_band_mix(n_bands, form, acc, T)
