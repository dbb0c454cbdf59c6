"""GPU: the multi-band-diffusion kernels other than the convolutions (csrc/mbd.cu) one launch at a time through
mvb_mbd_op_test, each against a float64 reference of the same operation, plus two engine-level identities.

u = 2^-24 is the fp32 unit roundoff and e = 2^-53 the fp64 one; g_k = k e / (1 - k e).  Every output buffer sits between
NaN guards: a kernel must write every element of its output and nothing outside it.  Bounds are elementwise:

GroupNorm statistics (k_gn_partial + k_gn_final).  The reference is the float64 two-pass mean and 1 / sqrt(var + eps)
(biased variance, eps = fp32 1e-5 widened to double).  The kernel sums v and v^2 (both exact in fp64 for fp32 v) in one
pass: a per-thread strided sum of m = ceil(ceil(n / 64) / 256) terms (m - 1 roundings), a 5-level shuffle, 8 warp
totals (7), the two partials of each lane (1) and a 5-level shuffle: depth d = m + 17, so |dS| <= g_d sum|v|,
|dQ| <= g_d Q.  With the divisions by n, Em = g_(d+1) sum|v| / n, and
    Evar = g_(d+2) Q / n + 2 |mean| Em + Em^2 + 2 e (|mean| + Em)^2,
    Er   = 1 / sqrt(var + eps - Evar) - 1 / sqrt(var + eps) + 4 e rstd   (eps add, sqrt, divide),
and the fp32 results carry one more rounding: bound = u |ref| + (1 + u) E.  The one-pass cancellation makes Evar grow with
(mean / std)^2: up to mean / std = 1e3 at every production shape E stays below u |ref|, and the tests also require
|err| <= 2 u |ref| there.  At mean / std = 1e5 the bound is ~1e3 u on rstd and the kernel's error is several u (printed):
GroupNorm inputs that far off centre lose that many bits of rstd.  The MBD UNet feeds GroupNorm conv outputs and ReLU
activations with mean / std of order 1.

relu(GroupNorm) in place (k_gn_relu_inplace): a = fl(fl(x - m) r) reproduced in fp32, then relu(a gw + gb) in float64;
the kernel rounds the last step once or twice: 6 u (|a gw| + |gb|), the prologue bound of tests/test_mbd_conv_ops_gpu.py.

FIR bank (k_fir_bank through split_lows): float64 correlation of the same fp32 bank (mbd._lowpass_bank) with the input
padded by replicating its end samples; one fmaf per tap from zero: (L + 1) u sum_j |f_j| |x_clamp(t + j - half)|.

Band std (k_band_std): the bands are the fp32 differences the kernel forms, fl(low[b] - low[b - 1]) and
fl(x - low[n - 2]), reproduced exactly; the reference is their float64 two-pass unbiased std.  One pass over T with
depth d = ceil(T / 256) + 11: |dS| <= g_d A, |dQ| <= g_d Q, and
    Evar = (g_(d+1) Q + (2 |S| dS + dS^2) / T + 3 e S^2 / T) / (T - 1) + 2 e var,
    Estd = sqrt(var) - sqrt(max(var - Evar, 0)) + e std;   bound = u std + (1 + u) Estd.

Band mix (k_band_mix): out (+)= sum_b band_b fl(num_b / den_b) + shift_b, accumulated sequentially in fp32 (fp32 division
is correctly rounded and reproduced exactly): (2 n + 1) u sum_b (|band_b scale_b| + |shift_b|), plus u |out| when
accumulating.

Schedule step (k_sched_step): v = (cur - a (est ns)) b + (sigma noise) ns, clamped to +-clip when clip > 0.  Without
contraction the first term takes four roundings, 4 u |b| (|cur| + |a est ns|), the noise term two, and the sum one, so
|err| <= 5 u (|b| (|cur| + |a est ns|) + |sigma noise ns|); an FMA only removes roundings.  The clamp is 1-Lipschitz, so
the same bound holds after it, including at and beyond +-clip.

randn (k_randn): the Philox4x32-10 words are recomputed on the host (counter (i, stream, 0x6d6264, 0), key (seed lo,
seed hi)); u1, u2 = ((w >> 8) + 0.5) 2^-24 are reproduced exactly in fp32, then Box-Muller in float64.  logf and
sincospif are within 1 ulp (2 u relative), sqrtf and the final product are correctly rounded: rad = sqrt(-2 log u1) is
within 2 u (half the logf error, plus u), cos / sin within 2 u, the product adds u: bound = 5 u |ref| + 1e-15 rad (the
float64 cos / sin of 2 pi u2 near a zero crossing, where |ref| >= 2 pi 2^-25 rad).

add_interp, add_crop, sum_blocks and scale_copy do one fp32 operation per element in a fixed order: bitwise equal to
PyTorch fp32 (add_interp against F.interpolate(mode="nearest") on the CPU)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
E64 = 2.0 ** -53
GUARD = 1024
EPS = float(np.float32(1e-5))
# default MBDSettings (hidden 48, growth 4, depth 4): level widths and lengths at 12 frames (3833 samples) and 6 s
WIDTHS = [48, 192, 768, 3072]
LEVELS = {3833: [959, 240, 60, 15], 144000: [36000, 9000, 2250, 563]}


def _g(k):
    return k * E64 / (1 - k * E64)


def _lib():
    from mvb200 import _lib as L
    return L, L.load()


def _op(op, out, a=None, b=None, c=None, d=None, e=None, i0=0, i1=0, i2=0, f=(0.0, 0.0, 0.0, 0.0, 0.0), seed=0):
    L, lib = _lib()
    p = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.check(lib.mvb_mbd_op_test(op, p(a), p(b), p(c), p(d), p(e), out.data_ptr(), i0, i1, i2, *[float(v) for v in f],
                                int(seed) & (2 ** 64 - 1), st))


def _guarded(n, init=None):
    buf = torch.full((2 * GUARD + n,), float("nan"), device="cuda")
    if init is not None:
        buf[GUARD:GUARD + n] = init.reshape(-1)
    return buf, buf[GUARD:GUARD + n]


def _unguard(buf, n, label):
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + n:]).all(), f"{label}: write outside the output"
    out = buf[GUARD:GUARD + n]
    assert not torch.isnan(out).any(), f"{label}: output elements not written"
    return out


def _check(label, got, ref, bound):
    err = (got.double() - ref).abs()
    ratio = float((err / bound).max())
    print(f"{label}: max |err|/bound {ratio:.3e}")
    bad = (err > bound).nonzero()
    assert bad.numel() == 0, f"{label}: {bad.shape[0]} elements over the bound, first at {bad[0].tolist()}"
    return ratio


def _rand(shape, seed, scale=1.0, offset=0.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=g, device="cuda") * scale + offset


# ---- GroupNorm statistics -------------------------------------------------------------------------------------------
def _gn_hook(x, groups, eps=EPS):
    buf, _ = _guarded(2 * groups)
    _op(0, buf[GUARD:], a=x, i0=x.shape[0], i1=x.shape[1], i2=groups, f=(eps, 0, 0, 0, 0))
    return _unguard(buf, 2 * groups, "gn stats").view(groups, 2)


def _gn_reference(x, groups, eps=EPS):
    """(mean, rstd, bound on mean, bound on rstd), float64 [groups] each."""
    xg = x.double().view(groups, -1)
    n = xg.shape[1]
    mean = xg.mean(1)
    var = ((xg - mean[:, None]) ** 2).mean(1)
    rstd = 1.0 / torch.sqrt(var + eps)
    d = -(-(-(-n // 64)) // 256) + 17
    A, Q = xg.abs().sum(1), (xg * xg).sum(1)
    Em = _g(d + 1) * A / n
    Evar = _g(d + 2) * Q / n + 2 * mean.abs() * Em + Em ** 2 + 2 * E64 * (mean.abs() + Em) ** 2
    lo = (var + eps - Evar).clamp(min=1e-300)
    Er = 1.0 / torch.sqrt(lo) - rstd + 4 * E64 * rstd
    return mean, rstd, U * mean.abs() + (1 + U) * Em, U * rstd + (1 + U) * Er


def _gn_case(label, x, groups, strict):
    got = _gn_hook(x, groups)
    mean, rstd, bm, br = _gn_reference(x, groups)
    rm = _check(f"{label} mean", got[:, 0], mean, bm)
    rr = _check(f"{label} rstd", got[:, 1], rstd, br)
    e2m = float(((got[:, 0].double() - mean).abs() / (U * mean.abs())).max())
    e2r = float(((got[:, 1].double() - rstd).abs() / (U * rstd)).max())
    print(f"{label}: |err| in u of |ref|: mean {e2m:.2f}, rstd {e2r:.2f}")
    if strict:
        assert e2m <= 2 and e2r <= 2, f"{label}: more than 2 u from the reference"
    return rm, rr, e2m, e2r


@pytest.mark.parametrize("T", [3833, 144000])
@pytest.mark.parametrize("lvl", [0, 1, 2, 3])
@pytest.mark.parametrize("mean,std", [(0.2, 1.0), (1e3, 1.0), (-300.0, 0.3)])
def test_gn_stats_production(T, lvl, mean, std):
    C, t = WIDTHS[lvl], LEVELS[T][lvl]
    x = _rand((C, t), 100 * lvl + T % 97, std, mean)
    _gn_case(f"gn C={C} T={t} mean/std={mean / std:g}", x, 4, strict=True)


@pytest.mark.parametrize("C,T,groups", [(1, 1, 1), (1, 63, 1), (4, 15, 4), (3, 5, 3), (96, 1, 32), (96, 300, 1),
                                        (96, 300, 3), (96, 300, 4), (96, 300, 32), (64, 1, 64)])
def test_gn_stats_edges(C, T, groups):
    """n < GN_SPLIT (empty splits) down to one element (var 0, rstd = 1 / sqrt(eps)); 1, 3, 4, 32 (and the hook's 64)
    groups."""
    x = _rand((C, T), C * 1000 + T + groups, 1.5, 0.4)
    _gn_case(f"gn edge C={C} T={T} groups={groups}", x, groups, strict=False)
    if C * T == groups:
        got = _gn_hook(x, groups)
        assert torch.equal(got[:, 0], x.reshape(-1)) and torch.equal(got[:, 1], torch.full_like(got[:, 1], float(1 / math.sqrt(EPS))))


def test_gn_stats_constant_group():
    """A group that is exactly constant: var = 0 up to the fp64 round-off of Q, rstd = 1 / sqrt(eps) to fp32."""
    x = _rand((96, 1000), 3, 1.0, 0.0)
    x[24:48] = 0.3
    x[72:96] = -1234.5
    got = _gn_hook(x, 4)
    _gn_case("gn constant groups", x, 4, strict=False)
    r0 = np.float32(1 / math.sqrt(EPS))
    assert got[1, 0].item() == np.float32(0.3) and got[3, 0].item() == -1234.5
    assert abs(got[1, 1].item() - r0) <= 2 * U * r0


def test_gn_stats_far_off_centre():
    """mean / std = 1e5: the one-pass fp64 formula loses ~(mean / std)^2 e of var; reported against 2 u, bounded by the
    derived (honest) bound."""
    rows = []
    for lvl in (0, 3):
        x = _rand((WIDTHS[lvl], LEVELS[3833][lvl]), 7 + lvl, 1.0, 1e5)
        rows.append(_gn_case(f"gn C={WIDTHS[lvl]} mean/std=1e5", x, 4, strict=False))
    print("mean/std = 1e5: worst |err| on rstd = %.1f u (mean %.2f u)" % (max(r[3] for r in rows), max(r[2] for r in rows)))


# ---- relu(GroupNorm) in place ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,T,groups", [(48, 959, 4), (192, 240, 4), (768, 60, 4), (3072, 15, 4), (48, 36000, 4),
                                        (96, 301, 1), (96, 301, 3), (96, 301, 32)])
def test_gn_relu_inplace(C, T, groups):
    x = _rand((C, T), C + T + groups, 1.3, 0.25)
    g = torch.Generator(device="cuda").manual_seed(C)
    gw = 1 + 0.2 * torch.randn(C, generator=g, device="cuda")
    gb = 0.1 * torch.randn(C, generator=g, device="cuda")
    stats = _gn_hook(x, groups).contiguous()
    buf, _ = _guarded(C * T, x)
    _op(1, buf[GUARD:], a=stats, b=gw, c=gb, i0=C, i1=T, i2=groups)
    got = _unguard(buf, C * T, "gn relu").view(C, T)
    m = stats[:, 0].repeat_interleave(C // groups)[:, None]
    r = stats[:, 1].repeat_interleave(C // groups)[:, None]
    a = (x - m) * r
    agw = a.double() * gw.double()[:, None]
    ref = torch.relu(agw + gb.double()[:, None])
    _check(f"gn relu C={C} T={T} groups={groups}", got, ref, 6 * U * (agw.abs() + gb.double().abs()[:, None]) + 1e-30)


# ---- FIR bank -------------------------------------------------------------------------------------------------------
def _bank(n_bands):
    from mvb200.mbd import _lowpass_bank
    return _lowpass_bank(n_bands, 24000).cuda().contiguous()


def _xcorr(x, w):
    """out[f][t] = sum_j w[f][j] x[t + j] for t < len(x) - L + 1, float64 via FFT."""
    n, L = x.shape[-1], w.shape[-1]
    N = 1 << (n + L).bit_length()
    y = torch.fft.irfft(torch.fft.rfft(x, N)[None, :] * torch.conj(torch.fft.rfft(w, N)), N)
    return y[:, :n - L + 1]


def _fir_reference(x, bank):
    L = bank.shape[1]
    half = (L - 1) // 2
    T = x.shape[0]
    idx = torch.arange(-half, T + half, device=x.device).clamp(0, T - 1)
    xp = x.double()[idx]
    w = bank.double()
    ref = _xcorr(xp, w)
    bound = (L + 1) * U * _xcorr(xp.abs(), w.abs()).clamp(min=0) + 1e-30
    # the FFT's own round-off (~1e-16 of the l2 norms) stays far below the bound; keep it explicit
    bound = bound + 1e-13 * float(xp.abs().max()) * float(w.abs().sum(1).max())
    return ref, bound


def _fir_hook(x, bank):
    nf, L = bank.shape
    T = x.shape[0]
    buf, _ = _guarded(nf * T)
    _op(2, buf[GUARD:], a=x, b=bank, i0=nf, i1=T, i2=L)
    return _unguard(buf, nf * T, "fir").view(nf, T)


@pytest.mark.parametrize("n_bands", [2, 8, 32, 64])
@pytest.mark.parametrize("T", [64, 1023, 1024, 1025, 3833, 144000])
def test_fir_bank(n_bands, T):
    """Both production banks (8 bands / 629 taps, 32 / 2893), 2 bands, and 64 (5921 taps, more than 64 KB of shared
    memory); every nf is odd, so the last CTA has no second filter and row nf must stay untouched.  T = 64 is far
    shorter than half a filter: nearly every tap reads replicate padding."""
    bank = _bank(n_bands)
    x = _rand((T,), T + n_bands, 0.5, 0.05)
    if T >= 1024:
        x = x + 0.3 * torch.sin(torch.arange(T, device="cuda") * 0.01)
    got = _fir_hook(x, bank)
    ref, bound = _fir_reference(x, bank)
    _check(f"fir {n_bands} bands ({bank.shape[1]} taps) T={T}", got, ref, bound)


# ---- band std / band mix --------------------------------------------------------------------------------------------
def _bands32(low, x):
    """The fp32 bands k_band_std / k_band_mix form: low[0], fl(low[b] - low[b-1]), fl(x - low[n-2])."""
    rows = [low[0]] + [low[b] - low[b - 1] for b in range(1, low.shape[0])] + [x - low[-1]]
    return torch.stack(rows)


def _signal(T, seed, dc=0.0):
    t = torch.arange(T, device="cuda", dtype=torch.float64)
    x = _rand((T,), seed, 0.2) + (0.5 * torch.sin(t * 0.003) + 0.3 * torch.sin(t * 0.7)).float()
    return (x + dc).contiguous()


@pytest.mark.parametrize("n_bands", [2, 8, 32, 64])
@pytest.mark.parametrize("T,dc", [(3833, 0.0), (3833, 100.0), (144000, 0.0), (144000, 100.0)])
def test_band_std(n_bands, T, dc):
    """Unbiased per-band std; with a DC offset 100x the AC content band 0 carries it and the one-pass formula cancels."""
    x = _signal(T, n_bands + T, dc)
    low = _fir_hook(x, _bank(n_bands)).contiguous()
    buf, _ = _guarded(n_bands)
    _op(3, buf[GUARD:], a=low, b=x, i0=n_bands, i1=T)
    got = _unguard(buf, n_bands, "band std")
    v = _bands32(low, x).double()
    mean = v.mean(1)
    var = ((v - mean[:, None]) ** 2).sum(1) / (T - 1)
    std = var.sqrt()
    d = -(-T // 256) + 11
    A, Q, S = v.abs().sum(1), (v * v).sum(1), v.sum(1)
    dS = _g(d) * A
    Evar = (_g(d + 1) * Q + (2 * S.abs() * dS + dS ** 2) / T + 3 * E64 * S ** 2 / T) / (T - 1) + 2 * E64 * var
    Estd = std - (var - Evar).clamp(min=0).sqrt() + E64 * std
    _check(f"band std {n_bands} bands T={T} dc={dc:g}", got, std, U * std + (1 + U) * Estd + 1e-30)


@pytest.mark.parametrize("n_bands", [2, 8, 32, 64])
@pytest.mark.parametrize("form", ["processor", "re_eq"])
@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("T", [3833, 144000])
def test_band_mix(n_bands, form, accumulate, T):
    """Processor form (den = NULL, with shift) and re-EQ form (num / den, no shift), overwriting and accumulating."""
    x = _signal(T, 3 * n_bands + T, 0.0 if form == "processor" else 0.7)
    low = _fir_hook(x, _bank(n_bands)).contiguous()
    g = torch.Generator(device="cuda").manual_seed(n_bands + accumulate)
    num = (0.5 + torch.rand(n_bands, generator=g, device="cuda")).contiguous()
    den = (0.2 + torch.rand(n_bands, generator=g, device="cuda")).contiguous() if form == "re_eq" else None
    shift = (0.05 * torch.randn(n_bands, generator=g, device="cuda")).contiguous() if form == "processor" else None
    prev = _rand((T,), 11 + T, 0.4)
    buf, _ = _guarded(T, prev if accumulate else None)
    _op(4, buf[GUARD:], a=low, b=x, c=num, d=den, e=shift, i0=n_bands, i1=T, i2=accumulate)
    got = _unguard(buf, T, "band mix")
    scale = (num / den if den is not None else num).double()
    terms = _bands32(low, x).double() * scale[:, None]
    absum = terms.abs().sum(0)
    ref = terms.sum(0)
    if shift is not None:
        ref = ref + shift.double().sum()
        absum = absum + shift.double().abs().sum()
    bound = (2 * n_bands + 1) * U * absum
    if accumulate:
        ref = ref + prev.double()
        bound = bound + U * ref.abs()
    _check(f"band mix {form} {n_bands} bands T={T} accumulate={accumulate}", got, ref, bound + 1e-30)


# ---- add_interp, add_crop, sum_blocks, scale_copy: bitwise --------------------------------------------------------
def _interp_pairs():
    pairs = set()
    for Tf in list(range(1, 401)) + [1500]:
        for r in (0, 7):
            T = 320 * Tf - r
            for down in (4 ** 4, 4 ** 2, 2 ** 4):      # default UNet (k8 s4, depth 4), depth 2, and (k4, s2) depth 4
                Tz = -(-T // down)
                if Tf <= 2 * Tz:
                    pairs.add((Tf, Tz))
        pairs.add((Tf, Tf))
        pairs.add((Tf, 2 * Tf))
    return sorted(pairs)


def test_add_interp_bitexact():
    """Every (Tf, Tz) tokens_to_wav produces for Tf = 1 .. 400 and 1500 frames (T = 320 Tf - r, r in {0, 7}), plus
    Tz = Tf and 2 Tf: z + F.interpolate(cond, Tz, mode="nearest") in fp32 on the CPU, bit for bit."""
    pairs = _interp_pairs()
    Cn = 3
    g = torch.Generator().manual_seed(0)
    n_bad = []
    for Tf, Tz in pairs:
        cond = torch.randn(Cn, Tf, generator=g)
        z = torch.randn(Cn, Tz, generator=g)
        buf, _ = _guarded(Cn * Tz, z.cuda())
        _op(5, buf[GUARD:], a=cond.cuda(), i0=Cn, i1=Tz, i2=Tf)
        got = _unguard(buf, Cn * Tz, f"interp {Tf}->{Tz}").view(Cn, Tz).cpu()
        want = z + F.interpolate(cond[None], size=Tz, mode="nearest")[0]
        if not torch.equal(got, want):
            n_bad.append((Tf, Tz))
    print(f"add_interp: {len(pairs)} (Tf, Tz) pairs, {len(n_bad)} mismatches")
    assert not n_bad, f"add_interp differs from F.interpolate at {n_bad[:10]}"
    # the bottleneck width at 30 s (T = 480000: Tz = 1875)
    cond = torch.randn(3072, 1500, generator=g)
    z = torch.randn(3072, 1875, generator=g)
    buf, _ = _guarded(z.numel(), z.cuda())
    _op(5, buf[GUARD:], a=cond.cuda(), i0=3072, i1=1875, i2=1500)
    got = _unguard(buf, z.numel(), "interp 3072").view(3072, 1875).cpu()
    assert torch.equal(got, z + F.interpolate(cond[None], size=1875, mode="nearest")[0])


@pytest.mark.parametrize("C,Ts,Tz", [(1, 1, 1), (3, 7, 8), (48, 3833, 3836), (3072, 15, 16), (192, 959, 960)])
def test_add_crop_bitexact(C, Ts, Tz):
    z, s = _rand((C, Tz), C + Tz), _rand((C, Ts), C + Ts + 1)
    buf, _ = _guarded(C * Ts)
    _op(6, buf[GUARD:], a=z, b=s, i0=C, i1=Ts, i2=Tz)
    got = _unguard(buf, C * Ts, "add_crop").view(C, Ts)
    assert torch.equal(got, z[:, :Ts] + s)


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("T", [1, 3833])
def test_sum_blocks_bitexact(n, T):
    """wav0 = sum of n per-model blocks in model order; nothing but block 0's first T floats changes."""
    stride = T + 37
    blocks = _rand((n * stride,), n + T, 1.0)
    buf, _ = _guarded(n * stride, blocks)
    _op(9, buf[GUARD:], i0=n, i1=T, i2=stride)
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + n * stride:]).all()
    got = buf[GUARD:GUARD + n * stride]
    want = blocks[:T].clone()
    for m in range(1, n):
        want = want + blocks[m * stride:m * stride + T]
    assert torch.equal(got[:T], want)
    assert torch.equal(got[T:], blocks[T:])


@pytest.mark.parametrize("T", [1, 3833, 144001])
def test_scale_copy_bitexact(T):
    src = _rand((T,), T)
    for s in (1.0, 0.7, -3.25):
        buf, _ = _guarded(T)
        _op(10, buf[GUARD:], a=src, i1=T, f=(s, 0, 0, 0, 0))
        assert torch.equal(_unguard(buf, T, "scale_copy"), src * s)


# ---- schedule step --------------------------------------------------------------------------------------------------
def _sched_case(label, cur, est, noise, a, b, sigma, ns, clip):
    T = cur.numel()
    buf, _ = _guarded(T, cur)
    _op(7, buf[GUARD:], a=est, b=noise, i1=T, f=(a, b, sigma, ns, clip))
    got = _unguard(buf, T, label)
    f32 = lambda v: float(np.float32(v))   # noqa: E731
    a, b, sigma, ns, clip = map(f32, (a, b, sigma, ns, clip))
    c, e = cur.double(), est.double()
    first = c - a * e * ns
    ref = first * b
    mag = abs(b) * (c.abs() + abs(a) * e.abs() * ns)
    if sigma > 0:
        nd = noise.double() * sigma * ns
        ref, mag = ref + nd, mag + nd.abs()
    if clip > 0:
        ref = ref.clamp(-clip, clip)
    return _check(label, got, ref, 5 * U * mag * (1 + 1e-6) + 1e-30)


def test_sched_step_schedule_rows():
    """Every row of the default 20-call schedule (mbd._schedule_table), noise scale 1, clip 5."""
    from mvb200.mbd import MBDSettings, _schedule_table
    s = MBDSettings()
    rows = _schedule_table(s.schedule, s.steps())
    assert rows.shape[0] == 20
    T = 3833
    for i, (a, b, sigma, _) in enumerate(rows.tolist()):
        cur, est, noise = _rand((T,), 3 * i, 2.5), _rand((T,), 3 * i + 1), _rand((T,), 3 * i + 2)
        _sched_case(f"sched row {i} (a={a:.3g} b={b:.3g} sigma={sigma:.3g})", cur, est, noise if sigma > 0 else None,
                    a, b, sigma, 1.0, 5.0)


def test_sched_step_edges():
    T = 1001
    cur, est, noise = _rand((T,), 1, 3.0), _rand((T,), 2), _rand((T,), 3)
    # sigma = 0 with a NULL noise pointer (must not be read), clip off, noise scale != 1
    _sched_case("sched sigma=0 noise=NULL", cur, est, None, 0.3, 1.2, 0.0, 0.8, 5.0)
    _sched_case("sched clip=0", cur * 10, est, noise, 0.3, 1.2, 0.4, 1.0, 0.0)
    # values exactly at and beyond +-clip (a = 0, b = 1, no noise: v = cur exactly)
    edge = torch.tensor([5.0, -5.0, 5.000001, -5.000001, 4.999999, 7.0, -1e30, 1e30, 0.0, -0.0], device="cuda")
    buf, _ = _guarded(edge.numel(), edge)
    _op(7, buf[GUARD:], a=torch.zeros_like(edge), i1=edge.numel(), f=(0.0, 1.0, 0.0, 1.0, 5.0))
    got = _unguard(buf, edge.numel(), "sched clamp")
    assert torch.equal(got, edge.clamp(-5.0, 5.0))
    _sched_case("sched at the clamp", torch.linspace(-6, 6, T, device="cuda"), est * 1e-3, noise, 0.01, 1.0, 0.05, 1.0, 5.0)


# ---- randn ----------------------------------------------------------------------------------------------------------
def philox4(v, c1, c2, c3, seed):
    """The four output words of Philox4x32-10 for counters (v, c1, c2, c3) (broadcast) and key (seed lo, seed hi)."""
    M = np.uint64(0xFFFFFFFF)
    c0, c1, c2, c3 = (np.asarray(c, np.uint64) & M for c in np.broadcast_arrays(*(np.asarray(c, np.int64) for c in (v, c1, c2, c3))))
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M, (k1 + np.uint64(0xBB67AE85)) & M
    return c0, c1, c2, c3


def test_philox_known_answer():
    """Random123's Philox4x32-10 known-answer vector: counter 0, key 0."""
    words = [int(w) for w in philox4(0, 0, 0, 0, 0)]
    assert words == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8], [hex(w) for w in words]


def _randn_reference(T, seed, stream, swap=False):
    """(ref, rad) float64 [T]: pairs i -> (rad cos(2 pi u2), rad sin(2 pi u2)), the last pair cut to T."""
    i = np.arange((T + 1) // 2)
    w0, w1, _, _ = philox4(i, stream, 0x6D6264, 0, seed)
    u1 = ((w0 >> np.uint64(8)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -24)
    u2 = ((w1 >> np.uint64(8)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -24)
    rad = np.sqrt(-2.0 * np.log(u1.astype(np.float64)))
    ang = 2.0 * np.pi * u2.astype(np.float64)
    cs, sn = rad * np.cos(ang), rad * np.sin(ang)
    if swap:
        cs, sn = sn, cs
    ref = np.stack([cs, sn], 1).reshape(-1)[:T]
    return torch.from_numpy(ref), torch.from_numpy(np.repeat(rad, 2)[:T])


def _randn_hook(T, seed, stream):
    buf, _ = _guarded(T)
    _op(8, buf[GUARD:], i1=T, i2=stream, seed=seed)
    return _unguard(buf, T, "randn").cpu()


@pytest.mark.parametrize("T,seed,stream", [(3833, 0, 0), (3832, 5, 1), (1, 12345, 7), (144001, 2 ** 32 + 7, 7 * 1024 + 1000),
                                           (4097, 2 ** 64 - 1, 7 * 1024), (20001, 0xDEADBEEF12345678, 3 * 1024 + 19)])
def test_randn_values(T, seed, stream):
    """Odd T (the last pair writes only the cosine half), a seed >= 2^32 (the key's high word), stream ids m 1024 + i at
    the extremes (m = 7, i = 1000)."""
    got = _randn_hook(T, seed, stream)
    ref, rad = _randn_reference(T, seed, stream)
    _check(f"randn T={T} seed={seed:#x} stream={stream}", got, ref, 5 * U * ref.abs() + 1e-15 * rad)


def test_randn_swapped_halves_fail_the_bound():
    """Sensitivity: a reference with the sine and cosine halves exchanged must put elements over the bound."""
    T = 4097
    got = _randn_hook(T, 99, 5).double()
    ref, rad = _randn_reference(T, 99, 5, swap=True)
    n_over = int(((got - ref).abs() > 5 * U * ref.abs() + 1e-15 * rad).sum())
    print(f"randn swapped halves: {n_over} of {T} elements over the bound")
    assert n_over > T // 2


def test_randn_distribution():
    """>= 1e6 draws: KS against N(0, 1), mean and variance within 5 sigma, lag-1 and adjacent-stream correlation below
    5 / sqrt(n)."""
    from scipy import stats
    n = (1 << 20) + 1
    x = _randn_hook(n, 2024, 3 * 1024 + 4).double().numpy()
    y = _randn_hook(n, 2024, 3 * 1024 + 5).double().numpy()
    ks = stats.kstest(x, "norm")
    lim = 5 / math.sqrt(n)
    lag1 = float(np.corrcoef(x[:-1], x[1:])[0, 1])
    adj = float(np.corrcoef(x, y)[0, 1])
    print(f"randn n={n}: KS p={ks.pvalue:.3g}, mean {x.mean():.2e}, var-1 {x.var() - 1:.2e}, lag-1 {lag1:.2e}, "
          f"adjacent streams {adj:.2e} (limit {lim:.2e})")
    assert ks.pvalue > 1e-3
    assert abs(x.mean()) < lim and abs(x.var() - 1) < 5 * math.sqrt(2 / n)
    assert abs(lag1) < lim and abs(adj) < lim


# ---- engine-level identities ----------------------------------------------------------------------------------------
def _engine(settings, oracle_cfg, seed=0, band_streams=True):
    from mvb200 import synth
    from mvb200.mbd import MultiBandDiffusionEngine
    return MultiBandDiffusionEngine(synth.mbd_checkpoint(oracle_cfg, seed), settings, device="cuda:0", max_seconds=1.0,
                                    band_streams=band_streams)


def _small(n_models=4, proc_bands=4, eq_bands=8):
    from mvb200.mbd import MBDSettings, UnetSettings
    from oracle import mbd_port as M
    u = dict(hidden=16, depth=2, growth=2.0, kernel=8, stride=4, res_blocks=1, norm_groups=4)
    steps = [999, 749, 499, 249, 0]
    return (MBDSettings(n_models=n_models, unet=UnetSettings(**u), proc_bands=proc_bands, eq_bands=eq_bands, step_list=steps),
            M.MBDConfig(n_models=n_models, unet=M.UnetCfg(**u), proc_bands=proc_bands, eq_bands=eq_bands, step_list=steps))


def _inputs(frames, T, seed):
    from mvb200 import synth
    g = torch.Generator().manual_seed(seed)
    cond = torch.randn(128, frames, generator=g)
    wav_e = torch.from_numpy(synth.synthetic_waveform(frames * 320 / 24000.0, 24000, seed=seed))[:T].float()
    return cond, wav_e, g


def test_seeded_noise_equals_supplied_noise():
    """tokens_to_wav(seed=s) draws row 0 of band model m from Philox stream m 1024 and row i + 1 from m 1024 + i + 1:
    supplying those rows (from the randn hook) as `noise` gives the same waveform bit for bit."""
    settings, ocfg = _small()
    eng = _engine(settings, ocfg, 3)
    frames, T, seed = 12, 12 * 320 - 7, 2 ** 32 + 99
    cond, wav_e, _ = _inputs(frames, T, 1)
    noise = torch.stack([torch.stack([_randn_hook(T, seed, m * 1024 + r) for r in range(eng.n_calls)])
                         for m in range(settings.n_models)])
    a = eng.tokens_to_wav(cond, wav_e, seed=seed).cpu()
    b = eng.tokens_to_wav(cond, wav_e, noise=noise).cpu()
    assert torch.isfinite(a).all() and torch.equal(a, b)
    c = eng.tokens_to_wav(cond, wav_e, seed=seed + 1).cpu()
    assert not torch.equal(a, c)


@pytest.mark.parametrize("config", ["small", "default"])
def test_one_stream_equals_four_streams(config):
    """band_streams=False (MVB_MBD_ONE_STREAM, fixed at create time) runs the band models one after another on the
    caller's stream and accumulates their outputs in place with k_band_mix; the default runs them on four streams and adds
    the blocks with k_sum_blocks afterwards.  Both add in model order, so the waveforms are bitwise equal."""
    from mvb200.mbd import MBDSettings
    from oracle import mbd_port as M
    if config == "small":
        settings, ocfg = _small()
    else:
        steps = [999, 499, 0]
        settings, ocfg = MBDSettings(n_models=4, step_list=steps), M.MBDConfig(n_models=4, step_list=steps)
    frames, T = 12, 12 * 320 - 7
    cond, wav_e, g = _inputs(frames, T, 2)
    one = _engine(settings, ocfg, 4, band_streams=False)
    four = _engine(settings, ocfg, 4)
    noise = torch.randn(4, one.n_calls, T, generator=g)
    a = one.tokens_to_wav(cond, wav_e, noise=noise).cpu()
    b = four.tokens_to_wav(cond, wav_e, noise=noise).cpu()
    one.close()
    four.close()
    assert torch.isfinite(a).all() and torch.equal(a, b)


def test_sixty_four_bands_end_to_end():
    """64 processor and re-EQ bands (5921 taps, more than 64 KB of FIR shared memory) run and match the restatement."""
    from oracle import mbd_port as M
    settings, ocfg = _small(n_models=2, proc_bands=64, eq_bands=64)
    from mvb200 import synth
    ck = synth.mbd_checkpoint(ocfg, 5)
    from mvb200.mbd import MultiBandDiffusionEngine
    eng = MultiBandDiffusionEngine(ck, settings, device="cuda:0", max_seconds=1.0, tensor_cores=False)
    assert eng.cfg.proc_taps == eng.cfg.eq_taps == 5921
    frames, T = 12, 12 * 320
    cond, wav_e, g = _inputs(frames, T, 6)
    noise = torch.randn(2, eng.n_calls, T, generator=g)
    got = eng.tokens_to_wav(cond, wav_e, noise=noise).cpu()
    want = M.MBDOracle(ck, ocfg).tokens_to_wav(wav_e, cond, noise)
    err = float((got - want).abs().max() / want.abs().max())
    print(f"MBD 64 bands ({T} samples): rel err vs restatement {err:.2e}")
    eng.close()
    assert err < 2e-3
