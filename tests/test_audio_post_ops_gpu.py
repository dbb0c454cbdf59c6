"""GPU: the audio post-processing kernels of csrc/audio_post.cu one at a time (hook `mvb_audio_post_test`) against float64
references of the same operations, and the edge-case contract of `mvb_audio_post` / `audio_out.wav_bytes_on_device`.
u = 2^-23 throughout.

k_kweight.  Reference: y = clip(hp(clip(shelf(x)))) in float64 (scipy lfilter), on the kernel's fp32-rounded
coefficients (recomputed here exactly as `treble_shelf` / `highpass` do, then rounded to fp32); the clamps act on each
biquad's output, not on its state (torchaudio's lfilter).  Bound, per section with all-pole impulse response h:
  rounding    each step evaluates 5 products and 4 adds in fp32: delta_t <= 5u (|b0 x_t| + |b1 x_t-1| + |b2 x_t-2| +
              |a1 y_t-1| + |a2 y_t-2|) (+ its own rounding), and the error of y obeys the all-pole recursion driven by
              delta, so |e| <= ||h||_1 max delta.  ||h||_1 is computed numerically in float64 (about 1.0e4 for the 38 Hz
              double pole at 24 kHz, 4.1e4 at 48 kHz);
  warm-up     every 2048-sample chunk starts from a zero state 4096 samples earlier; the dropped state decays like the
              impulse response, so the term is 4 sup_{m >= 4094} |h_m| (sum |b| max|in| + sum |a| max|out|).  For the
              high-pass at 24 kHz sup |h_m| = 1.0e-14 (the double pole gives m r^m, not the e^-40 of r^m alone);
              1e-6 at 44.1 kHz, 6e-6 at 48 kHz;
  the shelf's error E_u reaches the high-pass through the 1-Lipschitz clamp and its full response (||h_hp,full||_1 ~ 2.25).
Sensitivity: a reference restarted from zero at every chunk (no warm-up) and one without the clamps must violate.

k_block_energy.  Compared with float64 block means of the kernel's own y^2 (and sum x^2 for the whole-signal slot).  Every
term is >= 0, so the fp32 sum (sequential fmaf per thread over ceil(n / 256) terms, a 5-level warp tree, 8 warp partials,
one division) is within (ceil(n / 256) + 14) u of the exact value, relatively.

k_loudness_gain.  float64 BS.1770 gating over the kernel's own energies.  A block's fp32 level l = -0.691 + 10 log10f(e)
is within 4u (10 |log10 e| + |l|) of the exact one (log10f: 2 ulp); the relative threshold carries in addition the fp32
mean over cnt blocks, 4.343 (cnt + 2) u dB.  A gate decision may differ from float64 only when the float64 level lies
inside that band around its threshold (audited: every such block is tried both ways).  LKFS: 4.343 (cnt + 2) u +
4u (10 |log10 m| + |LKFS|); gain = powf(10, (-headroom - LKFS) / 20): ln(10) / 20 (dLKFS + 2u (headroom + |LKFS|)) + 6u
relative.  Sensitivity: the reference without the relative gate must violate.

k_apply_pcm16.  Without the compressor the kernel's arithmetic is two fp32 products and a round-half-even, emulated here
exactly (numpy float32): PCM must be bit-identical, exact .5 ties included.  With it, float64
clip(tanh(g x)) 32767 is within m = 32767 (u |g x| + 2u |t|) + u 32767 |t| of the kernel's pre-rounding value
(tanhf: 2 ulp); PCM must equal round-half-even of the float64 value wherever that is more than m from a .5 boundary, and
one of its two neighbours inside it.

Every output buffer is surrounded by NaN guards: the kernels must write all of it and nothing else."""
import ctypes as C
import math
import time

import numpy as np
import pytest
import scipy.signal as ss
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
GUARD = 256
W_WARM, CHUNK = 4096, 2048
HEADROOM = 14.0


def _f32(v):
    return float(np.float32(v))


def _coeffs(sr):
    """(shelf, highpass) as float64 arrays [b0, b1, b2, a1, a2] of the kernel's fp32 coefficients."""
    w0 = 2 * math.pi * 1500.0 / sr
    alpha, A = math.sin(w0) / 2 / (1.0 / math.sqrt(2.0)), math.exp(4.0 / 40 * math.log(10.0))
    t1, t2, t3 = 2 * math.sqrt(A) * alpha, (A - 1) * math.cos(w0), (A + 1) * math.cos(w0)
    b = [A * ((A + 1) + t2 + t1), -2 * A * ((A - 1) + t3), A * ((A + 1) + t2 - t1)]
    a = [(A + 1) - t2 + t1, 2 * ((A - 1) - t3), (A + 1) - t2 - t1]
    shelf = np.array([_f32(v / a[0]) for v in b + a[1:]])
    w0 = 2 * math.pi * 38.0 / sr
    alpha = math.sin(w0) / 2 / 0.5
    b = [(1 + math.cos(w0)) / 2, -1 - math.cos(w0), (1 + math.cos(w0)) / 2]
    a = [1 + alpha, -2 * math.cos(w0), 1 - alpha]
    hp = np.array([_f32(v / a[0]) for v in b + a[1:]])
    return shelf, hp


def _responses(c, n=1 << 18):
    imp = np.zeros(n)
    imp[0] = 1.0
    return ss.lfilter([1.0], [1.0, c[3], c[4]], imp), ss.lfilter(c[:3], [1.0, c[3], c[4]], imp)


def _biquad(c, x, restart=False):
    if not restart:
        return ss.lfilter(c[:3], [1.0, c[3], c[4]], x)
    return np.concatenate([ss.lfilter(c[:3], [1.0, c[3], c[4]], x[i:i + CHUNK]) for i in range(0, len(x), CHUNK)])


def kweight_ref(x, sr, clamp=True, restart=False):
    """(y, u, v): float64 K-weighting of the fp32 input x with the kernel's coefficients."""
    s, h = _coeffs(sr)
    u = _biquad(s, np.asarray(x, np.float64), restart)
    c = np.clip(u, -1, 1) if clamp else u
    v = _biquad(h, c, restart)
    return (np.clip(v, -1, 1) if clamp else v), u, v


def kweight_bound(x, u, v, sr):
    s, h = _coeffs(sr)
    hs, _ = _responses(s)
    hh, hh_full = _responses(h)
    x = np.abs(np.asarray(x, np.float64))
    c = np.minimum(np.abs(u), 1.0)

    def lagged(a, k):
        return np.concatenate([np.zeros(k), a[:len(a) - k]]) if k else a

    def step_delta(coef, inp, out):
        t = sum(abs(coef[k]) * lagged(inp, k) for k in range(3)) + abs(coef[3]) * lagged(out, 1) + abs(coef[4]) * lagged(out, 2)
        return 6 * U * (t + np.abs(out))

    def warm(coef, hresp, inp, out):
        return 4 * np.abs(hresp[W_WARM - 2:]).max() * (np.abs(coef[:3]).sum() * inp.max() + np.abs(coef[3:]).sum() * np.abs(out).max())

    e_u = np.abs(hs).sum() * step_delta(s, x, np.abs(u)).max() + warm(s, hs, x, u)
    e_v = np.abs(hh_full).sum() * e_u + np.abs(hh).sum() * step_delta(h, c, np.abs(v)).max() + warm(h, hh, c, v)
    # the deltas are taken on the float64 magnitudes; the kernel's own differ from them by at most the bound (10 %)
    return e_v * 1.1 + 1e-30, dict(h1_shelf=np.abs(hs).sum(), h1_hp=np.abs(hh).sum(), tail_hp=np.abs(hh[W_WARM - 2:]).max())


def _run(x, sr, comp=1, headroom=HEADROOM, expect=0):
    from mvb200 import _lib as L
    lib = L.load()
    x = torch.as_tensor(np.asarray(x, np.float32)).cuda().contiguous()
    n = x.numel()
    gate = round(0.4 * sr)
    nb_max = (n - gate) // round(gate * 0.25) + 1 if n >= gate else 0

    def guarded(k, dtype=torch.float32):
        fill = float("nan") if dtype == torch.float32 else -12345
        buf = torch.full((2 * GUARD + k,), fill, dtype=dtype, device="cuda")
        return buf, buf[GUARD:GUARD + k]

    pb, pcm = guarded(n, torch.int16)
    wb, wav = guarded(n)
    yb, y = guarded(n)
    eb, en = guarded(nb_max + 1)
    rb, res = guarded(3)
    nb = C.c_int32(-1)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = lib.mvb_audio_post_test(x.data_ptr(), n, sr, C.c_float(headroom), comp, pcm.data_ptr(), wav.data_ptr(), y.data_ptr(),
                                 en.data_ptr(), res.data_ptr(), C.byref(nb), st)
    if expect:
        assert rc == expect, (rc, lib.mvb_last_error())
        assert bool((pb == -12345).all()) and bool(torch.isnan(yb).all()) and bool(torch.isnan(rb).all()), "launched anyway"
        return None
    L.check(rc)
    assert nb.value == nb_max
    for b, v in ((wb, wav), (yb, y), (eb, en), (rb, res)):
        assert torch.isnan(b[:GUARD]).all() and torch.isnan(b[-GUARD:]).all(), "write outside the output"
    assert bool((pb[:GUARD] == -12345).all()) and bool((pb[-GUARD:] == -12345).all()), "PCM written outside [0, n)"
    # (the whole-signal slot en[-1] is NaN for a NaN input; the clamps keep y, and so the block energies, finite)
    assert not torch.isnan(y).any() and not torch.isnan(en[:-1]).any() and not torch.isnan(res[1:]).any(), "not written"
    return dict(x=x.cpu().numpy(), y=y.cpu().numpy().astype(np.float64), energy=en.cpu().numpy().astype(np.float64),
                res=res.cpu().numpy().astype(np.float64), pcm=pcm.cpu().numpy(), wav=wav.cpu().numpy(), n_blocks=nb.value,
                gate=gate, step=round(gate * 0.25))


def _signal(sr, secs, seed, amp=0.3, low=True):
    """Tones, a low-frequency component (exercises the 38 Hz high-pass state across chunk seams) and noise."""
    rng = np.random.default_rng(seed)
    t = np.arange(int(round(secs * sr))) / sr
    x = amp * (0.5 * np.sin(2 * np.pi * 440 * t) + 0.3 * np.sin(2 * np.pi * 3100 * t + 1) + 0.2 * rng.standard_normal(t.size))
    if low:
        x = x + amp * 0.8 * np.sin(2 * np.pi * 31 * t + 0.3)
    return x.astype(np.float32)


# ---- k_kweight ---------------------------------------------------------------------------------------------------------
def _check_kweight(label, x, sr, **run):
    r = _run(x, sr, **run)
    ref, u, v = kweight_ref(r["x"], sr)
    bound, info = kweight_bound(r["x"], u, v, sr)
    err = np.abs(r["y"] - ref)
    n = len(ref)
    seams = [t for k in range(1, (n - 1) // CHUNK + 1) for t in (k * CHUNK - 1, k * CHUNK, k * CHUNK + 1) if t < n]
    nw = float(np.linalg.norm(err) / max(np.linalg.norm(ref), 1e-30))
    print(f"k_kweight {label} sr={sr} T={n}: max |err|/bound {err.max() / bound:.2e} (bound {bound:.2e}, ||h_hp||_1 "
          f"{info['h1_hp']:.3g}, hp tail {info['tail_hp']:.2e}), seams {err[seams].max() / bound if seams else 0:.2e}, "
          f"normwise {nw:.2e}")
    assert (err <= bound).all(), f"{label}: {(err > bound).sum()} samples over the bound, first at {np.argmax(err > bound)}"
    return r, bound


@pytest.mark.parametrize("T", [1, 2047, 2048, 2049, 4097, 6145])
def test_kweight_chunk_seams(T):
    _check_kweight("seams", _signal(24000, T / 24000, seed=T), 24000)


@pytest.mark.parametrize("sr", [8000, 16000, 24000, 44100, 48000])
def test_kweight_sample_rates(sr):
    _check_kweight("rate", _signal(sr, 1.3, seed=sr), sr)


def test_kweight_60s_and_restart_sensitivity():
    """60 s at 24 kHz (704 chunks, the last one partial).  A reference restarted from zero at every chunk must violate
    the bound."""
    r, bound = _check_kweight("60 s", _signal(24000, 60.0, seed=60), 24000)
    bad, _, _ = kweight_ref(r["x"], 24000, restart=True)
    over = int((np.abs(r["y"] - bad) > bound).sum())
    print(f"restarted-chunk reference: {over} samples over the bound, worst {np.abs(r['y'] - bad).max() / bound:.1e} x bound")
    assert over > 0


def test_kweight_active_clamps_and_sensitivity():
    """Shelf output driven past +-1 (the +4 dB treble shelf on a 0.95 full-scale 5 kHz tone); a reference without the
    clamps must violate."""
    sr = 24000
    t = np.arange(3 * CHUNK + 5) / sr
    x = (0.95 * np.sin(2 * np.pi * 5000 * t) * np.minimum(1, t * 8)).astype(np.float32)
    r, bound = _check_kweight("clamped", x, sr)
    _, u, _ = kweight_ref(r["x"], sr)
    assert np.abs(u).max() > 1.2, "the clamps are not active"
    bad, _, _ = kweight_ref(r["x"], sr, clamp=False)
    over = int((np.abs(r["y"] - bad) > bound).sum())
    print(f"no-clamp reference: {over} samples over the bound")
    assert over > 0


# ---- k_block_energy + k_loudness_gain ----------------------------------------------------------------------------------
def _check_energies(r):
    y2 = r["y"] ** 2
    gate, step, nb = r["gate"], r["step"], r["n_blocks"]
    if nb:
        blocks = np.lib.stride_tricks.sliding_window_view(y2, gate)[::step][:nb].sum(1) / gate
    else:
        blocks = np.zeros(0)
    whole = float((r["x"].astype(np.float64) ** 2).sum())
    gb = (math.ceil(gate / 256) + 14) * U
    gw = (math.ceil(len(r["x"]) / 256) + 14) * U
    eb = np.abs(r["energy"][:nb] - blocks)
    assert (eb <= gb * blocks + 1e-38).all(), f"block energy over the bound at {np.argmax(eb > gb * blocks)}"
    assert abs(r["energy"][nb] - whole) <= gw * whole + 1e-38, (r["energy"][nb], whole)
    worst = max(float((eb / (gb * blocks + 1e-38)).max()) if nb else 0.0, abs(r["energy"][nb] - whole) / (gw * whole + 1e-38))
    return worst


def loudness_ref(energy, rel_gate=True, flip=frozenset()):
    """float64 BS.1770 gating of the given block energies -> (lkfs, kept mask, near-tie blocks).  A near-tie block is
    one whose float64 level lies within the fp32 band of a threshold; `flip` reverses the decision of such blocks (the
    near-tie audit)."""
    e = np.asarray(energy, np.float64)
    idx = np.arange(e.size)
    with np.errstate(divide="ignore"):
        lg = np.log10(e)
    l = -0.691 + 10 * lg
    band = 4 * U * (10 * np.abs(lg) + np.abs(l))
    near_abs = set(np.nonzero(np.abs(l + 70.0) <= band)[0].tolist())
    keep_abs = (l > -70.0) ^ np.isin(idx, sorted(flip & near_abs))
    if not keep_abs.any():
        return float("nan"), keep_abs, near_abs
    m = e[keep_abs].mean()
    g_rel = -0.691 + 10 * math.log10(m) - 10.0
    rel_band = 4.343 * (keep_abs.sum() + 2) * U + 4 * U * (10 * abs(math.log10(m)) + abs(g_rel))
    near_rel = set(np.nonzero(keep_abs & (np.abs(l - g_rel) <= band + rel_band))[0].tolist()) if rel_gate else set()
    keep = keep_abs & ((l > g_rel) ^ np.isin(idx, sorted(flip & near_rel))) if rel_gate else keep_abs
    return -0.691 + 10 * math.log10(e[keep].mean()), keep, near_abs | near_rel


def _check_gain(r, headroom=HEADROOM):
    nb = r["n_blocks"]
    e = r["energy"][:nb]
    lk, keep, near = loudness_ref(e)
    assert len(near) <= 10, f"{len(near)} near-tie gate decisions"
    cands = [lk]
    for mask in range(1, 1 << len(near)):       # every near-tie block either way
        cands.append(loudness_ref(e, flip=frozenset(b for i, b in enumerate(sorted(near)) if mask >> i & 1))[0])
    got_lk, got_g, comp = r["res"]
    cnt = int(keep.sum())
    m = 10 ** ((lk + 0.691) / 10)
    b_lk = 4.343 * (cnt + 2) * U + 4 * U * (10 * abs(math.log10(m)) + abs(lk))
    d = min(abs(got_lk - c) for c in cands)
    assert d <= b_lk, (got_lk, lk, b_lk)
    g = 10 ** ((-headroom - lk) / 20)
    b_g = g * (math.log(10) / 20 * (b_lk + 2 * U * (headroom + abs(lk))) + 6 * U)
    assert abs(got_g - g) <= b_g, (got_g, g, b_g)
    assert comp == 1.0
    return d / b_lk, abs(got_g - g) / b_g, len(near), lk, b_lk


@pytest.mark.parametrize("extra", [-1, 0, "step-1", "step"])
def test_block_energy_at_block_boundaries(extra):
    sr = 16000
    gate, step = 6400, 1600
    n = gate + {-1: -1, 0: 0, "step-1": step - 1, "step": step}[extra]
    x = _signal(sr, n / sr, seed=7)
    r = _run(x, sr)
    assert r["n_blocks"] == {-1: 0, 0: 1, "step-1": 1, "step": 2}[extra]
    worst = _check_energies(r)
    print(f"k_block_energy n={n}: {r['n_blocks']} blocks, max |err|/bound {worst:.2e}")
    if r["n_blocks"]:
        _check_gain(r)
    else:
        assert math.isnan(r["res"][0]) and r["res"][1] == 1.0 and r["res"][2] == 0.0


def test_block_limit_and_loudness_over_16000_blocks():
    """n_blocks = 15996 (the most the workspace holds) at 8 kHz, 26.7 min: energies and the gating over all of them; one
    sample more returns MVB_ERR_UNSUPPORTED and launches nothing."""
    from mvb200 import _lib as L
    sr, gate, step = 8000, 3200, 800
    n = gate + 15995 * step + step - 1
    rng = np.random.default_rng(11)
    t = np.arange(n) / sr
    env = 10 ** (np.interp(t, [0, t[-1] / 3, 2 * t[-1] / 3, t[-1]], [-4.5, -0.5, -3.2, -1.5]))   # -90 ... -10 dBFS
    x = (env * (np.sin(2 * np.pi * 440 * t) + 0.1 * rng.standard_normal(n))).astype(np.float32)
    t0 = time.time()
    r = _run(x, sr)
    assert r["n_blocks"] == 15996
    worst = _check_energies(r)
    q_lk, q_g, n_near, lk, b_lk = _check_gain(r)
    print(f"16000-block run ({time.time() - t0:.1f} s): energies {worst:.2e}, LKFS {lk:.3f} (|err|/bound {q_lk:.2e}, bound "
          f"{b_lk:.1e} dB), gain {q_g:.2e}, {n_near} near-tie decisions")
    bad = loudness_ref(r["energy"][:15996], rel_gate=False)[0]
    print(f"reference without the relative gate: {abs(bad - r['res'][0]) / b_lk:.1e} x bound")
    assert abs(bad - r["res"][0]) > b_lk
    _run(np.zeros(n + 1, np.float32), sr, expect=L.MVB_ERR_UNSUPPORTED)


def test_gating_near_both_thresholds():
    """An exponential level ramp (-95 ... -25 LKFS) after a loud section: blocks land densely around -70 LKFS and
    around the relative gate."""
    sr = 16000
    rng = np.random.default_rng(5)
    t = np.arange(25 * sr) / sr
    env = np.where(t < 5, 0.3, 10 ** np.interp(t, [5, 25], [-4.7, -1.0]))
    x = (env * (np.sin(2 * np.pi * 1000 * t) + 0.05 * rng.standard_normal(t.size))).astype(np.float32)
    r = _run(x, sr)
    _check_energies(r)
    e = r["energy"][:r["n_blocks"]]
    l = -0.691 + 10 * np.log10(e)
    g_rel = -0.691 + 10 * math.log10(e[l > -70].mean()) - 10
    print(f"closest block to -70 LKFS: {np.abs(l + 70).min():.2e} dB; to the relative gate {g_rel:.2f}: "
          f"{np.abs(l - g_rel).min():.2e} dB")
    assert np.abs(l + 70).min() < 0.2 and np.abs(l - g_rel).min() < 0.2
    q_lk, q_g, n_near, lk, b_lk = _check_gain(r)
    print(f"k_loudness_gain near thresholds: LKFS |err|/bound {q_lk:.2e}, gain {q_g:.2e}, {n_near} near-tie decisions")
    assert abs(loudness_ref(e, rel_gate=False)[0] - r["res"][0]) > b_lk


# ---- k_apply_pcm16 -----------------------------------------------------------------------------------------------------
def test_pcm16_no_compressor_bit_exact_with_ties():
    """Without the compressor PCM is two fp32 products and round-half-even: exact, including exact .5 ties."""
    sr = 24000
    x = _signal(sr, 2.0, seed=3, amp=0.9)
    r = _run(x, sr, comp=0)
    g = np.float32(r["res"][1])
    v = np.clip(g * r["x"], np.float32(-1), np.float32(1))
    want = np.rint(v * np.float32(32767)).astype(np.int16)
    assert np.array_equal(r["pcm"], want) and np.array_equal(r["wav"], v)
    # below the floor (gain 1): samples whose fp32 product with 32767 is exactly k + 0.5
    ks = np.arange(-60, 60)
    cand = ((ks + 0.5) / 32767).astype(np.float32)
    ties = cand[(cand * np.float32(32767)) == (ks + 0.5).astype(np.float32)]
    assert ties.size >= 20
    q = np.zeros(24000, np.float32)
    q[::97][:ties.size] = ties
    r = _run(q, sr, comp=1)
    assert r["res"][0] == -np.inf and r["res"][1] == 1.0 and r["res"][2] == 0.0
    want = np.rint(q * np.float32(32767)).astype(np.int16)
    assert np.array_equal(r["pcm"], want)
    print(f"k_apply_pcm16 no compressor: bit-exact, {ties.size} exact ties")


def test_pcm16_compressor_within_tanhf_margin():
    sr = 24000
    x = _signal(sr, 3.0, seed=4, amp=0.9)
    r = _run(x, sr, comp=1)
    g = float(np.float32(r["res"][1]))
    gx = g * r["x"].astype(np.float64)
    th = np.tanh(gx)
    val = np.clip(th, -1, 1) * 32767
    margin = 32767 * (U * np.abs(gx) + 2 * U * np.abs(th)) + U * 32767 * np.abs(th) + 1e-9
    frac = np.abs(val - np.floor(val) - 0.5)
    exact = frac > margin
    want = np.rint(val)
    got = r["pcm"].astype(np.float64)
    assert np.array_equal(got[exact], want[exact]), f"{int((got[exact] != want[exact]).sum())} PCM samples differ"
    assert (np.abs(got[~exact] - val[~exact]) <= 0.5 + margin[~exact]).all()
    print(f"k_apply_pcm16 compressor: {int((~exact).sum())} of {exact.size} samples within the tanhf margin of a tie")


# ---- edge-case contract: device == host writer ---------------------------------------------------------------------------
def _host(x, sr, tmp_path):
    from mvb200 import audio_out as A
    try:
        p = A.audio_write_wav(str(tmp_path / "h"), torch.from_numpy(x)[None], sr)
        return open(p, "rb").read()
    except Exception as e:          # noqa: BLE001 -- the type is what is compared
        return type(e)


def _device(x, sr):
    from mvb200 import audio_out as A
    try:
        return A.wav_bytes_on_device(torch.from_numpy(x).cuda(), sr)
    except Exception as e:          # noqa: BLE001
        return type(e)


def _same(x, sr, tmp_path):
    h, d = _host(x, sr, tmp_path), _device(x, sr)
    if isinstance(h, type) or isinstance(d, type):
        assert h == d, (h, d)
        return h
    assert d[:44] == h[:44] and len(d) == len(h)
    a = np.frombuffer(d[44:], dtype="<i2").astype(np.int32)
    b = np.frombuffer(h[44:], dtype="<i2").astype(np.int32)
    assert np.abs(a - b).max() <= 2
    return "bytes"


def test_rumble_below_the_gate_is_not_full_scale(tmp_path):
    """2 s of a 5 Hz rumble at 0.01: RMS 7.1e-3 (above the floor) but every K-weighted block below -78 LKFS.  The meter
    is undefined (torchaudio: NaN; the host writer's finiteness assert fails); the device must report NaN, keep the
    gain at 1 with the compressor off, and write the clipped input -- not -32767 everywhere."""
    sr = 24000
    t = np.arange(2 * sr) / sr
    x = (0.01 * np.sin(2 * np.pi * 5 * t)).astype(np.float32)
    r = _run(x, sr)
    e = r["energy"][:r["n_blocks"]]
    assert (-0.691 + 10 * np.log10(e)).max() < -78
    assert math.isnan(r["res"][0]) and r["res"][1] == 1.0 and r["res"][2] == 0.0, r["res"]
    assert np.array_equal(r["pcm"], np.rint(x * np.float32(32767)).astype(np.int16))
    assert _same(x, sr, tmp_path) is AssertionError


def test_signal_shorter_than_one_block(tmp_path):
    sr = 24000
    x = (0.3 * np.sin(2 * np.pi * 440 * np.arange(int(0.3 * sr)) / sr)).astype(np.float32)
    r = _run(x, sr)
    assert r["n_blocks"] == 0 and math.isnan(r["res"][0]) and r["res"][1] == 1.0 and r["res"][2] == 0.0
    assert _same(x, sr, tmp_path) is RuntimeError
    assert _same(x * np.float32(1e-3), sr, tmp_path) == "bytes"        # below the floor: passes through on both


def test_non_finite_sample(tmp_path):
    sr = 24000
    x = _signal(sr, 2.0, seed=9)
    x[12345] = np.nan
    r = _run(x, sr)
    assert math.isnan(r["res"][0]) and r["res"][1] == 1.0 and r["res"][2] == 0.0
    finite = np.isfinite(x)
    assert r["pcm"][12345] == 0
    assert np.array_equal(r["pcm"][finite], np.rint(np.clip(x[finite], -1, 1) * np.float32(32767)).astype(np.int16))
    assert _same(x, sr, tmp_path) is AssertionError
    x[12345] = np.inf
    assert math.isnan(_run(x, sr)["res"][0])
    assert _same(x, sr, tmp_path) is AssertionError


def floor_signal(rms):
    """2^15 samples on the grid 2^-13 (a quantised 440 Hz tone, then +-1-step clicks in a silent tail) whose sum of
    squares N 2^-26 is exact in any summation order, with N chosen so that fp32 sqrt(mean) == rms exactly."""
    T, h = 1 << 15, 13
    target = np.float32(rms)
    n0 = int(round(float(target) ** 2 * 2.0 ** (2 * h) * T))
    N = next(k for d in range(4096) for k in (n0 + d, n0 - d)
             if np.sqrt(np.float32(k * 2.0 ** (-2 * h)) / np.float32(T)) == target)
    idx = np.arange(T - 4096)
    lo, hi = 0.0, 40.0
    for _ in range(60):
        a = (lo + hi) / 2
        if (np.rint(a * np.sin(2 * np.pi * 437.3 * idx / 24000)) ** 2).sum() <= N:
            lo = a
        else:
            hi = a
    j = np.zeros(T)
    j[:T - 4096] = np.rint(lo * np.sin(2 * np.pi * 437.3 * idx / 24000))
    d = N - int((j ** 2).sum())
    assert 0 <= d < 4096
    j[T - 4096:T - 4096 + d] = np.where(np.arange(d) % 2, -1.0, 1.0)
    x = (j * 2.0 ** -h).astype(np.float32)
    assert (j ** 2).sum() == N and np.float32(torch.from_numpy(x).pow(2).mean().sqrt().item()) == target
    return x


@pytest.mark.parametrize("side", [-1, 0, 1])
def test_energy_floor_one_ulp_either_side(side, tmp_path):
    """RMS exactly fp32(2e-3) and one ulp below / above: device and host take the same branch (pass through below,
    normalise at and above; no fp32 value lies between 2e-3 and fp32(2e-3))."""
    f = np.float32(2e-3)
    rms = {-1: np.nextafter(f, np.float32(0)), 0: f, 1: np.nextafter(f, np.float32(1))}[side]
    x = floor_signal(rms)
    r = _run(x, 24000)
    assert np.float32(math.sqrt(r["energy"][r["n_blocks"]] / x.size)) == rms
    assert (r["res"][0] == -np.inf) == (side < 0)
    assert _same(x, 24000, tmp_path) == "bytes"
