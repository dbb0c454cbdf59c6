"""GPU: the multi-band-diffusion convolutions one at a time (csrc/mbd.cu, csrc/mbd_tc.cuh), tensor-core shifted-GEMM kernel
and CUDA-core kernels, against float64 F.conv1d / F.conv_transpose1d of the same operation.

Reference.  The optional relu(GroupNorm) prologue is applied with the same caller-supplied fp32 (mean, rstd):
a = fl(fl(x - mean) * rstd) as the kernels compute it, then f = relu(a * gain + bias) in float64 (the kernels round that
last step once or twice in fp32: |df| <= 3 u (|a gain| + |bias|)).  The tensor-core path then sees x^ = hi + lo with
hi = bf16(f), lo = bf16(f - hi) (a perturbed f can also move lo by one bf16 ulp, 2^-16 |f|), and bf16-rounded taps; the
reference is the float64 convolution of x^ with the bf16 taps.  The CUDA-core path sees f and the fp32 taps.

Elementwise bound, with A = conv(|x^|, |W|) (K_eff = taps x Cp products per output, Cp = Cin rounded up to 64):
  tensor cores  gamma = 18 u * 2 K_eff / 16: each mma.sync.m16n8k16 (hi and lo products of 16 channels) changes the exact
                value by at most 18 u (|c| + sum |p|) (alignment of 17 addends with truncation, truncating normalisation,
                u = 2^-23; see tests/test_gemm_ops_gpu.py), and one output accumulates 2 K_eff / 16 of them sequentially;
  CUDA cores    gamma = (K_eff + 2) u: one fmaf per product (Cin x taps of them, two taps per input channel for the
                transposed convolution);
plus conv(|dx^|, |W|) for the prologue and 2 u (|y| + |bias| + |emb| + |out|) for the fp32 epilogue adds.
Normwise: ||out - ref||_F / ||conv||_F < 1e-4, far below the ~1.7e-3 of a dropped lo term or of fp32 taps against bf16 ones.

The output buffer is surrounded by NaN guards: the kernel must write every element of [Cout, Tout] and nothing else."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
NORMWISE = 1e-4
GUARD = 1024
# default MBDSettings (hidden 48, growth 4, depth 4) at 12 frames = 3833 samples: level lengths 959 / 240 / 60 / 15
WIDTHS, LENGTHS = [48, 192, 768, 3072], [959, 240, 60, 15]


def _cp(cin):
    return (cin + 63) // 64 * 64


def _gamma(kind, cin, K, use_tc):
    taps = 2 if kind == 2 else K
    if use_tc:
        return 18 * U * 2 * taps * _cp(cin) / 16
    return (taps * cin + 2) * U


def _make(kind, cin, cout, K, stride, tin, seed, gn, bias, emb, resid, groups=4, exact_taps=True):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"
    x = torch.randn(cin, tin, generator=g, device=dev) * 0.7 + 0.2
    wshape = (cin, cout, K) if kind == 2 else (cout, cin, K)
    w = torch.randn(*wshape, generator=g, device=dev) / (cin * K) ** 0.5
    if exact_taps:
        w = w.to(torch.bfloat16).float()
    tout = tin if kind == 0 else (-(-tin // stride) if kind == 1 else tin * stride)
    d = dict(x=x, w=w, tout=tout, gn=None, bias=None, emb=None, resid=None, groups=groups)
    if gn:
        xg = x.double().view(groups, -1)
        mean, var = xg.mean(1), xg.var(1, unbiased=False)
        stats = torch.stack([mean, 1.0 / torch.sqrt(var + 1e-5)], 1).float().contiguous()
        gw = 1 + 0.2 * torch.randn(cin, generator=g, device=dev)
        gb = 0.1 * torch.randn(cin, generator=g, device=dev)
        d["gn"] = (stats, gw, gb)
    if bias:
        d["bias"] = 0.1 * torch.randn(cout, generator=g, device=dev)
    if emb:
        d["emb"] = 0.1 * torch.randn(cout, generator=g, device=dev)
    if resid:
        d["resid"] = torch.randn(cout, tout, generator=g, device=dev)
    return d


def _run(kind, d, cin, cout, K, stride, dil, pad, use_tc):
    from mvb200 import _lib as L
    lib = L.load()
    tout = d["tout"]
    buf = torch.full((2 * GUARD + cout * tout,), float("nan"), device="cuda")
    y = buf[GUARD:GUARD + cout * tout]
    ptr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    stats, gw, gb = d["gn"] if d["gn"] is not None else (None, None, None)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.check(lib.mvb_mbd_conv_test(kind, d["x"].data_ptr(), cin, d["x"].shape[1], d["w"].data_ptr(), cout, K, stride, dil, pad,
                                  ptr(stats), ptr(gw), ptr(gb), d["groups"], ptr(d["bias"]), ptr(d["emb"]), ptr(d["resid"]),
                                  y.data_ptr(), int(use_tc), st))
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + cout * tout:]).all(), "write outside [Cout, Tout]"
    assert not torch.isnan(y).any(), "elements of [Cout, Tout] not written"
    return y.view(cout, tout)


def _conv(kind, x, w, stride, dil, pad):
    x = x.unsqueeze(0)
    if kind == 0:
        return F.conv1d(x, w, padding=pad, dilation=dil)[0]
    if kind == 1:
        tpad = -(-x.shape[-1] // stride) * stride
        return F.conv1d(F.pad(x, (0, tpad - x.shape[-1])), w, stride=stride, padding=pad)[0]
    return F.conv_transpose1d(x, w, stride=stride, padding=pad)[0]


def _reference(kind, d, K, stride, dil, pad, use_tc, cin):
    """(ref, elementwise bound, ||conv||) for one call."""
    x = d["x"]
    dx = torch.zeros_like(x, dtype=torch.float64)
    f = x
    if d["gn"] is not None:
        stats, gw, gb = d["gn"]
        cpg = cin // d["groups"]
        m = stats[:, 0].repeat_interleave(cpg)[:, None]
        r = stats[:, 1].repeat_interleave(cpg)[:, None]
        a = (x - m) * r
        pre = a.double() * gw.double()[:, None] + gb.double()[:, None]
        f = torch.relu(pre).float()
        dx = 3 * U * ((a.double() * gw.double()[:, None]).abs() + gb.double().abs()[:, None])
    if use_tc:
        hi = f.to(torch.bfloat16).float()
        xh = hi.double() + (f - hi).to(torch.bfloat16).double()
        if d["gn"] is not None:
            dx = dx + 2.0 ** -16 * f.double().abs()
        wd = d["w"].to(torch.bfloat16).double()
    else:
        xh, wd = f.double(), d["w"].double()
    y = _conv(kind, xh, wd, stride, dil, pad)
    A = _conv(kind, xh.abs(), wd.abs(), stride, dil, pad)
    bound = _gamma(kind, cin, K, use_tc) * A + _conv(kind, dx, wd.abs(), stride, dil, pad)
    ref = y.clone()
    extra = y.abs()
    for key in ("bias", "emb"):
        if d[key] is not None:
            ref = ref + d[key].double()[:, None]
            extra = extra + d[key].double().abs()[:, None]
    if d["resid"] is not None:
        ref = ref + d["resid"].double()
    bound = bound + 2 * U * (extra + ref.abs()) + 1e-30
    return ref, bound, float(y.norm())


def _case(label, kind, cin, cout, K, stride, dil, pad, tin, *, gn=True, bias=False, emb=False, resid=False, groups=4,
          use_tc=True, seed=0):
    d = _make(kind, cin, cout, K, stride, tin, seed, gn, bias, emb, resid, groups)
    got = _run(kind, d, cin, cout, K, stride, dil, pad, use_tc).double()
    ref, bound, ynorm = _reference(kind, d, K, stride, dil, pad, use_tc, cin)
    err = (got - ref).abs()
    ratio, nw = float((err / bound).max()), float(err.norm() / ynorm)
    gam = _gamma(kind, cin, K, use_tc)
    print(f"{label} {'tc' if use_tc else 'cuda-core'}: max |err|/bound {ratio:.2e} [gamma={gam:.2e}], normwise {nw:.2e}")
    bad = (err > bound).nonzero()
    assert bad.numel() == 0, f"{label}: {bad.shape[0]} elements over the bound, first at {bad[0].tolist()}"
    assert nw < NORMWISE, f"{label}: normwise {nw:.2e}"


# ---- every tensor-core convolution of the default configuration at 12 frames ----------------------------------------
@pytest.mark.parametrize("lvl", [1, 2, 3])
def test_default_strided(lvl):
    cin, cout, tin = WIDTHS[lvl - 1], WIDTHS[lvl], LENGTHS[lvl - 1]
    for use_tc in (True, False):
        _case(f"strided {cin}->{cout} Tin={tin}", 1, cin, cout, 8, 4, 1, 2, tin, gn=False, use_tc=use_tc, seed=lvl)


@pytest.mark.parametrize("lvl", [0, 1, 2, 3])
@pytest.mark.parametrize("dil", [1, 2, 4])
def test_default_resblock_conv(lvl, dil):
    c, t = WIDTHS[lvl], LENGTHS[lvl]
    for use_tc in (True, False):
        _case(f"resblock k3 C={c} T={t} dil={dil}", 0, c, c, 3, 1, dil, dil, t, gn=True, bias=True, emb=True, resid=True,
              use_tc=use_tc, seed=10 * lvl + dil)


@pytest.mark.parametrize("lvl", [3, 2, 1, 0])
def test_default_transposed(lvl):
    cin, cout, tin = WIDTHS[lvl], (WIDTHS[lvl - 1] if lvl else 1), LENGTHS[lvl]
    for use_tc in (True, False):
        _case(f"transposed {cin}->{cout} Tin={tin}", 2, cin, cout, 8, 4, 1, 2, tin, gn=True, use_tc=use_tc, seed=20 + lvl)


# ---- edges ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tin", [1, 2, 127, 128, 129])
def test_short_and_ragged_lengths(tin):
    """Lengths at and around one 128-column tile, down to a single column where every tap shift but one reads padding."""
    _case(f"k3 C=192 T={tin}", 0, 192, 192, 3, 1, 2, 2, tin, bias=True, emb=True, resid=True, seed=tin)
    _case(f"strided 192->768 Tin={tin}", 1, 192, 768, 8, 4, 1, 2, tin, gn=False, seed=tin + 1)
    _case(f"transposed 768->192 Tin={tin}", 2, 768, 192, 8, 4, 1, 2, tin, seed=tin + 2)


def test_long_level0_run():
    _case("k3 C=48 T=30000", 0, 48, 48, 3, 1, 1, 1, 30000, bias=True, emb=True, resid=True, seed=5)
    _case("strided 48->192 Tin=30000", 1, 48, 192, 8, 4, 1, 2, 30000, gn=False, seed=6)
    _case("transposed 48->1 Tin=30000", 2, 48, 1, 8, 4, 1, 2, 30000, seed=7)


@pytest.mark.parametrize("cin,groups", [(32, 4), (33, 3), (100, 4)])
@pytest.mark.parametrize("cout", [1, 200])
def test_channel_padding_and_partial_warps(cin, groups, cout):
    """Cin not a multiple of 64 (zero-padded taps and activation columns); Cout = 1 and 200 (partial consumer warps,
    a second 128-channel tile)."""
    _case(f"k3 {cin}->{cout}", 0, cin, cout, 3, 1, 1, 1, 300, groups=groups, bias=True, emb=True, resid=True, seed=cin + cout)
    _case(f"strided {cin}->{cout} (k4 s2)", 1, cin, cout, 4, 2, 1, 1, 301, gn=False, seed=cin + cout + 1)
    _case(f"transposed {cin}->{cout} (k4 s2)", 2, cin, cout, 4, 2, 1, 1, 150, groups=groups, seed=cin + cout + 2)


# ---- CUDA-core kernels the engine runs for narrow inputs (and everywhere under MVB_MBD_CUDA_CORES) --------------------
@pytest.mark.parametrize("tin", [1, 7, 145, 3833, 144000])
def test_level0_encoder_conv_cuda_cores(tin):
    """The first encoder convolution of every UNet call, Cin = 1 -> 48, k8 s4 (k_mbd_conv<8, 4, 1>, always on the CUDA
    cores): lengths that are and are not multiples of the stride, up to 6 s."""
    _case(f"strided 1->48 Tin={tin}", 1, 1, 48, 8, 4, 1, 2, tin, gn=False, use_tc=False, seed=tin)


@pytest.mark.parametrize("tf", [1, 12, 375])
def test_codec_conv_cuda_cores(tf):
    """conv_codec: K = 1, 128 -> 3072 with bias (k_mbd_conv<1, 1, 4>)."""
    _case(f"codec 128->3072 Tf={tf}", 0, 128, 3072, 1, 1, 1, 0, tf, gn=False, bias=True, use_tc=False, seed=tf)


@pytest.mark.parametrize("cin,cout", [(1, 16), (16, 32), (64, 128), (48, 192)])
@pytest.mark.parametrize("tin", [1, 129, 3833])
def test_k4_s2_cuda_cores(cin, cout, tin):
    """The (k4, s2) UNet on the CUDA cores: k_mbd_conv<4, 2, 2> and k_mbd_convtr<2>, including widths below 32 channels."""
    _case(f"strided {cin}->{cout} (k4 s2) Tin={tin}", 1, cin, cout, 4, 2, 1, 1, tin, gn=False, use_tc=False, seed=cin + tin)
    if cin > 1:
        _case(f"transposed {cout}->{cin} (k4 s2) Tin={tin}", 2, cout, cin, 4, 2, 1, 1, tin, use_tc=False, seed=cout + tin)


# ---- GroupNorm statistics from the engine's kernels feeding the convolution ---------------------------------------
def _gn_stats_hook(x, groups):
    from mvb200 import _lib as L
    lib = L.load()
    out = torch.full((2 * GUARD + 2 * groups,), float("nan"), device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.check(lib.mvb_mbd_op_test(0, x.data_ptr(), None, None, None, None, out[GUARD:].data_ptr(), x.shape[0], x.shape[1], groups,
                                1e-5, 0.0, 0.0, 0.0, 0.0, 0, st))
    assert torch.isnan(out[:GUARD]).all() and torch.isnan(out[GUARD + 2 * groups:]).all()
    return out[GUARD:GUARD + 2 * groups].view(groups, 2).contiguous()


@pytest.mark.parametrize("lvl", [0, 1, 2, 3])
@pytest.mark.parametrize("use_tc", [True, False])
def test_gn_stats_feed_the_resblock_conv(lvl, use_tc):
    """GroupNorm statistics from k_gn_partial + k_gn_final (mvb_mbd_op_test) feed one ResBlock convolution per level.
    The reference is the one above with the correctly rounded float64 statistics; the kernel's statistics are within
    2 u24 of the exact ones (tests/test_mbd_ops_gpu.py), so within 3 u24 (u24 = 2^-24) of the rounded ones: per element
    the prologue input moves by at most |gain| (|x - mean| d_rstd + (rstd + d_rstd) d_mean), propagated through |W|."""
    c, t = WIDTHS[lvl], LENGTHS[lvl]
    d = _make(0, c, c, 3, 1, t, 40 + lvl, True, True, True, True)
    ref, bound, ynorm = _reference(0, d, 3, 1, 1, 1, use_tc, c)
    stats, gw, gb = d["gn"]
    hook = _gn_stats_hook(d["x"], d["groups"])
    got = _run(0, dict(d, gn=(hook, gw, gb)), c, c, 3, 1, 1, 1, use_tc).double()
    cpg = c // d["groups"]
    m = stats[:, 0].double().repeat_interleave(cpg)[:, None]
    r = stats[:, 1].double().repeat_interleave(cpg)[:, None]
    em, er = 1.5 * U * m.abs(), 1.5 * U * r
    df = gw.double().abs()[:, None] * ((d["x"].double() - m).abs() * er + (r + er) * em) * (1 + 4 * U)
    wd = (d["w"].to(torch.bfloat16) if use_tc else d["w"]).double().abs()
    bound = bound + _conv(0, df, wd, 1, 1, 1)
    err = (got - ref).abs()
    ratio, nw = float((err / bound).max()), float(err.norm() / ynorm)
    print(f"gn stats -> resblock k3 C={c} T={t} {'tc' if use_tc else 'cuda-core'}: max |err|/bound {ratio:.2e}, normwise {nw:.2e}")
    assert int((err > bound).sum()) == 0 and nw < NORMWISE


def test_fp32_taps_violate_the_bound():
    """Sensitivity: the tensor-core result (bf16 taps) must fail a reference built with the unrounded fp32 taps."""
    kind, cin, cout, K, T = 0, 64, 128, 3, 512
    d = _make(kind, cin, cout, K, 1, T, 9, False, False, False, False, exact_taps=False)
    got = _run(kind, d, cin, cout, K, 1, 1, 1, True).double()
    x = d["x"]
    hi = x.to(torch.bfloat16).float()
    xh = hi.double() + (x - hi).to(torch.bfloat16).double()
    ref = _conv(kind, xh, d["w"].double(), 1, 1, 1)
    bound = _gamma(kind, cin, K, True) * _conv(kind, xh.abs(), d["w"].double().abs(), 1, 1, 1) + 2 * U * ref.abs()
    err = (got - ref).abs()
    n_over, nw = int((err > bound).sum()), float(err.norm() / ref.norm())
    print(f"fp32-tap reference: {n_over} of {err.numel()} elements over the bound, normwise {nw:.2e}")
    assert n_over > 0 and nw > 10 * NORMWISE
