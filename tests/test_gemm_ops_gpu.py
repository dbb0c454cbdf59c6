"""GPU: the weight-streaming tensor-core GEMM (csrc/tc_gemm.cuh, k_tc_gemm<EPI, NC>) at every epilogue and
accumulator instance, against a float64 computation of the same operation.

Reference.  It reproduces every rounding the kernel declares, so that the only difference left is fp32 accumulation:
W is bf16; the activation row is v = x, or with the RMSNorm prologue v = (x * rs) * gain in fp32 with
rs = rsqrt(fl(fl(sum x^2) / K + eps)) as k_prep_b computes it; then hi = bf16(v), lo = bf16(v - hi) and
    ref = (hi + lo) . W^T   (hi . W^T when split_lo = 0)
in float64, followed by the epilogue in float64.

Elementwise bound.  With A = |x^| . |W|^T (x^ = hi + lo, all in float64) every element must satisfy
    |out - ref| <= gamma_K * A + tiny.
Derivation of gamma_K for this kernel's order of accumulation.  Each mma.sync.m16n8k16 adds 16 exact bf16 x bf16 products to
the fp32 accumulator c.  Modelled worst case (alignment of the 17 addends to the largest exponent with truncation, then a
truncating normalisation): one MMA changes the exact value by at most 18 u (|c| + sum |p_i|), u = 2^-23.  A split runs
n = 4 (1 + split_lo) MMAs per 64-wide k-block, sequentially over its k-blocks (hi then lo into the same accumulator);
|c| never exceeds the sum of the magnitudes already added, so its error is at most 18 u n sum|p|.  The split-K reduction
adds ksplit fp32 partials in a fixed order, at most ksplit u sum|p| more.  With n taken over all K / 64 k-blocks (an
upper bound for any split):
    gamma_K = (18 * 4 * (K / 64) * (1 + split_lo) + ksplit) * u.
The RMSNorm prologue adds one explicit term: rsqrtf is within 2 ulp of the correctly rounded value (the test inputs make
the sum of squares exact, so nothing else differs), which moves v by <= 2^-22 |v| and can move lo by one bf16 ulp of
|v - hi| <= 2^-8 |v|, i.e. tau = 2^-22 + 2^-16 relative to |x^|.  Epilogues add their own fp32 roundings (below).
A wrong row, column or tile is off by |y| itself, orders of magnitude above the bound wherever it lands.

Normwise bound.  ||out - ref||_F / ||y_ref||_F < NORMWISE = 1e-4.  Dropping the lo term gives ~1.7e-3 (the rms
relative bf16 rounding error of the activations), one bf16 rounding of the result about the same: both are > 15x above.

Every call also writes into a NaN-filled output with ldo > M and spare rows: only [0, R) x [0, M) may change and
nothing inside it may stay NaN (stray writes are detected by reading back, nothing is provoked)."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
NORMWISE = 1e-4
TAU_GAIN = 2.0 ** -22 + 2.0 ** -16
EPS = 1e-5
G_STORE, G_RESID, G_SWIGLU, G_QKV = 0, 1, 2, 3
R_ALL = [1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 48, 63, 64, 65, 96, 127, 128]


def _lib():
    from mvb200 import _lib as L
    return L, L.load()


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def gamma_k(K, split_lo, ksplit):
    return (18 * 4 * (K // 64) * (1 + int(split_lo)) + ksplit) * U


def _ksplit_bound(M, K, ksplit):
    """An upper bound of the split count the launcher may pick (auto: at most 16) -- it only enters gamma_K linearly."""
    return 16 if ksplit <= 0 else max(1, min(ksplit, _n_sm() // ((M + 127) // 128)))


def _inputs(M, K, R, seed, gain=False, w3=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    W = (torch.randn(M, K, generator=g, device="cuda") * 0.05).to(torch.bfloat16)
    W3 = (torch.randn(M, K, generator=g, device="cuda") * 0.05).to(torch.bfloat16) if w3 else None
    if gain:
        # x on a k/16 grid, |k| <= 32: every partial sum of squares is an integer / 256 below 2^24 / 256, so the kernel's
        # fp32 sum of squares is exact in any order and only rsqrtf's rounding differs from the reference
        x = torch.randint(-32, 33, (R, K), generator=g, device="cuda").float() / 16
        gw = (1 + 0.1 * torch.randn(K, generator=g, device="cuda")).to(torch.bfloat16)
    else:
        x = torch.randn(R, K, generator=g, device="cuda")
        gw = None
    return W, W3, x, gw


def _xhat(x, gw, split_lo):
    """k_prep_b's activation operand, exactly: fp32 RMSNorm prologue, then the two-term bf16 split (float64 result)."""
    K = x.shape[1]
    v = x
    if gw is not None:
        ss = (x.double() ** 2).sum(-1, keepdim=True).float()       # exact (see _inputs)
        rs = torch.rsqrt(ss / K + EPS)
        v = (x * rs) * gw.float()
    hi = v.to(torch.bfloat16).float()
    lo = (v - hi).to(torch.bfloat16).float()
    return (hi.double() + lo.double()) if split_lo else hi.double()


def _call(epi, W, x, R, M, K, *, W3=None, gw=None, split_lo=1, ksplit=0, out0=None, kv=None, ldo_pad=5, spare_rows=3):
    """Run the hook into a NaN-filled [R + spare_rows, M + ldo_pad] buffer (out0 preloaded into [0, R) x [0, M) for the
    residual epilogue); returns the whole buffer."""
    L, lib = _lib()
    ldo = M + ldo_pad
    out = torch.full((R + spare_rows, ldo), float("nan"), device="cuda")
    if out0 is not None:
        out[:R, :M] = out0
    kc = vc = rc = rp = None
    H = S_max = D = kv_fp32 = 0
    if kv is not None:
        kc, vc, rc, rp, H, S_max, D, kv_fp32 = kv
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ptr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    L.check(lib.mvb_gemm_test(epi, W.data_ptr(), ptr(W3), M, K, x.data_ptr(), x.shape[1], R, ptr(gw), EPS, int(split_lo), ksplit,
                              out.data_ptr(), ldo, ptr(kc), ptr(vc), ptr(rc), ptr(rp), H, S_max, D, kv_fp32, st))
    return out


def _check_footprint(out, R, M):
    inside = out[:R, :M]
    assert not torch.isnan(inside).any(), "elements of [0, R) x [0, M) were not written"
    mask = torch.ones_like(out, dtype=torch.bool)
    mask[:R, :M] = False
    assert torch.isnan(out[mask]).all(), "the kernel wrote outside [0, R) x [0, M)"


def _assess(label, got, ref, bound, y_norm):
    """Elementwise bound (returns the worst err / bound ratio) and the normwise check."""
    err = (got.double() - ref).abs()
    ratio = float((err / bound).max())
    nw = float(err.norm() / y_norm)
    print(f"{label}: max |err|/bound {ratio:.2e}, normwise {nw:.2e} (< {NORMWISE:.0e})")
    bad = (err > bound).nonzero()
    assert bad.numel() == 0, f"{label}: {bad.shape[0]} elements over the bound, first at {bad[0].tolist()}"
    assert nw < NORMWISE, f"{label}: normwise error {nw:.2e}"
    return ratio


def _store_case(M, K, R, *, split_lo=1, ksplit=0, gain=False, accumulate=False, seed=0, label=""):
    W, _, x, gw = _inputs(M, K, R, seed, gain=gain)
    xh = _xhat(x, gw, split_lo)
    Wd = W.double()
    y = xh @ Wd.t()
    A = xh.abs() @ Wd.abs().t()
    gam = gamma_k(K, split_lo, _ksplit_bound(M, K, ksplit)) + (TAU_GAIN if gain else 0.0)
    bound = gam * A + 1e-30
    out0 = None
    ref = y
    if accumulate:
        out0 = torch.randn(R, M, generator=torch.Generator(device="cuda").manual_seed(seed + 7), device="cuda")
        ref = y + out0.double()
        bound = bound + U * (ref.abs() + bound)          # the fp32 add of the residual epilogue
    out = _call(G_RESID if accumulate else G_STORE, W, x, R, M, K, gw=gw, split_lo=split_lo, ksplit=ksplit, out0=out0)
    _check_footprint(out, R, M)
    name = label or f"M={M} K={K} R={R} lo={split_lo} ks={ksplit} gain={int(gain)} acc={int(accumulate)}"
    return _assess(f"{name} [gamma_K={gam:.2e}]", out[:R, :M], ref, bound, y.norm())


@pytest.mark.parametrize("R", R_ALL)
def test_every_row_count(R):
    """All four accumulator instances (NC = 2/4/8/16) and every run-time early exit nc < NC; K = 576 is nine k-blocks,
    the smallest K the automatic rule splits; M = 1000 has a ragged last tile."""
    for ks in (1, 0):
        _store_case(1000, 576, R, ksplit=ks, seed=R)
    _store_case(1000, 576, R, ksplit=0, gain=True, accumulate=True, seed=100 + R)


@pytest.mark.parametrize("M", [64, 127, 129, 2562, 16512])
@pytest.mark.parametrize("K", [64, 128, 512, 576, 2048, 5632])
def test_shapes_and_split_rules(M, K):
    """Less than one tile, ragged tails and more than 128 tiles (the ksplit = 1 fallback); one k-block up to the FFN
    width; the nkb <= 8 / nkb = 9 split rule; ksplit 1, automatic and forced above the k-block count (splits that own
    no k-block and, for R = 9 < ksplit, splits that reduce no row)."""
    nkb = K // 64
    for ks in (1, 0, nkb + 3):
        _store_case(M, K, 9, ksplit=ks, seed=M + K)


# (one bf16 term after the RMSNorm is not listed: an ulp of rsqrtf can move hi itself by 2^-8, so no exact reference exists)
@pytest.mark.parametrize("split_lo,gain", [(0, False), (1, False), (1, True)])
@pytest.mark.parametrize("accumulate", [False, True])
def test_prologue_and_epilogue_variants(split_lo, gain, accumulate):
    for R, ks in ((2, 0), (33, 1), (128, 0)):
        _store_case(2048, 2048, R, split_lo=split_lo, ksplit=ks, gain=gain, accumulate=accumulate, seed=R + 3)


def test_split_k_is_bit_reproducible():
    W, _, x, _ = _inputs(2562, 2048, 24, 11)
    a = _call(G_STORE, W, x, 24, 2562, 2048, ksplit=0)
    b = _call(G_STORE, W, x, 24, 2562, 2048, ksplit=0)
    c = _call(G_STORE, W, x, 24, 2562, 2048, ksplit=7)
    d = _call(G_STORE, W, x, 24, 2562, 2048, ksplit=7)
    assert torch.equal(a[:24, :2562], b[:24, :2562]) and torch.equal(c[:24, :2562], d[:24, :2562])


def test_dropped_lo_term_violates_the_bound():
    """Sensitivity: the one-term (hi only) result must fail the two-term reference's elementwise and normwise bounds."""
    M, K, R = 1024, 512, 16
    W, _, x, _ = _inputs(M, K, R, 21)
    xh = _xhat(x, None, 1)
    Wd = W.double()
    ref = xh @ Wd.t()
    bound = gamma_k(K, 1, _ksplit_bound(M, K, 0)) * (xh.abs() @ Wd.abs().t())
    got = _call(G_STORE, W, x, R, M, K, split_lo=0)[:R, :M].double()
    err = (got - ref).abs()
    n_over, nw = int((err > bound).sum()), float(err.norm() / ref.norm())
    print(f"hi-only result vs hi+lo bound: {n_over} of {R * M} elements over, normwise {nw:.2e}")
    assert n_over > 0 and nw > 10 * NORMWISE


# ---------------------------------------------------------------------------------------------------------------
# SwiGLU: out = silu(y) * y3, y = x^ W^T, y3 = x^ W3^T.  With b1 = gamma_K A1, b3 = gamma_K A3 bounding the two GEMMs:
#     |out - ref| <= 1.1 b1 (|y3| + b3) + (|silu(y)| + 1.1 b1) b3 + 8 u |ref|
# (|silu'| <= 1.1; expf is within 2 ulp, the add, division and product round once each: < 8 u relative).

def _swiglu_bound(y, y3, b1, b3, ref):
    silu = y * torch.sigmoid(y)
    return 1.1 * b1 * (y3.abs() + b3) + (silu.abs() + 1.1 * b1) * b3 + 8 * U * ref.abs() + 1e-30


def _swiglu_ref(W, W3, x, split_lo=1):
    xh = _xhat(x, None, split_lo)
    y, y3 = xh @ W.double().t(), xh @ W3.double().t()
    return xh, y, y3, y * torch.sigmoid(y) * y3


@pytest.mark.parametrize("R", [5, 17, 48, 128])
@pytest.mark.parametrize("ksplit", [1, 0])
def test_swiglu(R, ksplit):
    """The only two-operand instance (NA = 2): every NC, ksplit = 1 and > 1 (auto = 16 splits here, so R = 5 < ksplit);
    the split-K reduction reads y3 at scratch row Rpad + n.  Split-K results are bit-reproducible."""
    M, K = 1000, 2048
    W, W3, x, _ = _inputs(M, K, R, 30 + R, w3=True)
    xh, y, y3, ref = _swiglu_ref(W, W3, x)
    gam = gamma_k(K, 1, _ksplit_bound(M, K, ksplit))
    b1, b3 = gam * (xh.abs() @ W.double().abs().t()), gam * (xh.abs() @ W3.double().abs().t())
    out = _call(G_SWIGLU, W, x, R, M, K, W3=W3, ksplit=ksplit)
    _check_footprint(out, R, M)
    _assess(f"swiglu M={M} K={K} R={R} ks={ksplit} [gamma_K={gam:.2e}]", out[:R, :M], ref, _swiglu_bound(y, y3, b1, b3, ref), ref.norm())
    again = _call(G_SWIGLU, W, x, R, M, K, W3=W3, ksplit=ksplit)
    assert torch.equal(out[:R, :M], again[:R, :M])


def test_swiglu_swapped_operands_violate_the_bound():
    """Sensitivity: silu(x W3^T) * (x W^T) is not the kernel's result; the bound must say so."""
    M, K, R = 1000, 2048, 16
    W, W3, x, _ = _inputs(M, K, R, 41, w3=True)
    xh, y, y3, _ = _swiglu_ref(W3, W, x)              # roles swapped
    gam = gamma_k(K, 1, 16)
    b1, b3 = gam * (xh.abs() @ W3.double().abs().t()), gam * (xh.abs() @ W.double().abs().t())
    ref = y * torch.sigmoid(y) * y3
    got = _call(G_SWIGLU, W, x, R, M, K, W3=W3)[:R, :M].double()
    n_over = int(((got - ref).abs() > _swiglu_bound(y, y3, b1, b3, ref)).sum())
    print(f"swiglu with W / W3 swapped in the reference: {n_over} of {R * M} elements over the bound")
    assert n_over > R * M // 2


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kv_fp32", [1, 0])
@pytest.mark.parametrize("R,ksplit", [(7, 1), (40, 0), (128, 0)])
def test_qkv_scatter(kv_fp32, R, ksplit):
    """out = x^ W^T (STORE bound), and the K / V thirds land at (row_cache[n], head, row_pos[n], d): bit for bit the
    kernel's own out value (fp32 cache) or bf16_rn of it (bf16 cache).  Caches start NaN-filled; every entry no row
    addresses must still be NaN.  Cache rows / positions are a non-monotonic selection that includes positions 0 and
    S_max - 1."""
    H, S_max, n_rows = 2, 67, 3
    D = 128 * H
    M, K = 3 * D, 512
    W, _, x, _ = _inputs(M, K, R, 50 + R)
    special = [S_max - 1, (n_rows - 1) * S_max, S_max]            # (row, position) = (0, S_max - 1), (2, 0), (1, 0)
    rest = [p for p in torch.randperm(n_rows * S_max, generator=torch.Generator().manual_seed(R)).tolist() if p not in special]
    pairs = torch.tensor([special[0]] + rest[:R - 3] + [special[1], special[2]])
    row_cache, row_pos = (pairs // S_max).int(), (pairs % S_max).int()
    dt = torch.float32 if kv_fp32 else torch.bfloat16
    kc = torch.full((n_rows, H, S_max, 128), float("nan"), dtype=dt, device="cuda")
    vc = torch.full_like(kc, float("nan"))
    rc, rp = row_cache.cuda(), row_pos.cuda()
    out = _call(G_QKV, W, x, R, M, K, ksplit=ksplit, kv=(kc, vc, rc, rp, H, S_max, D, kv_fp32))
    _check_footprint(out, R, M)
    xh = _xhat(x, None, 1)
    y = xh @ W.double().t()
    gam = gamma_k(K, 1, _ksplit_bound(M, K, ksplit))
    _assess(f"qkv R={R} ks={ksplit} kv_fp32={kv_fp32} [gamma_K={gam:.2e}]", out[:R, :M], y,
            gam * (xh.abs() @ W.double().abs().t()) + 1e-30, y.norm())
    o = out[:R, :M]
    want_k = o[:, D:2 * D].reshape(R, H, 128).to(dt)
    want_v = o[:, 2 * D:].reshape(R, H, 128).to(dt)
    got_k, got_v = kc[rc.long(), :, rp.long()], vc[rc.long(), :, rp.long()]
    view = torch.int32 if kv_fp32 else torch.int16
    assert torch.equal(got_k.view(view), want_k.view(view)), "K cache entries differ from the kernel's own output"
    assert torch.equal(got_v.view(view), want_v.view(view)), "V cache entries differ from the kernel's own output"
    for cache in (kc, vc):
        untouched = torch.ones(n_rows, S_max, dtype=torch.bool, device="cuda")
        untouched[rc.long(), rp.long()] = False
        assert torch.isnan(cache.permute(0, 2, 1, 3)[untouched].float()).all(), "a cache entry no row addresses was written"
