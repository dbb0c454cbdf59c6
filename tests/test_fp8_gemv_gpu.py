"""GPU: the fp8 decode GEMV (csrc/gemv_f8.cuh, k_gemv_f8<EPI, NB>) at every epilogue and production (M, K) for 1 to 8 slots,
and the fp8 widening (k_f8_widen), against float64 computations over the host's (q, s) (mvb200/quantize.py).

Reference.  q (e4m3) and s (bf16) are exact data.  The activation row is v = x, or with RMSNorm v = (x * rs) * gain with
rs = rsqrt(sum x^2 / K + eps) in fp32; then ref_j = s_j (v . q_j) in float64, followed by the epilogue in float64.

Elementwise bound.  With A_j = s_j (|v| . |q_j|) every element must satisfy |out - ref| <= gamma * A + u |ref| + tiny.
The kernel multiplies the exact bf16 weights by the activations carried as two bf16 terms, x = hi + lo to 2^-17 relative
(at most 2^-16 of |v| for every product).  Warp w sums its K / 8 in K / 128 k-steps, each adding a hi and a lo MMA of 16
exact products into the fp32 accumulator: 2 K / 128 accumulations, each allowed 2 ulp (2^-22), then 7 adds of the warps'
sums.  RMSNorm multiplies the gained sum by rs (the k/16 activation grid makes every sum of squares exact, so rs is the
reference's to rsqrtf's error, 2^-21 relative) and the fp32 gain product rounds once.  Hence gamma = (2 K / 128 + 8) 2^-22
+ 2^-16 (+ 2^-21 + 2^-23 with RMSNorm), and the scale multiply adds one rounding.

Sensitivity.  References built with each row's scale taken from its neighbour, with the subnormal codes flushed to zero,
and with the two CFG rows of a slot swapped must violate the bound.  Batch independence: every slot's outputs at 8 slots
are bit-identical to the same slot run alone.

SM counts.  The grid (f8_gemv_ctas) depends on the SM count: the float64 cases rerun with the grid planned for 114, 78,
60, 54 and 16 SMs, where CTAs own 2 or 3 of wo's and w2's 16-row blocks and lm_head's ragged tail block is a CTA's third
from 80 SMs down (a Python mirror of the deal asserts which)."""
import ctypes as C
import functools

import pytest
import torch

from mvb200 import quantize as Q

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
NORMWISE = 1e-4
EPS = 1e-5
STORE, RESID, SWIGLU, QKV = 0, 1, 2, 3
# batch entry -> slot (rows 2 s, 2 s + 1); never the identity.  3 and 5 leave an n8 block of MMA columns partly filled.
SLOTS = {1: [2], 2: [5, 1], 3: [4, 0, 2], 4: [6, 1, 3, 0], 5: [2, 7, 0, 5, 3], 8: [3, 7, 0, 9, 4, 1, 8, 5]}


def _lib():
    from mvb200 import _lib as L
    return L, L.load()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def gamma(K, gain):
    return (2 * K / 128 + 8) * 2.0 ** -22 + 2.0 ** -16 + ((2.0 ** -21 + 2.0 ** -23) if gain else 0.0)


@functools.lru_cache(maxsize=None)
def _mat(M, K, seed):
    """(fp8 matrix on the device, q float64 [M, K] and s float64 [M] on the device)"""
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(M, K, generator=g) * 0.03).to(torch.bfloat16)
    q, s = Q.quantize_fp8_per_channel(w)
    return Q.pack_fp8_matrix(q, s).cuda(), q.double().cuda(), s.double().cuda()


def _x(n_rows, K, seed, gain):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if gain:
        # x on a k/16 grid, |k| <= 32: every partial sum of squares is exact in fp32 in any order
        x = torch.randint(-32, 33, (n_rows, K), generator=g, device="cuda").float() / 16
        gw = (1 + 0.1 * torch.randn(K, generator=g, device="cuda")).to(torch.bfloat16)
    else:
        x = torch.randn(n_rows, K, generator=g, device="cuda")
        gw = None
    return x, gw


def _v(x, gw):
    if gw is None:
        return x.double()
    K = x.shape[1]
    ss = (x.double() ** 2).sum(-1, keepdim=True).float()
    rs = torch.rsqrt(ss / K + EPS)
    return ((x * rs) * gw.float()).double()


def _rows(slots):
    return [r for s in slots for r in (2 * s, 2 * s + 1)]


def _call(epi, Wp, M, K, x, slots, *, W3p=None, gw=None, out0=None, kv=None, ldo_pad=5):
    L, lib = _lib()
    out = torch.full((x.shape[0], M + ldo_pad), float("nan"), device="cuda")
    if out0 is not None:
        r = _rows(slots)
        out[r, :M] = out0[r]
    slot_map = torch.tensor(slots, dtype=torch.int32, device="cuda")
    kc = vc = pos = None
    H = S_max = D = kv_fp32 = 0
    if kv is not None:
        kc, vc, pos, H, S_max, D, kv_fp32 = kv
    if pos is None:
        pos = torch.zeros(x.shape[0] // 2, dtype=torch.int32, device="cuda")
    ptr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    L.check(lib.mvb_f8_gemv_test(epi, Wp.data_ptr(), ptr(W3p), M, K, x.data_ptr(), x.shape[1], len(slots), ptr(gw), EPS,
                                 out.data_ptr(), M + ldo_pad, ptr(kc), ptr(vc), slot_map.data_ptr(), pos.data_ptr(), H, S_max,
                                 D, kv_fp32, _stream()))
    return out


def _check_footprint(out, rows, M):
    assert not torch.isnan(out[rows, :M]).any(), "elements of the slots' rows x [0, M) were not written"
    mask = torch.ones_like(out, dtype=torch.bool)
    for r in rows:
        mask[r, :M] = False
    assert torch.isnan(out[mask]).all(), "the kernel wrote outside the slots' rows x [0, M)"


def _violations(got, ref, bound):
    return int(((got.double() - ref).abs() > bound).sum())


def _assess(label, got, ref, bound):
    err = (got.double() - ref).abs()
    nw = float(err.norm() / ref.norm())
    print(f"{label}: max |err|/bound {float((err / bound).max()):.2e}, normwise {nw:.2e}")
    bad = (err > bound).nonzero()
    assert bad.numel() == 0, f"{label}: {bad.shape[0]} elements over the bound, first at {bad[0].tolist()}"
    assert nw < NORMWISE, f"{label}: normwise error {nw:.2e}"


def _swiglu_bound(y, y3, b1, b3, ref):
    """|silu'| <= 1.1; expf within 2 ulp and the add, division and product round once each: < 8 u relative."""
    silu = y * torch.sigmoid(y)
    return 1.1 * b1 * (y3.abs() + b3) + (silu.abs() + 1.1 * b1) * b3 + 8 * U * ref.abs() + 1e-30


def _scaled(v, qd, sd, gam):
    """(ref = s (v . q^T), its bound gamma s (|v| . |q|^T) + the rounding of the scale multiply)"""
    y = (v @ qd.t()) * sd
    b = gam * ((v.abs() @ qd.abs().t()) * sd)
    return y, b + U * (y.abs() + b) + 1e-30


# every fp8 matrix of MetaVoice-1B under the epilogue the engine gives it (lm_head: STORE with the ln_f prologue)
CASES = [(QKV, 6144, 2048), (RESID, 2048, 2048), (SWIGLU, 5632, 2048), (RESID, 2048, 5632), (STORE, 2562, 2048)]
GAIN = {QKV: True, RESID: False, SWIGLU: True, STORE: True}


@pytest.mark.parametrize("n_utts", sorted(SLOTS))
@pytest.mark.parametrize("epi,M,K", CASES)
def test_gemv_f8(epi, M, K, n_utts):
    slots, gain = SLOTS[n_utts], GAIN[epi]
    Wp, qd, sd = _mat(M, K, 1000 * M + K)
    rows = _rows(slots)
    n_rows = 2 * max(slots) + 5
    x, gw = _x(n_rows, K, M + K + n_utts, gain)
    v = _v(x, gw)[rows]
    gam = gamma(K, gain)
    label = f"epi={epi} M={M} K={K} utts={n_utts} [gamma={gam:.2e}]"
    if epi == SWIGLU:
        W3p, q3d, s3d = _mat(M, K, 1000 * M + K + 1)
        (y, b1), (y3, b3) = _scaled(v, qd, sd, gam), _scaled(v, q3d, s3d, gam)
        ref = y * torch.sigmoid(y) * y3
        out = _call(SWIGLU, Wp, M, K, x, slots, W3p=W3p, gw=gw)
        _check_footprint(out, rows, M)
        _assess(label, out[rows, :M], ref, _swiglu_bound(y, y3, b1, b3, ref))
        return
    ref, bound = _scaled(v, qd, sd, gam)
    out0 = kv = None
    if epi == RESID:
        out0 = torch.randn(n_rows, M, generator=torch.Generator(device="cuda").manual_seed(K), device="cuda")
        ref = ref + out0[rows].double()
        bound = bound + U * (ref.abs() + bound)          # the fp32 add of the residual epilogue
    if epi == QKV:
        D = M // 3
        H, S_max = D // 128, 37
        pos = torch.randint(0, S_max, (n_rows // 2,), generator=torch.Generator().manual_seed(M + n_utts), dtype=torch.int32)
        kv_fp32 = int(n_utts % 2)                         # both cache types
        dt = torch.float32 if kv_fp32 else torch.bfloat16
        kc = torch.full((n_rows, H, S_max, 128), float("nan"), dtype=dt, device="cuda")
        vc = torch.full_like(kc, float("nan"))
        kv = (kc, vc, pos.cuda(), H, S_max, D, kv_fp32)
    out = _call(epi, Wp, M, K, x, slots, gw=gw, out0=out0, kv=kv)
    _check_footprint(out, rows, M)
    _assess(label, out[rows, :M], ref, bound)
    if epi == QKV:
        view = torch.int32 if kv_fp32 else torch.int16
        for s in slots:
            p = int(pos[s])
            for r in (2 * s, 2 * s + 1):
                assert torch.equal(kc[r, :, p].view(view), out[r, D:2 * D].reshape(H, 128).to(dt).view(view)), "K cache"
                assert torch.equal(vc[r, :, p].view(view), out[r, 2 * D:3 * D].reshape(H, 128).to(dt).view(view)), "V cache"


def f8_gemv_ctas(n_blocks, n_sm, ipc=3):
    """Mirror of f8_gemv_ctas (csrc/gemv_f8.cuh): one 16-row block per SM where there are enough, never more than F8_IPC
    = 3 per CTA."""
    return max(-(-n_blocks // ipc), min(n_blocks, n_sm))


def n_mine(n_blocks, n_sm):
    """Blocks CTA x owns (x, x + G, x + 2 G, ...) for every CTA of the launch, as k_gemv_f8 deals them."""
    G = f8_gemv_ctas(n_blocks, n_sm)
    return [(n_blocks - 1 - x) // G + 1 for x in range(G)]


# the capped counts of tests/test_sm_count_gpu.py that change k_gemv_f8's grid at production width: at 132 SMs wo / w2
# (128 blocks) give every CTA one block and lm_head's ragged tail (block 160) is its CTA's second
F8_SM = [114, 78, 60, 54, 16]


@pytest.mark.parametrize("G", F8_SM)
def test_gemv_f8_at_sm_counts(G):
    """test_gemv_f8's float64 cases (every production matrix and epilogue, NB = 1 and 2) with the grid planned for G SMs
    (mvb_test_set_sm_limit): wo / w2 at 2 or 3 blocks per CTA, and lm_head's tail block as a CTA's third (i = 2) from
    G = 78 down."""
    from test_sm_count_gpu import sm_limit
    with sm_limit(G) as g:
        if g != G:
            pytest.skip(f"this device has fewer than {G} SMs")
        blocks = n_mine(2048 // 16, G)
        assert max(blocks) in (2, 3), (G, sorted(set(blocks)))
        tail_cta_ctas = f8_gemv_ctas(-(-2562 // 16), G)
        tail_i = 160 // tail_cta_ctas
        assert tail_i == (2 if G <= 80 else 1), (G, tail_i)
        print(f"G={G}: wo / w2 blocks per CTA {sorted(set(blocks))} on {len(blocks)} CTAs; lm_head tail block is "
              f"i = {tail_i} of CTA {160 % tail_cta_ctas} of {tail_cta_ctas}")
        for epi, M, K in CASES:
            for n in (1, 5, 8):
                test_gemv_f8(epi, M, K, n)


@pytest.mark.parametrize("epi,M,K", CASES)
def test_batch_of_8_bit_identical_to_solo(epi, M, K):
    """Every slot's outputs at 8 slots equal, bit for bit, the same slot decoded alone (other MMA column, other n8 block)."""
    slots = SLOTS[8]
    Wp, _, _ = _mat(M, K, 1000 * M + K)
    W3p = _mat(M, K, 1000 * M + K + 1)[0] if epi == SWIGLU else None
    x, gw = _x(2 * max(slots) + 5, K, 77 + M, GAIN[epi])
    kw = dict(W3p=W3p, gw=gw)
    if epi == QKV:
        D = M // 3
        mk = lambda: (torch.zeros(x.shape[0], D // 128, 8, 128, device="cuda"), torch.zeros(x.shape[0], D // 128, 8, 128, device="cuda"),   # noqa: E731
                      None, D // 128, 8, D, 1)
        kw["kv"] = mk()
    out0 = torch.zeros(x.shape[0], M, device="cuda") if epi == RESID else None
    batch = _call(epi, Wp, M, K, x, slots, out0=out0, **kw)
    for s in slots:
        if epi == QKV:
            kw["kv"] = mk()
        solo = _call(epi, Wp, M, K, x, [s], out0=out0, **kw)
        for r in (2 * s, 2 * s + 1):
            assert torch.equal(batch[r, :M].view(torch.int32), solo[r, :M].view(torch.int32)), (epi, s, r)


def test_qkv_cache_scatter_matches_bf16_gemv():
    """With power-of-two scales s q is exact in bf16: the fp8 QKV epilogue's cache scatter lands where, and as, the bf16
    GEMV's (k_gemv via the non-production-architecture hook with no norm and no bias) does, within the GEMV bound."""
    L, lib = _lib()
    M, K, D = 768, 256, 256
    g = torch.Generator().manual_seed(4)
    q, _ = Q.quantize_fp8_per_channel((torch.randn(M, K, generator=g) * 0.03).to(torch.bfloat16))
    s = torch.exp2(torch.randint(-12, -6, (M,), generator=g).float()).to(torch.bfloat16)
    wsq = Q.dequantize_fp8(q, s).cuda()                 # exact: a power-of-two scale times an e4m3 value
    slots = SLOTS[3]
    x, _ = _x(2 * max(slots) + 2, K, 5, False)
    pos = torch.tensor([3, 6, 1, 0, 5], dtype=torch.int32, device="cuda")
    caches = []
    for hook in ("f8", "bf16"):
        kc = torch.full((x.shape[0], D // 128, 8, 128), float("nan"), device="cuda")
        vc = torch.full_like(kc, float("nan"))
        out = torch.full((x.shape[0], M), float("nan"), device="cuda")
        sm = torch.tensor(slots, dtype=torch.int32, device="cuda")
        if hook == "f8":
            Wp = Q.pack_fp8_matrix(q, s).cuda()
            L.check(lib.mvb_f8_gemv_test(QKV, Wp.data_ptr(), None, M, K, x.data_ptr(), K, 3, None, EPS, out.data_ptr(), M,
                                         kc.data_ptr(), vc.data_ptr(), sm.data_ptr(), pos.data_ptr(), D // 128, 8, D, 1, _stream()))
        else:
            L.check(lib.mvb_s1_arch_gemv_test(0, QKV, 0, wsq.data_ptr(), None, None, None, M, K, x.data_ptr(), K, 3, None, None,
                                              EPS, out.data_ptr(), M, kc.data_ptr(), vc.data_ptr(), sm.data_ptr(), pos.data_ptr(),
                                              D // 128, 8, D, 1, 0, _stream()))
        caches.append((kc, vc))
    (k8, v8), (kb, vb) = caches
    assert torch.equal(torch.isnan(k8), torch.isnan(kb)) and torch.equal(torch.isnan(v8), torch.isnan(vb)), "scatter positions"
    for a, b in ((k8, kb), (v8, vb)):
        fin = ~torch.isnan(b)
        assert fin.any()
        # the two kernels sum in different orders: equal to the fp32 accumulation error of a K = 256 dot product
        assert float((a[fin] - b[fin]).abs().max()) <= 1e-5 * float(b[fin].abs().max())


# ---- exact conversion: all 256 codes ------------------------------------------------------------------------------------
def _all_codes_matrix():
    """q [32, 256]: rows 0-15 hold every code once (row r rotated by 37 r), rows 16-31 only subnormal codes and zeros."""
    k = torch.arange(256)
    codes = torch.stack([(k + 37 * r) % 256 for r in range(16)] +
                        [torch.tensor([0x00, 0x80] + list(range(1, 8)) + list(range(0x81, 0x88)))[(k + r) % 16] for r in range(16)])
    codes = codes.to(torch.uint8)
    nan = (codes & 0x7F) == 0x7F
    return codes, nan


def _code_values(codes):
    """float64 values of e4m3 codes; the NaN codes 0x7f / 0xff read as +-480 (the kernels' documented reading)."""
    v = codes.view(torch.float8_e4m3fn).double()
    return torch.where((codes & 0x7F) == 0x7F, torch.where(codes >= 0x80, -480.0, 480.0).double(), v)


def test_widen_all_codes_exact():
    L, lib = _lib()
    codes, _ = _all_codes_matrix()
    M, K = codes.shape
    q = codes.view(torch.float8_e4m3fn)
    s = torch.ones(M, dtype=torch.bfloat16)
    buf = Q.pack_fp8_matrix(q, s).cuda()
    out = torch.empty(M, K, dtype=torch.bfloat16, device="cuda")
    L.check(lib.mvb_f8_widen_test(buf.data_ptr(), M, K, out.data_ptr(), _stream()))
    want = _code_values(codes).to(torch.bfloat16)
    assert torch.equal(out.cpu().view(torch.int16), want.view(torch.int16)), "widened codes differ from their exact values"


@pytest.mark.parametrize("M,K", [(2562, 2048), (6144, 2048), (2048, 5632), (2048, 256), (34, 512)])
def test_widen_bit_identical_to_host(M, K):
    L, lib = _lib()
    g = torch.Generator().manual_seed(M + K)
    q, s = Q.quantize_fp8_per_channel((torch.randn(M, K, generator=g) * 0.02).to(torch.bfloat16))
    out = torch.empty(M, K, dtype=torch.bfloat16, device="cuda")
    L.check(lib.mvb_f8_widen_test(Q.pack_fp8_matrix(q, s).cuda().data_ptr(), M, K, out.data_ptr(), _stream()))
    assert torch.equal(out.cpu().view(torch.int16), q.to(torch.bfloat16).view(torch.int16))


@pytest.mark.parametrize("n_utts", [1, 5])
def test_all_codes_gemv_and_sensitivity(n_utts):
    """The GEMV over every code: within the bound of the exact values; a reference with the subnormal codes flushed, one
    with each row's scale taken from its neighbour and one with a slot's two CFG rows swapped each violate it."""
    codes, nan = _all_codes_matrix()
    codes = torch.where(nan, torch.zeros_like(codes), codes)        # the quantiser never emits NaN codes
    M, K = codes.shape
    q = codes.view(torch.float8_e4m3fn)
    s = torch.exp2(torch.randint(-12, -4, (M,), generator=torch.Generator().manual_seed(1)).float()).to(torch.bfloat16)
    Wp = Q.pack_fp8_matrix(q, s).cuda()
    qd, sd = _code_values(codes).cuda(), s.double().cuda()
    slots = SLOTS[n_utts]
    rows = _rows(slots)
    x, _ = _x(2 * max(slots) + 5, K, 3 + n_utts, False)
    v = x.double()[rows]
    ref, bound = _scaled(v, qd, sd, gamma(K, False))
    out = _call(STORE, Wp, M, K, x, slots)[rows, :M]
    _assess(f"all codes utts={n_utts}", out, ref, bound)
    sub = ((codes & 0x78) == 0) & ((codes & 0x07) != 0)
    flushed = (v @ torch.where(sub.cuda(), torch.zeros_like(qd), qd).t()) * sd
    assert _violations(out, flushed, bound) > 0, "a flushed-subnormal reference passes the bound"
    wrong_scale = (v @ qd.t()) * torch.roll(sd, 1)
    assert _violations(out, wrong_scale, bound) > 0, "a wrong row scale passes the bound"
    swapped = v.clone()
    swapped[0], swapped[1] = v[1], v[0]
    assert _violations(out, (swapped @ qd.t()) * sd, bound) > 0, "a swapped CFG row passes the bound"
