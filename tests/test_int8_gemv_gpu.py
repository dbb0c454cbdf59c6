"""GPU: the int8 GEMV (csrc/gemv_w8.cuh, k_gemv_w8<EPI>) at every epilogue and production (M, K), lm_head and the tiny model's
shapes; the int8 widening (k_w8_widen); and the row-scale epilogue of the tensor-core GEMM (k_tc_gemm<EPI, NC, true>), against
float64 computations over the host's (q, s) (mvb200/quantize.py).

Reference.  q (int8) and s (bf16) are exact data.  The activation row is v = x, or with the RMSNorm prologue
v = (x * rs) * gain in fp32 with rs = rsqrt(fl(sum x^2) / K + eps); then ref_j = s_j (v . q_j) in float64, followed by the
epilogue in float64.

Elementwise bound (GEMV).  With A_j = s_j (|v| . |q_j|) every element must satisfy |out - ref| <= gamma * A + u |ref'| + tiny.
Derivation for this kernel's order of accumulation: K is cut into NT = ceil(K / 512) tiles; in each tile lane j sums, with one
fp32 fma each, the products of its 16 k, tile after tile: at most n1 = 16 NT roundings of a sum whose magnitudes are bounded
by sum |v_k q_k| (the int8 -> fp32 conversion is exact); a 5-level butterfly then adds the 32 lane sums.  So the sum carries
at most n = n1 + 5 roundings, |err| <= gamma_n sum |v_k q_k| with gamma_n = n u / (1 - n u), u = 2^-24; the test uses
gamma = n 2^-23 >= gamma_n.  The scale is exact bf16 and multiplies the rounded sum once: one more rounding, at most
2^-24 relative to the product (the test adds 2^-23 (|ref| + bound)).  The RMSNorm prologue adds tau = 2^-22 relative to |v|.
Epilogues add their own fp32 roundings (bounds below).

Normwise bound.  ||out - ref||_F / ||ref||_F < 1e-4.

Sensitivity.  References built with q read as unsigned, with the w1 and w3 scales swapped, with the fp32 scale s32 instead
of the stored bf16 s, and with each row's scale taken from the neighbouring row must violate the bounds.  Every call writes
into NaN-filled outputs with ldo > M and rows no utterance owns: only the rows of the utterances' slots x [0, M) may change
and none of them may stay NaN.

Tensor-core GEMM with row scales: the bound of tests/test_gemm_ops_gpu.py (gamma_K over the widened q, hi + lo activations)
scaled by s_j, plus the one rounding of the scale multiply, at ksplit 1 and above 1."""
import ctypes as C
import functools

import pytest
import torch

from mvb200 import quantize as Q

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
NORMWISE = 1e-4
TAU_GAIN = 2.0 ** -22
EPS = 1e-5
STORE, RESID, SWIGLU, QKV = 0, 1, 2, 3
SLOTS = {1: [2], 3: [4, 0, 2], 8: [3, 7, 0, 9, 4, 1, 8, 5]}   # utterance -> slot (rows 2 s, 2 s + 1); not the identity


def _lib():
    from mvb200 import _lib as L
    return L, L.load()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def gamma(K):
    return (16 * ((K + 511) // 512) + 5) * U


@functools.lru_cache(maxsize=None)
def _mat(M, K, seed):
    """(int8 matrix on the device, q float64 [M, K] and s float64 [M] on the device, (q, s) on the host)"""
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(M, K, generator=g) * 0.03).to(torch.bfloat16)
    q, s = Q.quantize_per_channel(w)
    return Q.pack_int8_matrix(q, s).cuda(), q.double().cuda(), s.double().cuda(), (q, s, w)


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


def _rows(n_utts):
    return sorted(r for s in SLOTS[n_utts] for r in (2 * s, 2 * s + 1))


def _call(epi, Wp, M, K, x, n_utts, *, W3p=None, gw=None, out0=None, kv=None, ldo_pad=5, spare_rows=3):
    L, lib = _lib()
    slots = SLOTS[n_utts]
    n_rows = 2 * max(slots) + 2 + spare_rows
    out = torch.full((n_rows, M + ldo_pad), float("nan"), device="cuda")
    if out0 is not None:
        r = _rows(n_utts)
        out[r, :M] = out0[r]
    slot_map = torch.tensor(slots, dtype=torch.int32, device="cuda")
    kc = vc = pos = None
    H = S_max = D = kv_fp32 = 0
    if kv is not None:
        kc, vc, pos, H, S_max, D, kv_fp32 = kv
    if pos is None:
        pos = torch.zeros(max(slots) + 1, dtype=torch.int32, device="cuda")
    ptr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    L.check(lib.mvb_w8_gemv_test(epi, Wp.data_ptr(), ptr(W3p), M, K, x.data_ptr(), x.shape[1], n_utts, ptr(gw), EPS,
                                 out.data_ptr(), M + ldo_pad, ptr(kc), ptr(vc), slot_map.data_ptr(), pos.data_ptr(), H, S_max,
                                 D, kv_fp32, _stream()))
    return out


def _check_footprint(out, rows, M):
    assert not torch.isnan(out[rows, :M]).any(), "elements of the utterances' rows x [0, M) were not written"
    mask = torch.ones_like(out, dtype=torch.bool)
    for r in rows:
        mask[r, :M] = False
    assert torch.isnan(out[mask]).all(), "the kernel wrote outside the utterances' rows x [0, M)"


def _assess(label, got, ref, bound):
    err = (got.double() - ref).abs()
    ratio = float((err / bound).max())
    nw = float(err.norm() / ref.norm())
    print(f"{label}: max |err|/bound {ratio:.2e}, normwise {nw:.2e}")
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


# (epilogue, M, K): every int8 matrix of MetaVoice-1B under the epilogue the engine gives it (lm_head: STORE with the ln_f
# prologue), the STORE epilogue at each production shape, and the tiny model's shapes (K = 256 is one trailing 256-wide
# tile, K = 768 a full and a trailing one).
CASES = [(QKV, 6144, 2048), (RESID, 2048, 2048), (SWIGLU, 5632, 2048), (RESID, 2048, 5632), (STORE, 2562, 2048),
         (STORE, 6144, 2048), (STORE, 5632, 2048), (STORE, 2048, 5632),
         (QKV, 768, 256), (RESID, 256, 256), (SWIGLU, 768, 256), (RESID, 256, 768), (STORE, 256, 768), (STORE, 2562, 256)]


@pytest.mark.parametrize("gain", [False, True], ids=["plain", "rmsnorm"])
@pytest.mark.parametrize("n_utts", [1, 3, 8])
@pytest.mark.parametrize("epi,M,K", CASES)
def test_gemv_w8(epi, M, K, n_utts, gain):
    Wp, qd, sd, _ = _mat(M, K, 1000 * M + K)
    rows = _rows(n_utts)
    x, gw = _x(2 * max(SLOTS[n_utts]) + 2, K, M + K + n_utts, gain)
    v = _v(x, gw)[rows]
    gam = gamma(K) + (TAU_GAIN if gain else 0.0)
    label = f"epi={epi} M={M} K={K} utts={n_utts} gain={int(gain)} [gamma={gam:.2e}]"
    if epi == SWIGLU:
        W3p, q3d, s3d, _ = _mat(M, K, 1000 * M + K + 1)
        (y, b1), (y3, b3) = _scaled(v, qd, sd, gam), _scaled(v, q3d, s3d, gam)
        ref = y * torch.sigmoid(y) * y3
        out = _call(SWIGLU, Wp, M, K, x, n_utts, W3p=W3p, gw=gw)
        _check_footprint(out, rows, M)
        _assess(label, out[rows, :M], ref, _swiglu_bound(y, y3, b1, b3, ref))
        return
    ref, bound = _scaled(v, qd, sd, gam)
    out0 = kv = None
    if epi == RESID:
        out0 = torch.randn(2 * max(SLOTS[n_utts]) + 2, M, generator=torch.Generator(device="cuda").manual_seed(K), device="cuda")
        ref = ref + out0[rows].double()
        bound = bound + U * (ref.abs() + bound)          # the fp32 add of the residual epilogue
    if epi == QKV:
        D = M // 3
        H, S_max = D // 128, 37
        n_cache_rows = 2 * max(SLOTS[n_utts]) + 2
        pos = torch.randint(0, S_max, (max(SLOTS[n_utts]) + 1,), generator=torch.Generator().manual_seed(M), dtype=torch.int32)
        pos[SLOTS[n_utts][0]] = S_max - 1
        kv_fp32 = int(n_utts != 3)                        # both cache types
        dt = torch.float32 if kv_fp32 else torch.bfloat16
        kc = torch.full((n_cache_rows, H, S_max, 128), float("nan"), dtype=dt, device="cuda")
        vc = torch.full_like(kc, float("nan"))
        kv = (kc, vc, pos.cuda(), H, S_max, D, kv_fp32)
    out = _call(epi, Wp, M, K, x, n_utts, gw=gw, out0=out0, kv=kv)
    _check_footprint(out, rows, M)
    _assess(label, out[rows, :M], ref, bound)
    if epi == QKV:
        view = torch.int32 if kv_fp32 else torch.int16
        written = torch.zeros(n_cache_rows, S_max, dtype=torch.bool, device="cuda")
        for s in SLOTS[n_utts]:
            p = int(pos[s])
            for r in (2 * s, 2 * s + 1):
                want_k = out[r, D:2 * D].reshape(H, 128).to(dt)
                want_v = out[r, 2 * D:3 * D].reshape(H, 128).to(dt)
                assert torch.equal(kc[r, :, p].view(view), want_k.view(view)), "K cache differs from the kernel's output"
                assert torch.equal(vc[r, :, p].view(view), want_v.view(view)), "V cache differs from the kernel's output"
                written[r, p] = True
        for cache in (kc, vc):
            assert torch.isnan(cache.permute(0, 2, 1, 3)[~written].float()).all(), "cache entries outside the scatter changed"


@pytest.mark.parametrize("M,K", [(6144, 2048), (2048, 2048), (5632, 2048), (2048, 5632), (2562, 2048), (768, 256), (256, 768)])
def test_widen_bit_identical_to_host(M, K):
    L, lib = _lib()
    Wp, _, _, (q, s, _) = _mat(M, K, 1000 * M + K)
    out = torch.full((M, K), float("nan"), dtype=torch.bfloat16, device="cuda")
    L.check(lib.mvb_w8_widen_test(Wp.data_ptr(), M, K, out.data_ptr(), _stream()))
    assert torch.equal(out.cpu().view(torch.int16), q.to(torch.bfloat16).view(torch.int16))


def _violates(label, got, ref, bound):
    err = (got - ref).abs()
    n_over, nw = int((err > bound).sum()), float(err.norm() / ref.norm())
    print(f"{label}: {n_over} of {err.numel()} elements over the bound, normwise {nw:.2e}")
    assert n_over > err.numel() // 10 and nw > NORMWISE, label


def test_wrong_references_violate_the_bound():
    M, K, n_utts = 2048, 2048, 3
    Wp, qd, sd, (q, s, w) = _mat(M, K, 77)
    rows = _rows(n_utts)
    x, _ = _x(2 * max(SLOTS[n_utts]) + 2, K, 5, False)
    v = x.double()[rows]
    out = _call(STORE, Wp, M, K, x, n_utts)[rows, :M].double()
    wf = w.float()
    s32 = torch.clamp(torch.maximum(-wf.amin(1).clamp(max=0), wf.amax(1).clamp(min=0)) / 127.5,
                      min=torch.finfo(torch.float32).eps).double().cuda()
    wrong = {"q read as unsigned": (q.to(torch.uint8).double().cuda(), sd),
             "fp32 scale s32": (qd, s32),
             "neighbouring row's scale": (qd, torch.roll(sd, 1))}
    for name, (qw, sw) in wrong.items():
        ref, bound = _scaled(v, qw, sw, gamma(K))
        _violates(name, out, ref, bound)
    # SwiGLU with the w1 and w3 scales swapped
    M = 5632
    Wp, qd, sd, _ = _mat(M, K, 78)
    W3p, q3d, s3d, _ = _mat(M, K, 79)
    out = _call(SWIGLU, Wp, M, K, x, n_utts, W3p=W3p)[rows, :M].double()
    (y, b1), (y3, b3) = _scaled(v, qd, s3d, gamma(K)), _scaled(v, q3d, sd, gamma(K))
    ref = y * torch.sigmoid(y) * y3
    _violates("w1 / w3 scales swapped", out, ref, _swiglu_bound(y, y3, b1, b3, ref))


# ---- k_tc_gemm<EPI, NC, true>: the prefill GEMM over the widened q with the row-scale epilogue -------------------------
def _gemm(epi, qb, sb, x, R, M, K, *, q3b=None, s3b=None, ksplit=0, out0=None, kv=None):
    L, lib = _lib()
    ldo = M + 3
    out = torch.full((R + 2, ldo), float("nan"), device="cuda")
    if out0 is not None:
        out[:R, :M] = out0
    kc = vc = rc = rp = None
    H = S_max = D = kv_fp32 = 0
    if kv is not None:
        kc, vc, rc, rp, H, S_max, D, kv_fp32 = kv
    ptr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    L.check(lib.mvb_w8_gemm_test(epi, qb.data_ptr(), ptr(q3b), sb.data_ptr(), ptr(s3b), M, K, x.data_ptr(), K, R, None, EPS,
                                 1, ksplit, out.data_ptr(), ldo, ptr(kc), ptr(vc), ptr(rc), ptr(rp), H, S_max, D, kv_fp32,
                                 _stream()))
    torch.cuda.synchronize()
    assert not torch.isnan(out[:R, :M]).any() and torch.isnan(out[R:]).all() and torch.isnan(out[:, M:]).all()
    return out[:R, :M]


def _xhat(x):
    hi = x.to(torch.bfloat16).float()
    lo = (x - hi).to(torch.bfloat16).float()
    return hi.double() + lo.double()


@pytest.mark.parametrize("ksplit", [1, 4])
@pytest.mark.parametrize("epi,M,K,R", [(STORE, 2562, 2048, 2), (RESID, 2048, 5632, 40), (SWIGLU, 5632, 2048, 128),
                                       (QKV, 6144, 2048, 24), (STORE, 768, 256, 16)])
def test_tc_gemm_row_scales(epi, M, K, R, ksplit):
    _, qd, sd, (q, s, _) = _mat(M, K, 3 * M + K)
    qb, sb = q.to(torch.bfloat16).cuda(), s.cuda()
    x = torch.randn(R, K, generator=torch.Generator(device="cuda").manual_seed(R + M), device="cuda")
    xh = _xhat(x)
    gam = (18 * 4 * (K // 64) * 2 + 16) * U
    ref, bound = _scaled(xh, qd, sd, gam)
    label = f"tc epi={epi} M={M} K={K} R={R} ksplit={ksplit}"
    if epi == SWIGLU:
        _, q3d, s3d, (q3, s3, _) = _mat(M, K, 3 * M + K + 1)
        y3, b3 = _scaled(xh, q3d, s3d, gam)
        y, b1 = ref, bound
        ref = y * torch.sigmoid(y) * y3
        out = _gemm(SWIGLU, qb, sb, x, R, M, K, q3b=q3.to(torch.bfloat16).cuda(), s3b=s3.cuda(), ksplit=ksplit)
        _assess(label, out, ref, _swiglu_bound(y, y3, b1, b3, ref))
        return
    out0 = kv = None
    if epi == RESID:
        out0 = torch.randn(R, M, generator=torch.Generator(device="cuda").manual_seed(K), device="cuda")
        ref = ref + out0.double()
        bound = bound + U * (ref.abs() + bound)
    if epi == QKV:
        D, S_max = M // 3, 9
        H = D // 128
        kc = torch.full((R, H, S_max, 128), float("nan"), device="cuda")
        vc = torch.full_like(kc, float("nan"))
        rc = torch.arange(R, dtype=torch.int32, device="cuda")
        rp = torch.randint(0, S_max, (R,), generator=torch.Generator().manual_seed(R), dtype=torch.int32).cuda()
        kv = (kc, vc, rc, rp, H, S_max, D, 1)
    out = _gemm(epi, qb, sb, x, R, M, K, ksplit=ksplit, out0=out0, kv=kv)
    _assess(label, out, ref, bound)
    if epi == QKV:
        for n in range(R):
            p = int(rp[n])
            assert torch.equal(kc[n, :, p], out[n, D:2 * D].reshape(H, 128))
            assert torch.equal(vc[n, :, p], out[n, 2 * D:].reshape(H, 128))
