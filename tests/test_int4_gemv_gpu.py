"""GPU: the int4 GEMV (csrc/gemv_w4.cuh, k_gemv_w4<EPI>) at every epilogue and production (M, K), and the int4 dequantiser
(k_w4_dequant), against float64 computations over the host's W_deq (mvb200/quantize.py).

Reference.  W_deq = bf16_rn((q - 8) s + z) is exact data (the kernel computes the same bf16 values; k_w4_dequant is
checked bit for bit against the host).  The activation row is v = x, or with the RMSNorm prologue v = (x * rs) * gain in
fp32 with rs = rsqrt(fl(sum x^2) / K + eps); then ref = v . W_deq^T in float64, followed by the epilogue in float64.

Elementwise bound.  With A = |v| . |W_deq|^T every element must satisfy |out - ref| <= gamma * A + tiny.  Derivation for this
kernel's order of accumulation: K is cut into NT = ceil(K / 512) tiles dealt alternately to the two half-warps of the
warp that owns the output; each lane sums, with one fp32 fma each, the products of its 32 k of each of its tiles, in k
order: at most n1 = 32 ceil(NT / 2) roundings; a 5-level butterfly then adds the 32 lane sums.  Every output therefore
carries at most n = n1 + 5 roundings on any path, and
the standard bound |err| <= gamma_n sum |v_k w_k| holds with gamma_n = n u / (1 - n u), u = 2^-24.  The test uses
gamma = n 2^-23 >= gamma_n.  The RMSNorm prologue adds tau = 2^-22 relative to |v| (rsqrtf within 2 ulp; the test inputs
make the sum of squares exact in any order).  Epilogues add their own fp32 roundings (bounds below).

Normwise bound.  ||out - ref||_F / ||ref||_F < 1e-4.

Sensitivity.  References built from swapped nibbles, from scale and zero swapped, or with offset 7 instead of 8 must
violate the bounds.  Every call writes into NaN-filled outputs with ldo > M and rows no utterance owns: only the rows of
the utterances' slots x [0, M) may change and none of them may stay NaN."""
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


def gamma(K):
    NT = (K + 511) // 512
    return (32 * ((NT + 1) // 2) + 5) * U


@functools.lru_cache(maxsize=None)
def _packed(M, K, seed):
    """(packed matrix on the device, W_deq float64 on the device, (q, s, z) on the host)"""
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(M, K, generator=g) * 0.03).to(torch.bfloat16)
    q, s, z = Q.group_quantize(w)
    return Q.pack_matrix(q, s, z).cuda(), Q.dequantize(q, s, z).cuda().double(), (q, s, z)


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


def _call(epi, Wp, M, K, x, n_utts, *, W3p=None, gw=None, out0=None, kv=None, ldo_pad=5, spare_rows=3):
    L, lib = _lib()
    slots = SLOTS[n_utts]
    n_rows = 2 * max(slots) + 2 + spare_rows
    ldo = M + ldo_pad
    out = torch.full((n_rows, ldo), float("nan"), device="cuda")
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
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ptr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    L.check(lib.mvb_w4_gemv_test(epi, Wp.data_ptr(), ptr(W3p), M, K, x.data_ptr(), x.shape[1], n_utts, ptr(gw), EPS,
                                 out.data_ptr(), ldo, ptr(kc), ptr(vc), slot_map.data_ptr(), pos.data_ptr(), H, S_max, D,
                                 kv_fp32, st))
    return out


def _rows(n_utts):
    return sorted(r for s in SLOTS[n_utts] for r in (2 * s, 2 * s + 1))


def _check_footprint(out, rows, M):
    inside = out[rows, :M]
    assert not torch.isnan(inside).any(), "elements of the utterances' rows x [0, M) were not written"
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


# (epilogue, M, K): every int4 matrix of MetaVoice-1B under the epilogue the engine gives it, the STORE epilogue at each
# production shape, and the tiny model's shapes (K = 768 exercises the trailing 256-wide tile).
CASES = [(QKV, 6144, 2048), (RESID, 2048, 2048), (SWIGLU, 5632, 2048), (RESID, 2048, 5632),
         (STORE, 6144, 2048), (STORE, 5632, 2048), (STORE, 2048, 5632),
         (QKV, 768, 256), (RESID, 256, 256), (SWIGLU, 768, 256), (RESID, 256, 768), (STORE, 256, 768)]


@pytest.mark.parametrize("gain", [False, True], ids=["plain", "rmsnorm"])
@pytest.mark.parametrize("n_utts", [1, 3, 8])
@pytest.mark.parametrize("epi,M,K", CASES)
def test_gemv_w4(epi, M, K, n_utts, gain):
    Wp, Wd, _ = _packed(M, K, 1000 * M + K)
    rows = _rows(n_utts)
    x, gw = _x(2 * max(SLOTS[n_utts]) + 2, K, M + K + n_utts, gain)
    v = _v(x, gw)
    gam = gamma(K) + (TAU_GAIN if gain else 0.0)
    label = f"epi={epi} M={M} K={K} utts={n_utts} gain={int(gain)} [gamma={gam:.2e}]"
    if epi == SWIGLU:
        W3p, W3d, _ = _packed(M, K, 1000 * M + K + 1)
        y, y3 = v[rows] @ Wd.t(), v[rows] @ W3d.t()
        ref = y * torch.sigmoid(y) * y3
        b1, b3 = gam * (v[rows].abs() @ Wd.abs().t()), gam * (v[rows].abs() @ W3d.abs().t())
        out = _call(SWIGLU, Wp, M, K, x, n_utts, W3p=W3p, gw=gw)
        _check_footprint(out, rows, M)
        _assess(label, out[rows, :M], ref, _swiglu_bound(y, y3, b1, b3, ref))
        return
    y = v[rows] @ Wd.t()
    bound = gam * (v[rows].abs() @ Wd.abs().t()) + 1e-30
    out0 = ref = None
    kv = None
    if epi == RESID:
        out0 = torch.randn(2 * max(SLOTS[n_utts]) + 2, M, generator=torch.Generator(device="cuda").manual_seed(K), device="cuda")
        ref = y + out0[rows].double()
        bound = bound + U * (ref.abs() + bound)          # the fp32 add of the residual epilogue
    else:
        ref = y
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


@pytest.mark.parametrize("M,K", [(6144, 2048), (2048, 2048), (5632, 2048), (2048, 5632), (768, 256), (256, 768), (2048, 256)])
def test_dequant_bit_identical_to_host(M, K):
    L, lib = _lib()
    Wp, Wd, (q, s, z) = _packed(M, K, 1000 * M + K)
    out = torch.full((M, K), float("nan"), dtype=torch.bfloat16, device="cuda")
    L.check(lib.mvb_w4_dequant_test(Wp.data_ptr(), M, K, out.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    want = Q.dequantize(q, s, z)
    assert torch.equal(out.cpu().view(torch.int16), want.view(torch.int16))


def _wrong_refs(q, s, z):
    """W_deq under three wrong readings of the packed matrix."""
    M, K = q.shape
    swapped = q.clone()
    swapped[:, 0::2], swapped[:, 1::2] = q[:, 1::2], q[:, 0::2]
    off7 = (q.double().reshape(M, K // 128, 128) - 7) * s.double()[..., None] + z.double()[..., None]
    return {"swapped nibbles": Q.dequantize(swapped, s, z).double(),
            "scale / zero swapped": Q.dequantize(q, z, s).double(),
            "offset 7": off7.reshape(M, K)}


def test_wrong_references_violate_the_bound():
    M, K, n_utts = 2048, 2048, 3
    Wp, Wd, (q, s, z) = _packed(M, K, 77)
    rows = _rows(n_utts)
    x, _ = _x(2 * max(SLOTS[n_utts]) + 2, K, 5, False)
    out = _call(STORE, Wp, M, K, x, n_utts)[rows, :M].double()
    v = x.double()[rows]
    for name, Wwrong in _wrong_refs(q, s, z).items():
        Wwrong = Wwrong.cuda()
        ref = v @ Wwrong.t()
        bound = gamma(K) * (v.abs() @ Wwrong.abs().t())
        err = (out - ref).abs()
        n_over, nw = int((err > bound).sum()), float(err.norm() / ref.norm())
        print(f"{name}: {n_over} of {err.numel()} elements over the bound, normwise {nw:.2e}")
        assert n_over > err.numel() // 2 and nw > 10 * NORMWISE
