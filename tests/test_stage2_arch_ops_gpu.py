"""GPU: the stage-2 prologues and epilogues of the weight-streaming GEMM (csrc/tc_gemm.cuh) -- the LayerNorm mode of
k_prep_b (with and without beta), the Linear-bias epilogues (store, residual, SwiGLU) and GELU -- at production widths
(E = 384, hidden 1536 / 1024, M = 3 E, vocab 1025), R in {1, 17, 128}, with the automatic K split and a forced one,
through mvb_s2_linear_test, against float64 on the same bf16 operands.

Reference.  v = the prologue of x in float64 (RMSNorm x rsqrt(mean x^2 + eps) g; LayerNorm (x - mean) rsqrt(var + eps) g
(+ beta) with the biased variance), y = v . W^T (+ b) in float64, then the epilogue in float64.

Elementwise bound on the pre-activation y, with A = |v| . |W|^T:
    |y - y_ref| <= (gamma_K + TAU) A + 2 u (|y_ref| + |b|)
gamma_K = (18 * 4 * (K / 64) * 2 + ksplit) u is the accumulation bound derived in test_gemm_ops_gpu.py (hi + lo terms,
split-K partials summed in a fixed order).  TAU = 2^-15 covers the operand the kernel multiplies: hi + lo represents the
fp32 prologue value to 2^-16 relative, and the fp32 statistics (mean, variance or sum of squares over K <= 1536, then
rsqrtf) move it by a few 1e-7 relative on these inputs.  The bias adds one fp32 rounding (the 2 u term).  Epilogues:
    store     |y|-bound as is;  residual + 2 u |out|;
    GELU      1.13 x (|gelu'| <= 1.13) + 4 u (|out| + |y|)  (erff within 2 ulp);
    SwiGLU    1.1 E1 |y3| + (|silu(y1)| + 1.1 E1) E3 + 4 u |out|  (|silu'| <= 1.1).
Normwise: ||out - ref||_F / ||ref||_F < NORMWISE = 2e-5 (observed errors are ~1e-6; a dropped lo term gives ~1.7e-3).

Sensitivity: a missing beta, a bias added once per K split instead of once, and the tanh GELU in place of the erf one
must each violate the bounds.  Every call writes into a NaN-filled output with ldo > M and spare rows: only
[0, R) x [0, M) may change and nothing inside it may stay NaN."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
TAU = 2.0 ** -15
NORMWISE = 2e-5
EPS = 1e-5
G_STORE, G_RESID, G_SWIGLU, G_GELU = 0, 1, 2, 4
N_NONE, N_RMS, N_LAYER = 0, 1, 2
E, VOCAB = 384, 1025
KSPLIT_FORCED = 3

# (id, epilogue, M, K, norm, beta, bias): every stage-2 Linear of every architecture
CASES = [
    ("qkv-rms", G_STORE, 3 * E, E, N_RMS, False, False),
    ("qkv-rms-bias", G_STORE, 3 * E, E, N_RMS, False, True),
    ("qkv-ln-beta-bias", G_STORE, 3 * E, E, N_LAYER, True, True),
    ("qkv-ln-nobeta", G_STORE, 3 * E, E, N_LAYER, False, False),
    ("attn_proj-bias", G_RESID, E, E, N_NONE, False, True),
    ("c_fc-gelu-ln-beta-bias", G_GELU, 4 * E, E, N_LAYER, True, True),
    ("c_fc-gelu-ln-nobeta", G_GELU, 4 * E, E, N_LAYER, False, False),
    ("c_fc-gelu-rms-bias", G_GELU, 4 * E, E, N_RMS, False, True),
    ("w1w3-swiglu-rms-bias", G_SWIGLU, 1024, E, N_RMS, False, True),
    ("w1w3-swiglu-ln-beta-bias", G_SWIGLU, 1024, E, N_LAYER, True, True),
    ("mlp_proj-gelu-bias", G_RESID, E, 4 * E, N_NONE, False, True),
    ("mlp_proj-swiglu-bias", G_RESID, E, 1024, N_NONE, False, True),
    ("head-ln-beta", G_STORE, VOCAB, E, N_LAYER, True, False),
]


def _lib():
    from mvb200 import _lib as L
    return L, L.load()


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ksplit_bound(M, K, ksplit):
    return 16 if ksplit <= 0 else max(1, min(ksplit, _n_sm() // ((M + 127) // 128)))


def _inputs(M, K, R, seed, swiglu, norm, beta, bias):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda")   # noqa: E731
    bf = lambda t: t.to(torch.bfloat16)                             # noqa: E731
    t = dict(W=bf(rn(M, K) * 0.05), x=rn(R, K) + 0.3)              # a non-zero row mean: LayerNorm's centring matters
    t["W3"] = bf(rn(M, K) * 0.05) if swiglu else None
    t["gw"] = bf(1 + 0.1 * rn(K)) if norm != N_NONE else None
    t["beta"] = bf(0.1 * rn(K)) if beta else None
    t["b"] = bf(0.02 * rn(M)) if bias else None
    t["b3"] = bf(0.02 * rn(M)) if bias and swiglu else None
    t["out0"] = rn(R, M)
    return t


def _call(epi, norm, t, R, M, K, ksplit, ldo_pad=5, spare_rows=3):
    L, lib = _lib()
    ldo = M + ldo_pad
    out = torch.full((R + spare_rows, ldo), float("nan"), device="cuda")
    if epi == G_RESID:
        out[:R, :M] = t["out0"]
    ptr = lambda v: None if v is None else v.data_ptr()   # noqa: E731
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    L.check(lib.mvb_s2_linear_test(epi, norm, t["W"].data_ptr(), ptr(t["W3"]), ptr(t["b"]), ptr(t["b3"]), M, K, t["x"].data_ptr(),
                                   K, R, ptr(t["gw"]), ptr(t["beta"]), EPS, 1, ksplit, out.data_ptr(), ldo, st))
    torch.cuda.synchronize()
    return out


def _check_footprint(out, R, M):
    assert not torch.isnan(out[:R, :M]).any(), "elements of [0, R) x [0, M) were not written"
    mask = torch.ones_like(out, dtype=torch.bool)
    mask[:R, :M] = False
    assert torch.isnan(out[mask]).all(), "the kernel wrote outside [0, R) x [0, M)"


def _prologue(x, norm, gw, beta):
    x = x.double()
    if norm == N_RMS:
        return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + EPS) * gw.double()
    if norm == N_LAYER:
        c = x - x.mean(-1, keepdim=True)
        v = c * torch.rsqrt(c.pow(2).mean(-1, keepdim=True) + EPS) * gw.double()
        return v if beta is None else v + beta.double()
    return x


def _reference(epi, norm, t, gamma, *, beta=True, bias_times=1, gelu="none"):
    """(ref, elementwise bound) in float64.  beta=False drops the LayerNorm beta, bias_times scales the Linear biases and
    gelu selects F.gelu's approximation: the sensitivity cases."""
    v = _prologue(t["x"], norm, t["gw"], t["beta"] if beta else None)
    av = v.abs()

    def lin(W, b):
        y = v @ W.double().t()
        bd = torch.zeros(W.shape[0], dtype=torch.float64, device=y.device) if b is None else b.double() * bias_times
        y = y + bd
        err = (gamma + TAU) * (av @ W.double().abs().t()) + 2 * U * (y.abs() + bd.abs())
        return y, err

    y, ey = lin(t["W"], t["b"])
    if epi == G_STORE:
        return y, ey
    if epi == G_RESID:
        ref = t["out0"].double() + y
        return ref, ey + 2 * U * ref.abs()
    if epi == G_GELU:
        ref = F.gelu(y, approximate=gelu)
        return ref, 1.13 * ey + 4 * U * (ref.abs() + y.abs())
    y3, e3 = lin(t["W3"], t["b3"])
    s = F.silu(y)
    ref = s * y3
    return ref, 1.1 * ey * y3.abs() + (s.abs() + 1.1 * ey) * e3 + 4 * U * ref.abs()


def _assess(got, ref, bound):
    err = (got.double() - ref).abs()
    ratio = float((err / (bound + 1e-30)).max())
    normwise = float(err.norm() / ref.norm())
    return ratio, normwise


def _run(case, R, ksplit, seed=0):
    _, epi, M, K, norm, beta, bias = case
    t = _inputs(M, K, R, seed, epi == G_SWIGLU, norm, beta, bias)
    out = _call(epi, norm, t, R, M, K, ksplit)
    _check_footprint(out, R, M)
    ks = _ksplit_bound(M, K, ksplit)
    gamma = (18 * 4 * (K // 64) * 2 + ks) * U
    return t, out[:R, :M], gamma


@pytest.mark.parametrize("ksplit", [0, KSPLIT_FORCED], ids=["auto_split", "forced_split"])
@pytest.mark.parametrize("R", [1, 17, 128])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_stage2_linear_vs_float64(case, R, ksplit):
    t, got, gamma = _run(case, R, ksplit, seed=R)
    ref, bound = _reference(case[1], case[4], t, gamma)
    ratio, normwise = _assess(got, ref, bound)
    print(f"{case[0]} R={R} ksplit={ksplit}: worst err / bound {ratio:.3f}, normwise {normwise:.2e}")
    assert ratio <= 1.0, f"elementwise bound exceeded x{ratio:.2f}"
    assert normwise < NORMWISE


def _case(name):
    return next(c for c in CASES if c[0] == name)


def test_missing_beta_violates_the_bound():
    case = _case("qkv-ln-beta-bias")
    t, got, gamma = _run(case, 17, KSPLIT_FORCED)
    ok = _assess(got, *_reference(case[1], case[4], t, gamma))
    bad = _assess(got, *_reference(case[1], case[4], t, gamma, beta=False))
    print(f"LayerNorm beta: with {ok}, dropped {bad}")
    assert ok[0] <= 1.0 and bad[0] > 1.0 and bad[1] > NORMWISE


@pytest.mark.parametrize("name", ["qkv-rms-bias", "attn_proj-bias", "w1w3-swiglu-rms-bias", "c_fc-gelu-rms-bias"])
def test_bias_added_per_split_violates_the_bound(name):
    """With the K split forced to 3, a bias added by every split (3 b) instead of once after the reduction is caught."""
    case = _case(name)
    t, got, gamma = _run(case, 17, KSPLIT_FORCED)
    ks = _ksplit_bound(case[2], case[3], KSPLIT_FORCED)
    assert ks == KSPLIT_FORCED
    ok = _assess(got, *_reference(case[1], case[4], t, gamma))
    bad = _assess(got, *_reference(case[1], case[4], t, gamma, bias_times=ks))
    print(f"{name}: bias once {ok}, once per split {bad}")
    assert ok[0] <= 1.0 and bad[0] > 1.0 and bad[1] > NORMWISE


def test_tanh_gelu_violates_the_bound():
    """The tanh approximation differs from the exact erf GELU by up to ~5e-4 at |y| ~ 2: above the normwise bound."""
    case = _case("c_fc-gelu-ln-beta-bias")
    t, got, gamma = _run(case, 128, 0)
    ok = _assess(got, *_reference(case[1], case[4], t, gamma))
    bad = _assess(got, *_reference(case[1], case[4], t, gamma, gelu="tanh"))
    print(f"GELU: erf {ok}, tanh {bad}")
    assert ok[0] <= 1.0 and ok[1] < NORMWISE and bad[1] > NORMWISE


def test_hook_rejects_bad_arguments():
    L, lib = _lib()
    M, K, R = 128, 128, 4
    W = torch.zeros(M, K, dtype=torch.bfloat16, device="cuda")
    x = torch.zeros(R, K, device="cuda")
    out = torch.zeros(R, M, device="cuda")
    g = torch.ones(K, dtype=torch.bfloat16, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = lambda epi, norm, gain, beta, W3=None, b=None, b3=None: (epi, norm, W.data_ptr(), W3, b, b3, M, K, x.data_ptr(), K, R,  # noqa: E731
                                                                   gain, beta, EPS, 1, 0, out.data_ptr(), M, st)
    for a, what in ((args(3, 0, None, None), "epilogue"), (args(0, 3, None, None), "norm"), (args(0, 1, None, None), "gain"),
                    (args(0, 1, g.data_ptr(), g.data_ptr()), "beta"), (args(G_SWIGLU, 0, None, None), "W3"),
                    (args(G_SWIGLU, 0, None, None, W.data_ptr(), g.data_ptr()), "bias3")):
        assert lib.mvb_s2_linear_test(*a) == L.MVB_ERR_ARG, what
    assert math.isfinite(float(out.sum()))
