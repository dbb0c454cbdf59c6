"""GPU: the projections of the non-production stage-1 architectures (LayerNorm prologue, Linear biases, GELU epilogue) at
production width (K = 2048; MLP widths 5632 and 8192, the GELU c_proj at K = 8192) and at the tiny width, against float64,
through mvb_s1_arch_gemv_test: every new k_gemv instance as path A launches it (1 / 3 / 8 utterances on a non-identity
slot map) and the BIASED QKV k_tc_gemm of path B with a forced K split.

OPERAND (the fp32 values the kernels stage, computed in float64 from the exact fp32 / bf16 inputs): n = RMSNorm or
LayerNorm of x times the bf16 gain (+ beta), or x itself; the reference uses the exact statistics.

ELEMENTWISE BOUND, for y = W n + b and A = |W| |n| + |b| (u = 2^-23):
    |y^ - y| <= gamma A + S_j,
  gamma, path A (k_gemv) = (K / 32 + 5 + 4) u: one fma chain of K / 32 products per lane, a 5-step butterfly, the bias
    add, the residual add, and 2 u for the operand's own rounding (fl(fl(x rs) g) (+ beta));
  gamma, path B (k_tc_gemm, split_lo) = (18 * 4 * 2 * ceil(KB / S) + S + 4) u + 2^-16: the m16n8k16 model of
    test_gemm_ops_gpu.py over the ceil(KB / S) k-blocks of a split, the S partials' sum, the bias add, and the hi / lo
    split of the staged operand (its lo term is rounded to bf16: 2^-16 relative);
  S_j, the norm statistics, (derived for LayerNorm; RMSNorm is its special case with mean 0): with m^ the fp32 mean (a
    strided sum of K / 256 terms per thread, a 5-step butterfly, 8 warp partials, one division),
        |m^ - m| <= dm = (K / 256 + 14) u mean|x|;
    the centred values d^ = fl(x - m^) = d (1 + t) + (m - m^)(1 + t), |t| <= u, and because sum d = 0 exactly,
        sum d^2 (exact) = (1 + O(u)) sum d^2 + K (m - m^)^2,
    so the fp32 variance (the same strided sum) has relative error
        e_v <= (K / 256 + 14 + 3) u + dm^2 / var;
    rsqrtf adds 2 ulp and the eps add 1 u: e_rs <= e_v / 2 + 3 u.  Each staged n_k = fl(fl(d^_k rs^) g_k) then differs
    from the exact LayerNorm by <= rs |g_k| ((e_rs + u) |d_k| + (1 + u) dm), and
        S_j = sum_k |W_jk| rs |g_k| ((e_rs + u) |d_k| + 1.01 dm).
    A one-pass variance (E[x^2] - m^2 in fp32) loses the centred second moment to cancellation once |m| >> sigma.  The
    rows of utterance slot 5 (FAR_ROWS) are x = 256 + j / 16, j uniform in [-12, 12] (sigma ~ 0.45): every partial sum
    of the mean (K <= 2048 terms) is a multiple of 2^-4 below 2^20, exact in fp32, and so is the mean (a multiple of
    2^-15 near 256), so dm = 0 there; x^2 = 65536 + 32 j + j^2 / 256 needs 25 bits, and a one-pass fp32 variance is off
    by ~1 % of 0.2, which moves y by ~0.5 % of |y|, far above the bound.
EPILOGUES (e_y the bound above): residual adds its u |out|; SwiGLU h = silu(g) v, e_h = 1.1 e_g |v| + |silu(g)| e_v +
  1.1 e_g e_v + (8 + floor(1.17 |g|)) u |h| (__expf, the 1 + e add, the division, the product); GELU h = 0.5 y (1 +
  erf(y / sqrt 2)), |gelu'| <= 1.13: e_h = 1.13 e_y + 8 u (|h| + |y|) (erff 2 ulp, the products; tanh-GELU is off by up
  to 4.7e-4 near |y| = 2.7).  A bf16 cache stores fl_bf16(y^): + 2^-8 (|y| + e_y).
Every altered reference (one-pass variance, no beta, the bias added per K split, tanh GELU, k stored without its bias)
must put some entry outside the bound.  Outputs are NaN-filled with ldo > M: entries outside the written rows and columns
must stay NaN; cache entries must equal the kernel's own output (bf16-rounded for a bf16 cache), every other entry
untouched.
"""
import ctypes as C
import math

import pytest
import torch

from mvb200 import _lib

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
EPS_RMS, EPS_LN = 1e-5, 1e-5
SLOTS = 12                         # cache / activation rows: 2 per slot
S_MAX = 8
STORE, RESID, SWIGLU, QKV, GELU = 0, 1, 2, 3, 4
FAR_ROWS = [10, 11]                # the rows of slot 5


def _bf16(t):
    return t.to(torch.bfloat16)


def _rand(shape, std, g, mean=0.0):
    return (torch.randn(shape, generator=g, dtype=torch.float64) * std + mean)


class Case:
    def __init__(self, K, M, n_utts, norm, beta, bias, seed, epi):
        g = torch.Generator().manual_seed(seed)
        self.K, self.M, self.n_utts, self.norm, self.epi = K, M, n_utts, norm, epi
        self.slots = [11, 2, 7, 0, 9, 5, 3, 10][:n_utts]            # non-identity slot map; slot 5: FAR_ROWS
        x = _rand((2 * SLOTS, K), 1.0, g)
        x[10:12] = 256 + torch.randint(-12, 13, (2, K), generator=g).double() / 16      # rows of slot 5: see FAR_ROWS
        self.x = x.float()                                          # exact fp32 inputs
        self.W = _bf16(_rand((M, K), 1.0 / math.sqrt(K), g))
        self.W3 = _bf16(_rand((M, K), 1.0 / math.sqrt(K), g)) if epi == SWIGLU else None
        self.gain = _bf16(1.0 + 0.1 * _rand((K,), 1.0, g)) if norm else None
        self.beta = _bf16(_rand((K,), 0.3, g)) if beta else None
        self.bias = _bf16(_rand((M,), 0.5, g)) if bias else None
        self.bias3 = _bf16(_rand((M,), 0.5, g)) if bias and epi == SWIGLU else None
        self.pos = torch.randint(0, S_MAX, (SLOTS,), generator=g, dtype=torch.int32)

    def rows(self):
        """Activation / cache rows of the active slots, in utterance order: 2 s, 2 s + 1."""
        return [r for s in self.slots for r in (2 * s, 2 * s + 1)]

    # float64 operand with the exact statistics, its LayerNorm pieces, and the one-pass / beta-less alterations
    def operand(self, one_pass=False, drop_beta=False):
        x = self.x.double()
        if self.norm == 0:
            return x, None
        gn = self.gain.double()
        if self.norm == 1:
            rs = torch.rsqrt((x * x).mean(-1, keepdim=True) + EPS_RMS)
            return x * rs * gn, (x, rs, torch.zeros_like(rs))
        m = x.mean(-1, keepdim=True)
        d = x - m
        if one_pass:    # E[x^2] - m^2 in fp32
            xf = self.x
            var = ((xf * xf).mean(-1, keepdim=True) - xf.mean(-1, keepdim=True) ** 2).double()
        else:
            var = (d * d).mean(-1, keepdim=True)
        rs = torch.rsqrt(var.clamp_min(0) + EPS_LN)
        n = d * rs * gn
        if self.beta is not None and not drop_beta:
            n = n + self.beta.double()
        return n, (d, rs, m)

    def stats_term(self, W, parts):
        if parts is None:
            return 0.0
        d, rs, m = parts
        K = self.K
        x = self.x.double()
        dm = (K / 256 + 14) * U * x.abs().mean(-1, keepdim=True)
        dm[FAR_ROWS] = 0.0
        var = (d * d).mean(-1, keepdim=True) if self.norm == 2 else (x * x).mean(-1, keepdim=True)
        e_v = (K / 256 + 17) * U + dm * dm / var
        e_rs = e_v / 2 + 3 * U
        if self.norm == 1:
            dm = torch.zeros_like(dm)
        per_k = rs * self.gain.double().abs() * ((e_rs + U) * d.abs() + 1.01 * dm)    # [rows, K]
        return per_k @ W.double().abs().t()

    def linear(self, W, b, n, parts, gamma):
        Wd = W.double()
        y = n @ Wd.t()
        A = n.abs() @ Wd.abs().t()
        if b is not None:
            y = y + b.double()
            A = A + b.double().abs()
        return y, gamma * A + self.stats_term(W, parts)


def gamma_a(K):
    return (K / 32 + 5 + 4) * U


def gamma_b(K, S):
    KB = K // 64
    return (18 * 4 * 2 * math.ceil(KB / S) + S + 4) * U + 2.0 ** -16


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def run(case, path=0, kv_fp32=True, ldo_pad=3, ksplit=0):
    """The kernel's out [2 SLOTS, ldo] (NaN-filled, RESID: x rows where written) and k / v caches (random, finite)."""
    lib = _lib.load()
    K, M = case.K, case.M
    ldo = M + ldo_pad
    dev = torch.device("cuda")
    out = torch.full((2 * SLOTS, ldo), float("nan"), device=dev)
    written = case.rows()
    if case.epi == RESID:
        out[written, :M] = case.resid0.to(dev)
    H = K // 128 if case.epi == QKV else 1
    D = 128 * H
    kvd = torch.float32 if kv_fp32 else torch.bfloat16
    kc = torch.randn(2 * SLOTS, H, S_MAX, 128, device=dev).to(kvd)
    vc = torch.randn(2 * SLOTS, H, S_MAX, 128, device=dev).to(kvd)
    k0, v0 = kc.clone(), vc.clone()
    sm = torch.tensor(case.slots, dtype=torch.int32, device=dev)
    pos = case.pos.to(dev)
    x = case.x.to(dev) if path == 0 else case.x[written].to(dev).contiguous()
    dW, dW3, db, db3, dg, dbe = (None if t is None else t.to(dev) for t in (case.W, case.W3, case.bias, case.bias3, case.gain,
                                                                           case.beta))
    rc = lib.mvb_s1_arch_gemv_test(path, case.epi, case.norm, _ptr(dW), _ptr(dW3), _ptr(db), _ptr(db3), M, K, _ptr(x), K,
                                   case.n_utts, _ptr(dg), _ptr(dbe), EPS_LN if case.norm == 2 else EPS_RMS, _ptr(out), ldo,
                                   _ptr(kc), _ptr(vc), _ptr(sm), _ptr(pos), H, S_MAX, D, int(kv_fp32), ksplit,
                                   C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, lib.mvb_last_error()
    return out.cpu(), kc.cpu(), vc.cpu(), k0.cpu(), v0.cpu()


def check_out(case, out, ref, bound, path=0):
    rows = case.rows()
    M = case.M
    if path == 0:
        got = out[rows, :M].double()
        rest = torch.ones(out.shape, dtype=torch.bool)
        rest[rows, :M] = False
    else:
        got = out[:len(rows), :M].double()
        rest = torch.ones(out.shape, dtype=torch.bool)
        rest[:len(rows), :M] = False
    assert torch.isnan(out[rest]).all(), "an entry outside the written rows / columns changed"
    err = (got - ref[rows]).abs()
    assert torch.isfinite(got).all()
    assert bool((err <= bound[rows]).all()), float((err / bound[rows]).max())
    return got


def n_over(got, alt, bound, rows):
    return int(((got - alt[rows]).abs() > bound[rows]).sum())


def ref_qkv(case, path=0, S=1, drop_bias_kv=False, one_pass=False, drop_beta=False, bias_per_split=False):
    n, parts = case.operand(one_pass, drop_beta)
    g = gamma_a(case.K) if path == 0 else gamma_b(case.K, S)
    b = case.bias
    y, bound = case.linear(case.W, b, n, parts, g)
    if bias_per_split and b is not None:
        y = y + (S - 1) * b.double()
    if drop_bias_kv and b is not None:
        D = case.M // 3
        y[:, D:] -= b.double()[D:]
    return y, bound


def check_cache(case, out, kc, vc, k0, v0, kv_fp32, path=0):
    """Cache entries at (2 s + c, head, pos[s]) equal the kernel's own k / v outputs; every other entry is untouched."""
    D = case.M // 3
    H = D // 128
    rows = case.rows()
    touched = torch.zeros(kc.shape, dtype=torch.bool)
    for i, r in enumerate(rows):
        s = r // 2
        p = int(case.pos[s])
        o = out[r if path == 0 else i]
        for which, cache in ((0, kc), (1, vc)):
            want = o[D * (1 + which): D * (2 + which)].view(H, 128)
            if not kv_fp32:
                want = want.to(torch.bfloat16)
            assert torch.equal(cache[r, :, p].to(want.dtype), want)
        touched[r, :, p] = True
    assert torch.equal(kc[~touched], k0[~touched]) and torch.equal(vc[~touched], v0[~touched])


# ------------------------------------------------------------------------------------------------ QKV
QKV_CASES = [  # (K, n_utts, norm, beta, bias, kv_fp32)
    (2048, 1, 2, True, True, True), (2048, 3, 2, True, True, False), (2048, 8, 2, False, True, True),
    (2048, 3, 1, False, True, True), (2048, 8, 0, False, True, False), (256, 3, 2, True, True, True),
    (256, 8, 2, True, False, False),
]


@pytest.mark.parametrize("K,n_utts,norm,beta,bias,kv_fp32", QKV_CASES)
def test_gemv_qkv(K, n_utts, norm, beta, bias, kv_fp32):
    case = Case(K, 3 * K, n_utts, norm, beta, bias, 100 + K + n_utts, QKV)
    out, kc, vc, k0, v0 = run(case, kv_fp32=kv_fp32)
    y, bound = ref_qkv(case)
    got = check_out(case, out, y, bound)
    check_cache(case, out, kc, vc, k0, v0, kv_fp32)
    rows = case.rows()
    if bias:
        assert n_over(got, ref_qkv(case, drop_bias_kv=True)[0], bound, rows) > 0
    if beta:
        assert n_over(got, ref_qkv(case, drop_beta=True)[0], bound, rows) > 0
    if norm == 2 and 5 in case.slots:
        assert n_over(got, ref_qkv(case, one_pass=True)[0], bound, rows) > 0


@pytest.mark.parametrize("K,n_utts,ksplit,norm,beta,kv_fp32", [
    (2048, 1, 1, 2, True, True), (2048, 3, 4, 2, True, False), (2048, 8, 8, 2, False, True), (2048, 8, 3, 1, False, True),
    (256, 3, 2, 2, True, True), (256, 1, 4, 0, False, False)])
def test_tc_qkv_biased(K, n_utts, ksplit, norm, beta, kv_fp32):
    case = Case(K, 3 * K, n_utts, norm, beta, True, 200 + K + ksplit, QKV)
    out, kc, vc, k0, v0 = run(case, path=1, kv_fp32=kv_fp32, ksplit=ksplit)
    y, bound = ref_qkv(case, path=1, S=ksplit)
    got = check_out(case, out, y, bound, path=1)
    check_cache(case, out, kc, vc, k0, v0, kv_fp32, path=1)
    rows = case.rows()
    assert n_over(got, ref_qkv(case, path=1, S=ksplit, drop_bias_kv=True)[0], bound, rows) > 0
    if ksplit > 1:
        assert n_over(got, ref_qkv(case, path=1, S=ksplit, bias_per_split=True)[0], bound, rows) > 0
    if beta:
        assert n_over(got, ref_qkv(case, path=1, S=ksplit, drop_beta=True)[0], bound, rows) > 0


# ------------------------------------------------------------------------------------------------ MLP, residual, head
def gelu(y, tanh=False):
    if tanh:
        return 0.5 * y * (1 + torch.tanh(math.sqrt(2 / math.pi) * (y + 0.044715 * y ** 3)))
    return 0.5 * y * (1 + torch.erf(y / math.sqrt(2)))


@pytest.mark.parametrize("K,M,n_utts,norm,beta,bias", [
    (2048, 8192, 1, 2, True, True), (2048, 8192, 3, 2, False, True), (2048, 8192, 8, 1, False, False),
    (256, 1024, 3, 2, True, True), (256, 1024, 8, 0, False, True)])
def test_gemv_gelu(K, M, n_utts, norm, beta, bias):
    case = Case(K, M, n_utts, norm, beta, bias, 300 + n_utts + K, GELU)
    out, *_ = run(case)
    n, parts = case.operand()
    y, e_y = case.linear(case.W, case.bias, n, parts, gamma_a(K))
    h = gelu(y)
    bound = 1.13 * e_y + 8 * U * (h.abs() + y.abs())
    got = check_out(case, out, h, bound)
    rows = case.rows()
    assert n_over(got, gelu(y, tanh=True), bound, rows) > 0
    if beta:
        n2, _ = case.operand(drop_beta=True)
        assert n_over(got, gelu(case.linear(case.W, case.bias, n2, parts, 0)[0]), bound, rows) > 0


@pytest.mark.parametrize("K,M,n_utts,norm,beta,bias", [
    (2048, 5632, 1, 2, True, True), (2048, 5632, 8, 1, False, True), (256, 768, 3, 2, True, True)])
def test_gemv_swiglu(K, M, n_utts, norm, beta, bias):
    case = Case(K, M, n_utts, norm, beta, bias, 400 + n_utts + K, SWIGLU)
    out, *_ = run(case)
    n, parts = case.operand()
    g_, e_g = case.linear(case.W, case.bias, n, parts, gamma_a(K))
    v_, e_v = case.linear(case.W3, case.bias3, n, parts, gamma_a(K))
    sg = g_ * torch.sigmoid(g_)
    h = sg * v_
    bound = 1.1 * e_g * v_.abs() + sg.abs() * e_v + 1.1 * e_g * e_v + (8 + torch.floor(1.17 * g_.abs())) * U * h.abs()
    got = check_out(case, out, h, bound)
    if bias:
        g2 = case.linear(case.W, None, n, parts, 0)[0]
        assert n_over(got, g2 * torch.sigmoid(g2) * v_, bound, case.rows()) > 0


@pytest.mark.parametrize("K,M,n_utts,bias", [(8192, 2048, 1, True), (8192, 2048, 8, False), (5632, 2048, 3, True),
                                             (2048, 2048, 3, True), (1024, 256, 8, True)])
def test_gemv_resid_biased(K, M, n_utts, bias):
    """wo / mlp.c_proj + bias + residual; K = 8192 is the GELU c_proj (staging rows past the default 48 KB)."""
    case = Case(K, M, n_utts, 0, False, bias, 500 + K + n_utts, RESID)
    g = torch.Generator().manual_seed(9)
    case.resid0 = torch.randn(len(case.rows()), M, generator=g).float()
    out, *_ = run(case)
    n, parts = case.operand()
    y, e_y = case.linear(case.W, case.bias, n, parts, gamma_a(K))
    r0 = torch.zeros(2 * SLOTS, M, dtype=torch.float64)
    r0[case.rows()] = case.resid0.double()
    ref = r0 + y
    got = check_out(case, out, ref, e_y + U * ref.abs())
    if bias:
        assert n_over(got, r0 + case.linear(case.W, None, n, parts, 0)[0], e_y + U * ref.abs(), case.rows()) > 0


@pytest.mark.parametrize("n_utts,beta", [(1, True), (3, True), (8, False)])
def test_gemv_head_layernorm(n_utts, beta):
    """ln_f (LayerNorm, optional beta) + the tied head over V = 2562, no bias (model.py:128-143)."""
    case = Case(2048, 2562, n_utts, 2, beta, False, 600 + n_utts, STORE)
    out, *_ = run(case)
    n, parts = case.operand()
    y, bound = case.linear(case.W, None, n, parts, gamma_a(2048))
    got = check_out(case, out, y, bound)
    if 5 in case.slots:
        assert n_over(got, case.linear(case.W, None, case.operand(one_pass=True)[0], parts, 0)[0], bound, case.rows()) > 0
