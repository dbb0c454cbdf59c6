"""GPU: the fp8 KV cache's kernels (kv_dtype="fp8"): k_kv_store_f8 bit for bit against mvb200/quantize.py
quantize_kv_fp8, and k_attn_decode_f8 / k_attn_rows_f8 against float64 attention over the DEQUANTISED cache.

Store.  Through the test hook mvb_s1_kv_f8_store_test (k_kv_store_f8 as path B launches it): codes and scales are
bit-identical to quantize_kv_fp8 on random vectors over 2^-30 .. 2^20, zero vectors, fp32-subnormal vectors, vectors whose
codes are e4m3 subnormals, exact e4m3 rounding ties and vectors holding NaN, +inf or -inf.

Attention.  The probe model of test_attention_ops_gpu.py (its docstring derives the bound) with an fp8 cache: injected
K / V are quantised with quantize_kv_fp8 and written as codes and scales, every other code is poisoned with 0x7f (NaN) and
every other scale with NaN.  After one mvb_s1_step_logits (or one prefill) every cache byte except the appended codes and
scales is unchanged, the appended entries dequantise to within one e4m3 step of n_sel (plus the 2^-15 of the projection),
and the merged output satisfies the fp32-cache bound of attn_core (paths A and B) against float64 attention over the
dequantised injected entries plus the appended ones read back.  The dequantised values are exact, so the bound is the
same as for an fp32 cache.  Which body ran is taken from the launch-count delta: with an fp8 cache the engine never takes
path C."""
import ctypes as C
import math

import pytest
import torch

import test_attention_ops_gpu as A
from mvb200 import quantize as Q

pytestmark = pytest.mark.gpu

BLOCK = A.BLOCK
# body -> launches of one mvb_s1_step_logits on the one-layer probe (k_identity_slots included): the store kernel adds
# one launch per layer to the bodies of test_attention_ops_gpu.BODY_LAUNCHES (A: embed + 6 + head; B: rows + embed +
# 4 linears x 2 + store + attention + head x 2)
BODY_LAUNCHES = {"A": 1 + 8, "B": 1 + 14}
# form -> (tensor_core_path, body for n utterances)
FORMS = {"A": ("", lambda n: "A"), "B": ("B", lambda n: "B"), "default": (None, lambda n: "A" if n == 1 else "B")}


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---- k_kv_store_f8 --------------------------------------------------------------------------------------------------
def _store(vecs_k, vecs_v, H):
    """Run the hook on R rows: vecs_k / vecs_v fp32 [R, H, 128] -> (codes [2, R, H, 128] uint8, scales [2, R, H] int16) of
    each row stored at cache row n, position n % 5 of a 5-slot cache."""
    from mvb200 import _lib
    lib = _lib.load()
    R = vecs_k.shape[0]
    D = 128 * H
    qkv = torch.full((R, 3 * D), 7.0, device="cuda")
    qkv[:, D:2 * D] = vecs_k.reshape(R, D).cuda()
    qkv[:, 2 * D:] = vecs_v.reshape(R, D).cuda()
    S = 5
    rows = torch.arange(R, dtype=torch.int32, device="cuda")
    pos = (rows % S).to(torch.int32)
    codes = torch.full((2, R, H, S, 128), 0xA5, dtype=torch.uint8, device="cuda")
    scales = torch.full((2, R, H, S), 0x1234, dtype=torch.int16, device="cuda")
    _lib.check(lib.mvb_s1_kv_f8_store_test(qkv.data_ptr(), R, H, R, S, rows.data_ptr(), pos.data_ptr(), codes.data_ptr(),
                                           scales.data_ptr(), _stream()))
    p = pos.long()
    r = torch.arange(R, device="cuda")
    got_c = codes[:, r, :, p].permute(1, 0, 2, 3).cpu()            # [2, R, H, 128]
    got_s = scales[:, r, :, p].permute(1, 0, 2).cpu()
    # nothing else written
    untouched = torch.ones(2, R, H, S, dtype=torch.bool)
    untouched[:, r.cpu(), :, p.cpu()] = False
    assert bool((codes.cpu()[untouched] == 0xA5).all()) and bool((scales.cpu()[untouched] == 0x1234).all())
    return got_c, got_s


def _check_store(vk, vv, H, label):
    got_c, got_s = _store(vk, vv, H)
    for i, v in enumerate((vk, vv)):
        c, s = Q.quantize_kv_fp8(v)
        bad = (got_c[i] != c.view(torch.uint8)).nonzero()
        assert bad.numel() == 0, f"{label}: {bad.shape[0]} codes differ, first {bad[0].tolist()}"
        assert torch.equal(got_s[i], s.view(torch.int16)), f"{label}: scales differ"


def _e4m3_values():
    v = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).float()
    return v[torch.isfinite(v)]


@pytest.mark.parametrize("H", [1, 16])
def test_store_bit_identical_to_quantize_kv_fp8(H):
    g = torch.Generator().manual_seed(H)
    R = 40
    # random vectors over 2^-30 .. 2^20 (one magnitude per vector, and a spread inside it)
    mag = torch.exp2(torch.randint(-30, 21, (R, H, 1), generator=g).float())
    spread = torch.exp2(torch.randint(-12, 1, (R, H, 128), generator=g).float())
    _check_store(torch.randn(R, H, 128, generator=g) * mag * spread, torch.randn(R, H, 128, generator=g) * mag, H, "random")
    # zero vectors (and -0)
    z = torch.zeros(R, H, 128)
    z[::2] = -0.0
    _check_store(z, z.clone(), H, "zero")
    # fp32-subnormal vectors: the scale is FLT_EPSILON, every code a signed zero
    sub = torch.randn(R, H, 128, generator=g) * 1e-40
    _check_store(sub, sub * -3, H, "fp32 subnormal")
    # e4m3-subnormal codes: one element at 448 2^e, the rest below 2^-6 of it
    es = torch.randn(R, H, 128, generator=g) * 2.0 ** -8
    es[..., 0] = 448.0
    _check_store(es * 2.0 ** 4, es * 2.0 ** -9, H, "e4m3 subnormal")
    # exact rounding ties: midpoints of adjacent e4m3 values at scale 1 (one element pins amax = 448)
    vals = _e4m3_values().unique()
    mids = (vals[1:] + vals[:-1]) / 2                                    # exact in fp32
    idx = torch.randint(0, mids.numel(), (R, H, 128), generator=g)
    t = mids[idx]
    t[..., 0] = 448.0
    _check_store(t, -t, H, "ties")
    # NaN, +inf, -inf (alone and together) at random places
    y = torch.randn(R, H, 128, generator=g)
    w = torch.randn(R, H, 128, generator=g)
    for r in range(R):
        j = int(torch.randint(0, 128, (1,), generator=g))
        kind = r % 4
        if kind == 0:
            y[r, 0, j] = float("nan")
        elif kind == 1:
            y[r, 0, j] = float("inf")
        elif kind == 2:
            y[r, 0, j] = -float("inf")
        else:
            y[r, 0, j], y[r, 0, (j + 1) % 128], w[r, 0, j] = float("inf"), float("nan"), -float("inf")
    _check_store(y, w, H, "non-finite")


# ---- attention through the probe model ------------------------------------------------------------------------------
class ProbeF8:
    """test_attention_ops_gpu.Probe's weights on an engine with an fp8 cache: codes [K|V][row][head][pos][128] and scales
    [K|V][row][head][pos] views of the one-layer cache."""

    def __init__(self, H, form, utts):
        tc, self.body_of = FORMS[form]
        self.p = A.Probe(H, "A-fp32", utts, seed=H)
        p = self.p
        p.m.setup_caches(2 * utts, BLOCK, kv_dtype="fp8", tensor_core_path=tc)
        p.kv, p.form = "fp8", f"fp8-{form}"
        n_vec = 2 * 2 * utts * H * BLOCK
        raw = p.m._kv
        assert raw.numel() == 130 * n_vec
        self.codes = raw[:128 * n_vec].view(2, 2 * utts, H, BLOCK, 128)
        self.scales = raw[128 * n_vec:].view(torch.bfloat16).view(2, 2 * utts, H, BLOCK)
        self.H, self.form = H, form

    def close(self):
        self.p.close()

    def write(self, which, row, t0, vals):
        """quantise float64 vals [H, n, 128] into entries [t0, t0 + n) of cache row `row`; returns the dequantised values."""
        c, s = Q.quantize_kv_fp8(vals.float())
        n = vals.shape[1]
        self.codes[which, row, :, t0:t0 + n] = c.view(torch.uint8).cuda()
        self.scales[which, row, :, t0:t0 + n] = s.cuda()
        return Q.dequantize_kv_fp8(c, s).double().cuda()

    def read(self, which, row, t0, t1):
        return Q.dequantize_kv_fp8(self.codes[which, row, :, t0:t1].cpu().view(torch.float8_e4m3fn),
                                   self.scales[which, row, :, t0:t1].cpu()).double().cuda()

    def poison(self):
        self.codes[:] = 0x7F
        self.scales[:] = float("nan")


def _check_appended(q8, got, ref, label):
    """appended dequantised k / v within one e4m3 step of n_sel (plus the projection's 2^-15)"""
    s = ref.abs().amax(-1, keepdim=True) / 448
    step = torch.maximum(ref.abs() * 2.0 ** -3, s * 2.0 ** -9)
    bound = step + 2.0 ** -14 * ref.abs() + 1e-30
    assert ((got - ref).abs() <= bound).all(), f"{label}: appended entry more than one e4m3 step from n_sel"


def _bound(p, r):
    y, s, Aa, PV = A.reference(r)
    L = r["L"]
    eps = A.softmax_eps(s, Aa, L / 64 + 2, L / 32 + 40, A.KAPPA_S1, 0.0) * PV
    tau = A.TAU_OBS_A if r["body"] == "A" else A.TAU_OBS
    return y, eps + tau * (r["x"].view(p.H, 128).abs() + y.abs() + eps) + 1e-30


def _check_rows(p, rows, label):
    worst = nw_worst = 0.0
    for r in rows:
        y, bound = _bound(p, r)
        err = (r["y_hat"] - y).abs()
        err[:, A.PILOT] = 0
        bad = (err > bound).nonzero()
        ratio = float((err / bound).max())
        assert bad.numel() == 0, f"{label} utt {r['u']} L={r['L']}: {bad.shape[0]} over the bound (max ratio {ratio:.2e})"
        nw = float(err.norm() / y.norm())
        assert nw < A.NORMWISE, f"{label} L={r['L']}: normwise {nw:.2e}"
        worst, nw_worst = max(worst, ratio), max(nw_worst, nw)
    return worst, nw_worst


def run_decode(q8, Ls, regime, seed, needles=None):
    from mvb200 import _lib
    p = q8.p
    n = len(Ls)
    g = torch.Generator(device="cuda").manual_seed(seed)
    toks = torch.randint(0, p.V, (n,), generator=torch.Generator().manual_seed(seed)).tolist()
    q8.poison()
    rows = []
    for u, L in enumerate(Ls):
        x = p.x(torch.tensor(toks[u], device="cuda"), torch.tensor(L - 1, device="cuda"))
        q, kc, vc = p.sel(x)
        for c in range(2):
            K, Vv = A.make_kv(p, q, L, regime, g, None if needles is None else needles[u])   # float64 of bf16 values
            Kd = q8.write(0, 2 * u + c, 0, K) if L > 1 else K
            Vd = q8.write(1, 2 * u + c, 0, Vv) if L > 1 else Vv
            rows.append(dict(u=u, c=c, L=L, x=x, q=q, kc=kc, vc=vc, K=Kd, V=Vd))
    before = p.m._kv.clone()
    lib, h, st = p.m._lib, p.m.handle, p.m._stream()
    sp = _lib.Sampling(1.0, 1.0, 0.0, 0, 9999, 1)
    for u, L in enumerate(Ls):
        _lib.check(lib.mvb_s1_begin(h, u, int(toks[u]), L - 1, C.byref(sp), None, None, st))
    n0 = A._launches(p)
    lg = torch.empty(2 * n, p.V, device="cuda")
    _lib.check(lib.mvb_s1_step_logits(h, n, lg.data_ptr(), st))
    torch.cuda.synchronize()
    body = q8.body_of(n)
    assert A._launches(p) - n0 == BODY_LAUNCHES[body], f"{q8.form}: body {body} did not run (path C must never run)"
    after = p.m._kv.clone()
    codes_b = before[:q8.codes.numel()].view(q8.codes.shape)
    scales_b = before[q8.codes.numel():].view(torch.bfloat16).view(q8.scales.shape)
    for r in rows:
        cr, L = 2 * r["u"] + r["c"], r["L"]
        codes_b[:, cr, :, L - 1] = q8.codes[:, cr, :, L - 1]
        scales_b[:, cr, :, L - 1] = q8.scales[:, cr, :, L - 1]
    assert torch.equal(after, before), f"{q8.form}: the step changed cache bytes other than the appended codes and scales"
    for r in rows:
        cr, L = 2 * r["u"] + r["c"], r["L"]
        ka, va = q8.read(0, cr, L - 1, L)[:, 0], q8.read(1, cr, L - 1, L)[:, 0]
        _check_appended(q8, ka, r["kc"], f"{q8.form} L={L} k")
        _check_appended(q8, va, r["vc"], f"{q8.form} L={L} v")
        r["K_all"] = torch.cat([r["K"], ka[:, None]], 1)
        r["V_all"] = torch.cat([r["V"], va[:, None]], 1)
        r["y_hat"] = p.recover(lg[cr], r["x"]).view(p.H, 128)
        r["body"] = body
    return rows


@pytest.fixture(scope="module")
def probes():
    cache = {}

    def get(H, form, utts):
        key = (H, form, utts)
        if key not in cache:
            for k in list(cache):
                cache.pop(k).close()
            torch.cuda.empty_cache()
            cache[key] = ProbeF8(H, form, utts)
        return cache[key]
    yield get
    for v in cache.values():
        v.close()


@pytest.mark.parametrize("H", [2, 16])
@pytest.mark.parametrize("form", ["A", "B"])
def test_decode_every_length(probes, form, H):
    """Every L of test_attention_ops_gpu.L_CASES (path A: 1 utterance, path B: 2 at the same L) and 8 utterances with
    mixed L in one step, flat / wide / tied scores, over the dequantised cache."""
    q8 = probes(H, form, 8)
    single = 2 if form == "B" else 1
    worst = nw = 0.0
    for regime in ("flat", "wide", "ties"):
        for i, L in enumerate(A.L_CASES):
            w, n = _check_rows(q8.p, run_decode(q8, [L] * single, regime, seed=1000 * H + 10 * i), f"fp8-{form} {regime}")
            worst, nw = max(worst, w), max(nw, n)
        w, n = _check_rows(q8.p, run_decode(q8, A.MIXED_8, regime, seed=7 + H), f"fp8-{form} {regime} mixed-8")
        worst, nw = max(worst, w), max(nw, n)
    print(f"fp8 KV decode {form} H={H}: every L in {A.L_CASES[0]}..{A.L_CASES[-1]} + mixed 8: max |err|/bound {worst:.2e}, "
          f"normwise {nw:.2e}")


@pytest.mark.parametrize("form", ["A", "B"])
def test_decode_needles(probes, form):
    q8 = probes(2, form, 8)
    worst = 0.0
    for L in A.NEEDLE_LS:
        for nd in A._needles(L):
            w, _ = _check_rows(q8.p, run_decode(q8, [L] * (2 if form == "B" else 1), "needle", seed=L, needles=[nd] * 2),
                               f"fp8-{form} needle {nd} L={L}")
            worst = max(worst, w)
    print(f"fp8 KV needles {form}: max |err|/bound {worst:.2e}")


def test_path_c_never_runs(probes):
    """The default engine (every path enabled) with an fp8 cache: one utterance decodes on path A, 2 and 8 on path B."""
    q8 = probes(2, "default", 8)
    for Ls in ([130], [2048, 1], A.MIXED_8):
        w, nw = _check_rows(q8.p, run_decode(q8, Ls, "wide", seed=len(Ls)), f"fp8-default n={len(Ls)}")
        print(f"fp8 KV default engine, {len(Ls)} utterance(s) [body {q8.body_of(len(Ls))}]: max |err|/bound {w:.2e}")


@pytest.mark.parametrize("pos0", [0, 1000, 1978])
def test_prefill_every_position(probes, pos0):
    """mvb_s1_forward, S = 70 from pos0 on path B (64-token chunks, causal inside the chunk, each chunk's entries stored
    before its attention reads them): every position against float64 attention over the injected [0, pos0) plus the
    entries the prefill appended, read back.  Nothing outside [pos0, pos0 + 70) of rows 0, 1 changes."""
    from mvb200 import _lib
    q8 = probes(2, "B", 1)
    p = q8.p
    S = 70
    g = torch.Generator(device="cuda").manual_seed(pos0)
    idx = torch.randint(0, p.V, (2, S), generator=torch.Generator().manual_seed(pos0), dtype=torch.int32)
    pos = torch.arange(pos0, pos0 + S, device="cuda")
    q8.poison()
    x = p.x(idx.cuda().long(), pos[None].expand(2, S))
    q, kc, vc = p.sel(x)
    inj = []
    for c in range(2):
        K, Vv = A.make_kv(p, q[c, 0], pos0 + 1, "flat", g)
        inj.append((q8.write(0, c, 0, K), q8.write(1, c, 0, Vv)) if pos0 else (K, Vv))
    before = p.m._kv.clone()
    lg = torch.empty(2, S, p.V, device="cuda")
    n0 = A._launches(p)
    _lib.check(p.m._lib.mvb_s1_forward(p.m.handle, 0, idx.cuda().contiguous().data_ptr(), S, pos0, lg.data_ptr(), 1,
                                       p.m._stream()))
    torch.cuda.synchronize()
    # per 64-token chunk: k_rows_prefill + embed + (4 linears x 2 + store + attention) + head (2); then k_gather_last + the
    # last position's head (2) + k_set_input
    assert A._launches(p) - n0 == -(-S // 64) * (1 + 1 + 10 + 2) + 4
    after = p.m._kv.clone()
    codes_b = before[:q8.codes.numel()].view(q8.codes.shape)
    scales_b = before[q8.codes.numel():].view(torch.bfloat16).view(q8.scales.shape)
    codes_b[:, :2, :, pos0:pos0 + S] = q8.codes[:, :2, :, pos0:pos0 + S]
    scales_b[:, :2, :, pos0:pos0 + S] = q8.scales[:, :2, :, pos0:pos0 + S]
    assert torch.equal(after, before), "the prefill changed cache bytes outside [pos0, pos0 + S)"
    worst = nw = 0.0
    for c in range(2):
        Ka, Va = q8.read(0, c, pos0, pos0 + S), q8.read(1, c, pos0, pos0 + S)
        _check_appended(q8, Ka, kc[c].transpose(0, 1), f"prefill pos0={pos0} k")
        _check_appended(q8, Va, vc[c].transpose(0, 1), f"prefill pos0={pos0} v")
        Kall = torch.cat([inj[c][0][:, :pos0], Ka], 1)
        Vall = torch.cat([inj[c][1][:, :pos0], Va], 1)
        for i in range(S):
            L = pos0 + i + 1
            r = dict(u=0, c=c, L=L, x=x[c, i], q=q[c, i], K_all=Kall[:, :L], V_all=Vall[:, :L], body="B",
                     y_hat=p.recover(lg[c, i], x[c, i]).view(p.H, 128))
            w, n = _check_rows(p, [r], f"fp8 prefill pos0={pos0} i={i}")
            worst, nw = max(worst, w), max(nw, n)
    print(f"fp8 KV prefill pos0={pos0}, 70 positions: max |err|/bound {worst:.2e}, normwise {nw:.2e}")
