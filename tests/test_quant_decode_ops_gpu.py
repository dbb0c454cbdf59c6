"""GPU: the int8, int4 and fp8 stage-1 engines at production width (metavoice-1B: D = 2048, H = 16, F = 5632, V = 2562,
24 layers, block_size 256) through the probe model of tests/test_decode_linear_ops_gpu.py, against float64.  The op
tests of the three GEMVs take a matrix and a scale pointer from the test; these check how the engine finds each layer's
matrices and scales (lw, tc_lscale, w8_scale_offset, the per-layer widen into the scratch the tensor maps point at).

PROBE MODEL.  One arena per format, packed by quantize.pack_arena_int8 / pack_arena_int4 / pack_arena_fp8 from an
all-zero state dict; the embedding tables, the speaker projection (0.5 x a selection matrix: q = 1, s = 0.5) and the
observation head [I_D; 0] (q = 1, s = 1; int4: bf16) are those of test_decode_linear_ops_gpu.py's Arena and are written
before the engine is created (an int8 / fp8 engine widens lm_head's q, an fp8 engine speaker_cond_pos's, at create).
Every layer matrix holds zero codes under its own bf16 scales that are not powers of two (int4: q = 0, z = 8 s, so
W_deq = 0 exactly): a wrong-layer or wrong-matrix scale read in the engine gives a wrong result, not an equal one.
Each case packs random matrices (quantize.pack_int8_matrix / pack_matrix / pack_fp8_matrix) into the slices of one
target layer l* in {0, 12, 23} and restores the zero layer afterwards.  Scales are drawn as bf16 values over two
octaves, never a power of two, one draw per matrix; codes hit the edges: int8 +-127, fp8 +-448 with every subnormal code
and both zeros, int4 codes 0 and 15 under non-zero zero points.  The function of each matrix is W = s q (int8, fp8,
exact in float64) or W_deq = bf16_rn((q - 8) s + z) (int4); reference_weight() is checked on the CPU against
quantize.dequantize_int8 / dequantize_fp8 / dequantize.

PROBES (test_decode_linear_ops_gpu.py): qkv (k, v read back from an fp32 and a bf16 cache), wo + residual (observed
through the pilot rows), the FFN (SwiGLU with separate w1 / w3 scales, nine w1 rows scaled to the __expf corners, then
w2), the head with ln_f (all 2562 logits, the ragged tail), mixed positions over three launches.  Batches: path A
(k_gemv_w8 / k_gemv_w4 / k_gemv_f8; fp8 at NB = 1 for 1 and 3 slots, NB = 2 for 5 and 8) at 1, 3, 5, 8 slots, each
slot with its own token, speaker and position; fp8 path B (k_f8_widen per layer, k_tc_gemm with row scales) at 9 and
12 slots; prefill through path B for all three formats at T = 70 (two chunks), k and v of every position checked.
The head on fp8's path B reads lm_head's q widened at create, so that probe creates its engine after writing lm_head.

BOUNDS (reused, not re-derived):
  path A: gamma of the format's GEMV test, tests/test_int8_gemv_gpu.py ((16 ceil(K / 512) + 5) u, + 2^-22 with the
    RMSNorm prologue), tests/test_int4_gemv_gpu.py ((32 ceil(NT / 2) + 5) u, + 2^-22) and tests/test_fp8_gemv_gpu.py
    ((2 K / 128 + 8) 2^-22 + 2^-16, + 2^-21 + 2^-23); the int4 engine's lm_head is bf16 (k_gemv: path A of
    test_decode_linear_ops_gpu.py);
  path B: lin_bound of test_decode_linear_ops_gpu.py (the m16n8k16 model per split, the plan_gemm K split) applied to W,
    as test_int8_gemv_gpu.py::test_tc_gemm_row_scales does;
  int8 / fp8 add u (|y| + bound) for the row-scale multiply;
  observation, FFN chain and mixed-position terms: test_decode_linear_ops_gpu.py (tau_obs 2^-20 for k_gemv / k_gemv_w8 /
    k_gemv_w4, 2^-15 for the hi + lo operand of k_gemv_f8 and path B).
Each check prints its worst |err| / bound and applies the normwise 1e-4 (1e-3 for a bf16 cache) check.

SENSITIVITY: references with (a) layer l* - 1's scales (layer 1's at l* = 0), (b) w1's scales on w3, (c) each row's
scale (int4: each group's) taken from its neighbour, (d) on path B at l* > 0 layer l* - 1's codes (the stale widen: the
scratch was not refreshed), (e) fp8: one slot's two CFG rows swapped at NB = 2, (f) int4: the zero point dropped, must
each put elements over the bound.  Every cache entry outside the appended positions and every logits row outside the
batch must be unchanged."""
import ctypes as C
import math
from types import SimpleNamespace

import pytest
import torch

import test_decode_linear_ops_gpu as dl
from mvb200 import quantize as Q

D, H, F, V, NL, BLOCK, SPK = dl.D, dl.H, dl.F, dl.V, dl.NL, dl.BLOCK, dl.SPK
U = dl.U
TAU_GAIN = 2.0 ** -22
FMTS = ("int8", "int4", "fp8")
LSTAR = dl.LSTAR
# layer tensor index (fast_model._LAYER_KEYS) -> (name, M, K)
MATS = {1: ("attn.c_attn.weight", 3 * D, D), 2: ("attn.c_proj.weight", D, D), 4: ("mlp.swiglu.w1.weight", F, D),
        5: ("mlp.swiglu.w3.weight", F, D), 6: ("mlp.c_proj.weight", D, F)}
DLMAT = {1: "qkv", 2: "o", 4: "w13", 5: "w13", 6: "w2"}
PATH_A_N = (1, 3, 5, 8)
PATH_B_N = (9, 12)
# launches of one mvb_s1_step_logits: A embed + 5 per layer + head; fp8's B rows + embed + per layer (widen + 9) + head 2
LAUNCHES = {"A": 1 + 1 + 5 * NL + 1, "B": 1 + 1 + 1 + 10 * NL + 2}
PREFILL_T, PREFILL_P0 = 70, 100


# ---- float64 reference helpers (CPU-checked) --------------------------------------------------------------------------
def nonpow2_bf16(n, base, g):
    """n bf16 values base * 2^U(-1, 1) (two octaves), none a power of two (a zero mantissa is moved up one ulp)."""
    v = (base * torch.exp2(2 * torch.rand(n, generator=g, dtype=torch.float64) - 1)).float().to(torch.bfloat16)
    bits = v.view(torch.int16)
    return torch.where((bits & 0x7F) == 0, bits + 1, bits).view(torch.bfloat16)


def reference_weight(fmt, q, s, z=None):
    """float64 W the engine computes with: s q (int8, fp8; exact) or W_deq = bf16_rn((q - 8) s + z) (int4)."""
    if fmt == "int4":
        return Q.dequantize(q, s, z).double()
    return q.double() * s.double()[:, None]


def fp8_codes(M, K, g):
    """e4m3 codes [M, K] uniform over the 254 finite codes; row 0 starts with both zeros, all 14 subnormals and +-448."""
    c = torch.randint(0, 254, (M, K), generator=g)
    c = c + (c >= 0x7F).long()                                     # skip 0x7f; 0xff is past the range
    edge = [0x00, 0x80] + list(range(1, 8)) + list(range(0x81, 0x88)) + [0x7E, 0xFE]
    c[0, :len(edge)] = torch.tensor(edge)
    return c.to(torch.uint8).view(torch.float8_e4m3fn)


def draw(fmt, M, K, std, g, zero_rows=None):
    """Random packed matrix with entries of about `std`: (packed uint8 CPU blob, q, s, z or None)."""
    if fmt == "int8":
        q = torch.randint(-127, 128, (M, K), generator=g, dtype=torch.int8)
        q[0, :2] = torch.tensor([127, -127], dtype=torch.int8)
        if zero_rows is not None:
            q[zero_rows] = 0
        s = nonpow2_bf16(M, std / 73.3, g)
        return Q.pack_int8_matrix(q, s), q, s, None
    if fmt == "fp8":
        q = fp8_codes(M, K, g)
        if zero_rows is not None:
            q[zero_rows] = torch.zeros((), dtype=torch.float8_e4m3fn)
        rms = float(q.float().pow(2).mean().sqrt())
        s = nonpow2_bf16(M, std / rms, g)
        return Q.pack_fp8_matrix(q, s), q, s, None
    q = torch.randint(0, 16, (M, K), generator=g, dtype=torch.uint8)
    q[0, :2] = torch.tensor([0, 15], dtype=torch.uint8)
    s = nonpow2_bf16(M * (K // 128), std / 4.6, g).view(M, K // 128)
    zf = s.float() * (0.5 + 2.5 * torch.rand(M, K // 128, generator=g)) * (torch.randint(0, 2, (M, K // 128), generator=g) * 2 - 1)
    z = zf.to(torch.bfloat16)
    if zero_rows is not None:
        q[zero_rows] = 0
        z[zero_rows] = (8 * s[zero_rows].float()).to(torch.bfloat16)     # W_deq = bf16_rn(-8 s + 8 s) = 0
    return Q.pack_matrix(q, s, z), q, s, z


def zero_layer(fmt, M, K, g):
    """Zero codes under distinct non-power-of-two scales (int4: q = 0, z = 8 s)."""
    if fmt == "int4":
        s = nonpow2_bf16(M * (K // 128), 2.0 ** -7, g).view(M, K // 128)
        q = torch.zeros(M, K, dtype=torch.uint8)
        z = (8 * s.float()).to(torch.bfloat16)
        return Q.pack_matrix(q, s, z), q, s, z
    s = nonpow2_bf16(M, 2.0 ** -7, g)
    if fmt == "int8":
        q = torch.zeros(M, K, dtype=torch.int8)
        return Q.pack_int8_matrix(q, s), q, s, None
    q = torch.zeros(M, K, dtype=torch.float8_e4m3fn)
    return Q.pack_fp8_matrix(q, s), q, s, None


def gamma_a(fmt, K, gain):
    """gamma of the format's path-A GEMV (module docstring: the three GEMV test files)."""
    if fmt == "int8":
        from test_int8_gemv_gpu import gamma
        return gamma(K) + (TAU_GAIN if gain else 0.0)
    if fmt == "int4":
        from test_int4_gemv_gpu import gamma
        return gamma(K) + (TAU_GAIN if gain else 0.0)
    from test_fp8_gemv_gpu import gamma
    return gamma(K, gain)


def lin_bound(fmt, body, t, y, A, gain, n_sm=None):
    """Elementwise bound of y = W n^ for layer tensor t (or "head") on `body`."""
    mat = "head" if t == "head" else DLMAT[t]
    if body == "A":
        K = D if mat != "w2" else F
        b = gamma_a(fmt, K, gain) * A
    else:
        b = dl.lin_bound("B", mat, y, A, n_sm)
    if fmt != "int4":
        b = b + U * (y.abs() + b)
    return b + 1e-30


def tau_obs(fmt, body):
    return dl.TAU_OBS["B"] if (body == "B" or fmt == "fp8") else dl.TAU_OBS["A"]


def ffn_ref(fmt, body, x, g2, W1, W3, W2, n_sm=None):
    """The float64 FFN and its bound: _ffn_ref of test_decode_linear_ops_gpu.py with the format's gammas."""
    nh, _, s = dl.operand(x, g2, body)
    G, AG = dl.linear(W1, nh, s)
    Uu, AU = dl.linear(W3, nh, s)
    eg = lin_bound(fmt, body, 4, G, AG, True, n_sm) + 2.0 ** -21 * G.abs()
    eu = lin_bound(fmt, body, 5, Uu, AU, True, n_sm) + 2.0 ** -21 * Uu.abs()
    sil = G * torch.sigmoid(G)
    h = sil * Uu
    eps_s = (6 + torch.floor(1.17 * G.abs())) * U
    eh = 1.1 * eg * Uu.abs() + sil.abs() * eu + 1.1 * eg * eu + (eps_s + U) * h.abs() + (G < -80) * h.abs()
    if body != "A" or fmt == "fp8":
        eh = eh + dl.HILO * (h.abs() + eh)
    y = h @ W2.t()
    Ah = (h.abs() + eh) @ W2.abs().t()
    b = lin_bound(fmt, body, 6, y, Ah, False, n_sm) + eh @ W2.abs().t() + (dl.n_split(body, "w2", n_sm) + 1) * U * x.abs()
    return y, b


# ---- CPU self-checks of the helpers -----------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
def test_reference_weight_matches_quantize(fmt):
    g = torch.Generator().manual_seed(1)
    blob, q, s, z = draw(fmt, 48, 256, 0.02, g, zero_rows=torch.tensor([5, 17]))
    W = reference_weight(fmt, q, s, z)
    if fmt == "int4":
        assert torch.equal(W, Q.dequantize(q, s, z).double())
        assert torch.equal(Q.unpack_matrix(blob, 48, 256)[0], q)
        assert bool((q == 0).any() and (q == 15).any()) and bool((z.float() != 0).all())
    else:
        deq = Q.dequantize_int8(q, s) if fmt == "int8" else Q.dequantize_fp8(q, s)
        assert torch.equal(Q._round_to_bf16(W), deq), "bf16_rn(s q) differs from quantize's dequantiser"
        un = Q.unpack_int8_matrix(blob, 48, 256) if fmt == "int8" else Q.unpack_fp8_matrix(blob, 48, 256)
        assert torch.equal(un[0].view(torch.uint8), q.view(torch.uint8)) and torch.equal(un[1], s)
    assert (W[[5, 17]] == 0).all()
    if fmt == "fp8":
        codes = set(q.view(torch.uint8).flatten().tolist())
        assert {0x00, 0x80, 0x7E, 0xFE} | set(range(1, 8)) | set(range(0x81, 0x88)) <= codes and 0x7F not in codes
        assert 0xFF not in codes
    if fmt == "int8":
        assert int(q.max()) == 127 and int(q.min()) == -127
    sv = s.float().flatten()
    assert not any(math.log2(v).is_integer() for v in sv.abs().tolist()), "a power-of-two scale"
    assert float(sv.max() / sv.min()) > 2.5, "scales do not spread over two octaves"
    zb, zq, zs, zz = zero_layer(fmt, 32, 256, g)
    assert (reference_weight(fmt, zq, zs, zz) == 0).all()
    assert not any(math.log2(v).is_integer() for v in zs.float().flatten().abs().tolist())


def test_fp8_cta_mirror():
    """The k_gemv_f8 grids the SM-count test relies on (tests/test_fp8_gemv_gpu.py::test_gemv_f8_at_sm_counts)."""
    from test_fp8_gemv_gpu import F8_SM, f8_gemv_ctas, n_mine
    assert n_mine(128, 132) == [1] * 128 and 160 // f8_gemv_ctas(161, 132) == 1
    for G in F8_SM:
        assert max(n_mine(128, G)) in (2, 3) and sum(n_mine(128, G)) == 128
        assert 160 // f8_gemv_ctas(161, G) == (2 if G <= 80 else 1)


# ---- GPU --------------------------------------------------------------------------------------------------------------
class QArena:
    """The probe arena of one format on the device, with the float64 scales of every zero layer matrix."""

    def __init__(self, fmt):
        from mvb200.fast_model import _GLOBAL_KEYS, _LAYER_KEYS
        self.fmt = fmt
        g = torch.Generator().manual_seed(0)                        # the draws of test_decode_linear_ops_gpu.Arena
        pil = torch.zeros(D, dtype=torch.bool)
        pil[dl.PILOT::128] = True
        tok = torch.randint(-12, 13, (V, D), generator=g).float()
        mag = torch.randint(12, 21, (V, int(pil.sum())), generator=g).float()
        tok[:, pil] = mag * (torch.randint(0, 2, mag.shape, generator=g) * 2 - 1)
        pos = torch.randint(-4, 5, (BLOCK, D), generator=g).float()
        pos[:, pil] = 0
        sel = torch.zeros(D, SPK)
        sel[torch.arange(D), torch.arange(D) % SPK] = 1
        sel[pil] = 0
        self.toks = torch.randperm(V, generator=g)[:3 * 16].view(3, 16).tolist()        # [launch][utterance]
        self.spks = (torch.randint(-8, 9, (16, SPK), generator=g).float() / 32).cuda()
        self.pil_d = pil.cuda()
        self.tok_d, self.pos_d, self.wspk_d = (tok / 32).double().cuda(), (pos / 32).double().cuda(), (0.5 * sel).double().cuda()
        bf = torch.bfloat16
        zero = torch.zeros((), dtype=bf)
        eye = torch.cat([torch.eye(D), torch.zeros(V - D, D)])
        sd = {"transformer.wtes.0.weight": (tok / 32).to(bf), "transformer.wpe.weight": (pos / 32).to(bf),
              "speaker_cond_pos.weight": (0.5 * sel).to(bf), "transformer.ln_f.weight": torch.ones(D, dtype=bf),
              "lm_heads.0.weight": eye.to(bf)}
        for i in range(NL):
            sd[f"transformer.h.{i}.ln_1.weight"] = zero.expand(D)
            sd[f"transformer.h.{i}.ln_2.weight"] = zero.expand(D)
            for t, (name, M, K) in MATS.items():
                sd[f"transformer.h.{i}.{name}"] = zero.expand(M, K)
        pack = {"int8": Q.pack_arena_int8, "int4": Q.pack_arena_int4, "fp8": Q.pack_arena_fp8}[fmt]
        arena, self.offsets = pack(sd, NL)[:2]
        self.keys = list(_GLOBAL_KEYS) + [f"transformer.h.{i}.{k}" for i in range(NL) for k in _LAYER_KEYS]
        self.buf = arena.cuda()
        del arena
        # exact speaker projection (q = 1, s = 0.5) and observation head (q = 1, s = 1); int4 holds both in bf16
        if fmt == "int4":
            self._put_global("speaker_cond_pos.weight", (0.5 * sel).to(bf).view(torch.uint8).flatten())
        else:
            packf = Q.pack_int8_matrix if fmt == "int8" else Q.pack_fp8_matrix
            qt = torch.int8 if fmt == "int8" else torch.float8_e4m3fn
            self._put_global("speaker_cond_pos.weight", packf(sel.to(qt), torch.full((D,), 0.5, dtype=bf)))
            self._put_global("lm_heads.0.weight", packf(eye.to(qt), torch.ones(V, dtype=bf)))
        # every layer matrix: zero codes under its own scales
        self.zero = {}
        gz = torch.Generator().manual_seed(77)
        for l in range(NL):
            for t, (name, M, K) in MATS.items():
                blob, q, s, z = zero_layer(fmt, M, K, gz)
                self.zero[(l, t)] = (s, z)
                self.put(l, t, blob)
        torch.cuda.synchronize()

    def zero_blob(self, l, t):
        """The packed zero matrix t of layer l under its own scales."""
        s, z = self.zero[(l, t)]
        _, M, K = MATS[t]
        if self.fmt == "int4":
            return Q.pack_matrix(torch.zeros(M, K, dtype=torch.uint8), s, z)
        if self.fmt == "int8":
            return Q.pack_int8_matrix(torch.zeros(M, K, dtype=torch.int8), s)
        return Q.pack_fp8_matrix(torch.zeros(M, K, dtype=torch.float8_e4m3fn), s)

    def off(self, key):
        return self.offsets[self.keys.index(key)]

    def _put_global(self, key, blob):
        o = self.off(key)
        self.buf[o:o + blob.numel()].copy_(blob.view(torch.uint8).flatten().cuda())

    def put(self, l, t, blob):
        o = self.off(f"transformer.h.{l}.{MATS[t][0]}")
        self.buf[o:o + blob.numel()].copy_(blob.cuda())

    def gain(self, l, which):
        o = self.off(f"transformer.h.{l}.{which}.weight")
        return self.buf[o:o + 2 * D].view(torch.bfloat16)

    def bf16_global(self, key, shape):
        o = self.off(key)
        return self.buf[o:o + 2 * math.prod(shape)].view(torch.bfloat16).view(*shape)


class QEngine:
    def __init__(self, qa, kv, utts, tc=None):
        from mvb200.fast_model import ModelArgs, Transformer
        self.qa, self.fmt, self.kv, self.utts = qa, qa.fmt, kv, utts
        self.n_sm = dl._n_sm()
        cfg = ModelArgs(block_size=BLOCK, vocab_size=V, n_layer=NL, n_head=H, dim=D, intermediate_size=F)
        self.m = Transformer(cfg, qa.buf, qa.offsets, device="cuda:0", quantisation_mode=qa.fmt)
        self.m.setup_caches(2 * utts, BLOCK, kv_dtype=kv, tensor_core_path=tc)
        self.dt = torch.float32 if kv == "fp32" else torch.bfloat16
        self.cache = self.m._kv.view(self.dt).view(NL, 2, 2 * utts, H, BLOCK, 128)
        for u in range(utts):
            self.m.set_speaker(u, qa.spks[u])
        torch.cuda.synchronize()

    def body(self, n):
        return "B" if (self.fmt == "fp8" and n > 8) else "A"

    def close(self):
        self.m.close()


def step(e, n, toks, poss):
    """begin every utterance at its (token, position), one mvb_s1_step_logits; logits [2 n, V] in float64."""
    from mvb200 import _lib
    lib, h, st = e.m._lib, e.m.handle, e.m._stream()
    sp = _lib.Sampling(1.0, 1.0, 0.0, 0, 9999, 1)
    for u in range(n):
        _lib.check(lib.mvb_s1_begin(h, u, int(toks[u]), int(poss[u]), C.byref(sp), None, None, st))
    n0 = int(lib.mvb_s1_launch_count(h))
    lg = torch.full((2 * n + 3, V), float("nan"), device="cuda")
    _lib.check(lib.mvb_s1_step_logits(h, n, lg.data_ptr(), st))
    torch.cuda.synchronize()
    body = e.body(n)
    assert int(lib.mvb_s1_launch_count(h)) - n0 == LAUNCHES[body], f"{e.fmt} n={n}: body {body} did not run"
    assert torch.isnan(lg[2 * n:]).all(), f"{e.fmt} n={n}: logits rows outside the batch were written"
    return lg[:2 * n].double()


def rows_x(qa, n, toks, poss):
    x = qa.tok_d[torch.tensor(toks[:n]).repeat_interleave(2).cuda()] + qa.pos_d[torch.tensor(poss[:n]).repeat_interleave(2).cuda()]
    x[0::2] += qa.spks[:n].double() @ qa.wspk_d.t()
    return x


def check_cache_rest(e, l, windows, before=None):
    """Every cache entry outside the appended (row pair, positions) windows of layer l is unchanged (zero elsewhere)."""
    for j in range(NL):
        if j != l:
            assert (e.cache[j] == 0).all(), f"{e.fmt}: zero layer {j} cache changed"
    cur = e.cache[l].clone()
    ref = before.clone() if before is not None else torch.zeros_like(cur)
    for u, ps in windows:
        cur[:, 2 * u:2 * u + 2, :, ps] = 0
        ref[:, 2 * u:2 * u + 2, :, ps] = 0
    assert torch.equal(cur.view(torch.uint8), ref.view(torch.uint8)), f"{e.fmt}: layer {l} cache entries outside the appended ones changed"


def appended(e, n, poss, l):
    ks, vs = [], []
    for u in range(n):
        for c in range(2):
            ks.append(e.cache[l, 0, 2 * u + c, :, poss[u]].reshape(D))
            vs.append(e.cache[l, 1, 2 * u + c, :, poss[u]].reshape(D))
    return torch.stack(ks).double(), torch.stack(vs).double()


class Tally:
    def __init__(self):
        self.worst, self.nw, self.sens = {}, {}, {}

    def check(self, key, label, got, ref, bound, mask=None, nw_ref=None, nw_limit=dl.NORMWISE):
        r, w = dl.assess(label, got, ref, bound, mask, nw_ref, nw_limit)
        self.worst[key] = max(self.worst.get(key, 0.0), r)
        self.nw[key] = max(self.nw.get(key, 0.0), w)

    def over(self, name, got, alt, bound, mask=None):
        self.sens[name] = self.sens.get(name, 0) + dl.n_over(got, alt, bound, mask)

    def report(self, title):
        for k in self.worst:
            print(f"{title} {k}: max |err|/bound {self.worst[k]:.2e}, normwise {self.nw[k]:.2e}")
        for k, v in self.sens.items():
            print(f"  sensitivity {title}: reference with {k}: {v} elements over the bound")
            assert v > 0, f"{title}: a reference with {k} satisfies the bound"


class Case:
    """Random matrices of one probe packed into layer l; float64 W and, with sens, the alternative Ws of the
    sensitivity checks."""

    def __init__(self, qa, l, seed, sens=False):
        self.qa, self.l, self.sens = qa, l, sens
        self.g = torch.Generator().manual_seed(seed)
        self.gd = torch.Generator(device="cuda").manual_seed(seed)
        self.written, self.gains = set(), []

    def mat(self, t, std, zero_rows=None):
        _, M, K = MATS[t]
        _, q, s, z = draw(self.qa.fmt, M, K, std, self.g, zero_rows)
        return self.write(t, q, s, z)

    def write(self, t, q, s, z):
        """Pack (q, s, z) into matrix t of layer l: (float64 W, {name: alternative W}, (q, s, z))."""
        fmt = self.qa.fmt
        if fmt == "int4":
            blob = Q.pack_matrix(q, s, z)
        else:
            blob = (Q.pack_int8_matrix if fmt == "int8" else Q.pack_fp8_matrix)(q, s)
        self.qa.put(self.l, t, blob)
        self.written.add(t)
        alt = {}
        if self.sens:
            os_, oz = self.qa.zero[(self.l - 1 if self.l > 0 else 1, t)]
            alt["layer l* - 1's scales (layer 1's at l* = 0)"] = reference_weight(fmt, q, os_, oz).cuda()
            alt["each row's (int4: group's) scale from its neighbour"] = reference_weight(
                fmt, q, torch.roll(s, 1, dims=s.dim() - 1), z).cuda()
            if fmt == "int4":
                alt["the zero point dropped"] = reference_weight(fmt, q, s, torch.zeros_like(z)).cuda()
        return reference_weight(fmt, q, s, z).cuda(), alt, (q, s, z)

    def gain(self, which, val):
        t = self.qa.gain(self.l, which)
        t.copy_(val)
        self.gains.append(t)
        return t

    def clear(self):
        for t in self.written:
            self.qa.put(self.l, t, self.qa.zero_blob(self.l, t))
        for t in self.gains:
            t.zero_()
        torch.cuda.synchronize()


def _gain(g):
    return (1 + 0.1 * torch.randn(D, generator=g, device="cuda")).to(torch.bfloat16)


POS = dl.POS
W1_TARGETS = dl.W1_TARGETS


def kv_check(tally, e, body, label, kv_got, y, A, alts=None):
    """appended k / v against the QKV reference y [R, 3D] (and the sensitivity references alts: name -> y_alt)."""
    for i, got in enumerate(kv_got):
        sl = slice((i + 1) * D, (i + 2) * D)
        ref = y[:, sl]
        b = lin_bound(e.fmt, body, 1, ref, A[:, sl], True, e.n_sm)
        nw_ref, lim = None, dl.NORMWISE
        if e.kv == "bf16":
            b = b + dl.BF16_U * (ref.abs() + b)
            nw_ref, lim = ref.to(torch.bfloat16).double(), dl.NORMWISE_BF16
        tally.check(f"{body} qkv kv={e.kv}", f"{label} {'kv'[i]}", got, ref, b, nw_ref=nw_ref, nw_limit=lim)
        for name, ya in (alts or {}).items():
            tally.over(name, got, ya[:, sl], b)


def run_probe(qa, e, probe, l, ns, tally):
    """One probe at target layer l for the batch sizes ns on engine e."""
    fmt = qa.fmt
    sens = l == 12
    case = Case(qa, l, seed=1000 * l + 17 * ["qkv", "wo", "ffn", "mixed"].index(probe) + FMTS.index(fmt), sens=sens)
    mask = (~qa.pil_d).double()
    try:
        g1 = case.gain("ln_1", _gain(case.gd)) if probe != "ffn" else None
        if probe in ("qkv", "wo", "mixed"):
            zr = torch.arange(D) if probe == "mixed" else None          # W_q = 0: every score exactly 0
            Wqkv, alt_qkv, _ = case.mat(1, D ** -0.5, zero_rows=zr)
        if probe in ("wo", "mixed"):
            Wo, alt_o, _ = case.mat(2, D ** -0.5, zero_rows=torch.arange(dl.PILOT, D, 128))
        if probe == "ffn":
            g2 = case.gain("ln_2", _gain(case.gd))
            # w1 rows scaled (through their scales) so that rs g of utterance 0's conditioned row is near the targets
            W1, _, (q, s, z) = case.mat(4, D ** -0.5)
            x0 = rows_x(qa, 1, qa.toks[0], POS)[:1]
            nh0, _, s0 = dl.operand(x0, g2, "A")
            rows = torch.tensor(list(W1_TARGETS))
            f = torch.ones(F, dtype=torch.float64)
            f[rows] = (torch.tensor(list(W1_TARGETS.values()), dtype=torch.float64) /
                       (nh0 @ W1[rows.cuda()].t() * s0)[0].cpu())
            fs = f[:, None] if s.dim() == 2 else f
            s = (s.double() * fs).float().to(torch.bfloat16)
            z = None if z is None else (z.double() * f[:, None]).float().to(torch.bfloat16)
            W1, alt_1, q1 = case.write(4, q, s, z)
            W3, alt_3, q3 = case.mat(5, D ** -0.5)
            W2, alt_2, _ = case.mat(6, F ** -0.5, zero_rows=torch.arange(dl.PILOT, D, 128))
            if sens:   # (b): w1's scales (and zero points) on w3's codes
                alt_3["w1's scales on w3"] = reference_weight(fmt, q3[0], q1[1], q1[2]).cuda()
        torch.cuda.synchronize()
        for n in ns:
            body = e.body(n)
            label = f"{fmt} {probe} l*={l} n={n} body {body} kv {e.kv}"
            if probe == "mixed":
                _run_mixed(qa, e, case, label, n, g1, Wqkv, Wo, mask, tally)
                continue
            e.m._kv.zero_()
            poss = [0] * n if probe == "wo" else POS[:n]
            toks = qa.toks[0][:n]
            x = rows_x(qa, n, toks, poss)
            lg = step(e, n, toks, poss)
            check_cache_rest(e, l, [(u, poss[u]) for u in range(n)])
            if probe in ("qkv", "wo"):
                nh, _, s = dl.operand(x, g1, body)
                y, A = dl.linear(Wqkv, nh, s)
                kv_got = appended(e, n, poss, l)
                alts = {}
                if sens and probe == "qkv":
                    alts = {k: dl.linear(W, nh, s)[0] for k, W in alt_qkv.items()}
                    if body == "B":
                        alts["layer l* - 1's codes (stale widen)"] = torch.zeros_like(y)
                    if fmt == "fp8" and n >= 5:
                        sw = nh.clone()
                        sw[[0, 1]] = nh[[1, 0]]
                        alts["slot 0's CFG rows swapped"] = dl.linear(Wqkv, sw, s)[0]
                kv_check(tally, e, body, label, kv_got, y, A, alts)
                if probe == "wo":
                    v = kv_got[1]
                    op = v if (body == "A" and fmt != "fp8") else dl.hilo(v.float())[0]
                    yo, Ao = dl.linear(Wo, op, 1.0)
                    b = lin_bound(fmt, body, 2, yo, Ao, False, e.n_sm) + (dl.n_split(body, "o", e.n_sm) + 1) * U * x.abs()
                    yh = dl.recover(qa, lg, x)
                    bo = b + tau_obs(fmt, body) * (x.abs() + yo.abs() + b)
                    tally.check(f"{body} wo", label + " y", yh, yo, bo, mask)
                    if sens:
                        for k, W in alt_o.items():
                            tally.over(k, yh, dl.linear(W, op, 1.0)[0], bo, mask)
            else:   # ffn
                yh = dl.recover(qa, lg, x)
                yr, b = ffn_ref(fmt, body, x, g2, W1, W3, W2, e.n_sm)
                bo = b + tau_obs(fmt, body) * (x.abs() + yr.abs() + b)
                tally.check(f"{body} ffn", label + " y", yh, yr, bo, mask)
                if sens:
                    for k, W in alt_1.items():
                        tally.over(f"w1: {k}", yh, ffn_ref(fmt, body, x, g2, W, W3, W2, e.n_sm)[0], bo, mask)
                    for k, W in alt_3.items():
                        tally.over(f"w3: {k}", yh, ffn_ref(fmt, body, x, g2, W1, W, W2, e.n_sm)[0], bo, mask)
                    for k, W in alt_2.items():
                        tally.over(f"w2: {k}", yh, ffn_ref(fmt, body, x, g2, W1, W3, W, e.n_sm)[0], bo, mask)
    finally:
        case.clear()


def _run_mixed(qa, e, case, label, n, g1, Wqkv, Wo, mask, tally):
    """Probe 5 of test_decode_linear_ops_gpu.py: K / V injected below p_u, NaN above, launches at p_u, p_u + 1, p_u + 2."""
    body, l, fmt = e.body(n), case.l, qa.fmt
    gi = torch.Generator(device="cuda").manual_seed(n + 7 * l)
    e.m._kv.zero_()
    base = dl.MIXED[:n]
    lay = e.cache[l]
    poison = torch.full((BLOCK, 128), float("nan"), dtype=e.dt, device="cuda")
    for u in range(n):
        for cr in (2 * u, 2 * u + 1):
            lay[:, cr] = poison
            p = base[u]
            lay[0, cr, :, :p] = (torch.randn(H, p, 128, generator=gi, device="cuda") * 0.7).to(e.dt)
            lay[1, cr, :, :p] = torch.randn(H, p, 128, generator=gi, device="cuda").to(e.dt)
    ns = SimpleNamespace(body=body, kv=e.kv)
    for it in range(3):
        poss = [p + it for p in base]
        toks = qa.toks[it][:n]
        x = rows_x(qa, n, toks, poss)
        before = lay.clone()
        lg = step(e, n, toks, poss)
        check_cache_rest(e, l, [(u, poss[u]) for u in range(n)], before)
        nh, _, s = dl.operand(x, g1, body)
        y, A = dl.linear(Wqkv, nh, s)
        kv_check(tally, e, body, f"{label} launch {it}", appended(e, n, poss, l), y, A)
        mean, em = [], []
        for u in range(n):
            L = poss[u] + 1
            for c in range(2):
                Vr = lay[1, 2 * u + c, :, :L].double()
                mean.append(Vr.mean(1).reshape(D))
                em.append(dl._att_eps(ns, L) * Vr.abs().mean(1).reshape(D))
        m, em = torch.stack(mean), torch.stack(em)
        hilo_op = body == "B" or fmt == "fp8"
        eop = em + (dl.HILO * (m.abs() + em) if hilo_op else 0.0)
        yo = m @ Wo.t()
        b = (lin_bound(fmt, body, 2, yo, (m.abs() + eop) @ Wo.abs().t(), False, e.n_sm) + eop @ Wo.abs().t()
             + (dl.n_split(body, "o", e.n_sm) + 1) * U * x.abs())
        yh = dl.recover(qa, lg, x)
        tally.check(f"{body} mixed", f"{label} launch {it} y", yh, yo, b + tau_obs(fmt, body) * (x.abs() + yo.abs() + b), mask)


def run_head(qa, e_get, ns, tally):
    """Probe 4: random ln_f gain and lm_head (every layer zero), all V logits.  int4: lm_head is bf16."""
    fmt = qa.fmt
    g = torch.Generator().manual_seed(404 + FMTS.index(fmt))
    gd = torch.Generator(device="cuda").manual_seed(405)
    gf = qa.bf16_global("transformer.ln_f.weight", (D,))
    o = qa.off("lm_heads.0.weight")
    if fmt == "int4":
        Wh = (torch.randn(V, D, generator=g) * D ** -0.5).to(torch.bfloat16)
        blob = Wh.view(torch.uint8).flatten()
        W, alts = Wh.double().cuda(), {}
    else:
        blob, q, s, _ = draw(fmt, V, D, D ** -0.5, g)
        W = reference_weight(fmt, q, s).cuda()
        alts = {"each row's scale from its neighbour": reference_weight(fmt, q, torch.roll(s, 1)).cuda()}
    keep = qa.buf[o:o + blob.numel()].clone()
    try:
        gf.copy_(_gain(gd))
        qa.buf[o:o + blob.numel()].copy_(blob.cuda())
        torch.cuda.synchronize()
        for n in ns:
            e = e_get(n)
            body = e.body(n)
            label = f"{fmt} head n={n} body {body}"
            e.m._kv.zero_()
            toks = qa.toks[0][:n]
            x = rows_x(qa, n, toks, POS[:n])
            lg = step(e, n, toks, POS[:n])
            check_cache_rest(e, 0, [])
            nh, _, s_ = dl.operand(x, gf, body)
            y, A = dl.linear(W, nh, s_)
            if fmt == "int4" and body == "A":       # lm_head through the bf16 k_gemv
                b = dl.lin_bound("A", "head", y, A)
            else:
                b = lin_bound(fmt, body, "head", y, A, True, e.n_sm)
            tally.check(f"{body} head", label, lg, y, b)
            for k, Wa in alts.items():
                tally.over(f"head: {k}", lg, dl.linear(Wa, nh, s_)[0], b)
            tail = torch.zeros_like(y)
            tail[:, V - 2:] = 1
            Wsh = W.clone()
            Wsh[V - 2:] = W[V - 2 - 128:V - 128]
            tally.over("ragged head tile shifted by 128 rows", lg, dl.linear(Wsh, nh, s_)[0], b, tail)
    finally:
        gf.fill_(1.0)
        qa.buf[o:o + blob.numel()].copy_(keep)
        torch.cuda.synchronize()


def run_prefill(qa, e, l, tally):
    """QKV probe through mvb_s1_forward at T = 70 from position 100 (two 64-token chunks on path B): k and v of every
    position against float64 with the path-B operand and bound."""
    from mvb200 import _lib
    fmt = qa.fmt
    case = Case(qa, l, seed=5000 + 10 * l + FMTS.index(fmt), sens=l == 12)
    T, p0, utt = PREFILL_T, PREFILL_P0, 1
    try:
        g1 = case.gain("ln_1", _gain(case.gd))
        Wqkv, alt, _ = case.mat(1, D ** -0.5)
        torch.cuda.synchronize()
        e.m._kv.zero_()
        gi = torch.Generator().manual_seed(l)
        idx = torch.randint(0, V, (2, T), generator=gi, dtype=torch.int32)
        e.m.set_speaker(utt, qa.spks[utt])
        d_idx = idx.cuda()
        lg = torch.full((2, V), float("nan"), device="cuda")
        _lib.check(e.m._lib.mvb_s1_forward(e.m.handle, utt, d_idx.data_ptr(), T, p0, lg.data_ptr(), 0, e.m._stream()))
        torch.cuda.synchronize()
        assert not torch.isnan(lg).any()
        check_cache_rest(e, l, [(utt, slice(p0, p0 + T))])
        x = qa.tok_d[idx.flatten().long().cuda()] + qa.pos_d[torch.arange(p0, p0 + T).repeat(2).cuda()]
        x[:T] += qa.spks[utt].double() @ qa.wspk_d.t()
        nh, _, s = dl.operand(x, g1, "B")
        y, A = dl.linear(Wqkv, nh, s)
        ks = torch.cat([e.cache[l, 0, 2 * utt + c, :, p0:p0 + T].permute(1, 0, 2).reshape(T, D) for c in range(2)]).double()
        vs = torch.cat([e.cache[l, 1, 2 * utt + c, :, p0:p0 + T].permute(1, 0, 2).reshape(T, D) for c in range(2)]).double()
        alts = {k: dl.linear(W, nh, s)[0] for k, W in alt.items()}
        if l > 0:
            alts["layer l* - 1's codes (stale widen)"] = torch.zeros_like(y)
        kv_check(tally, e, "B", f"{fmt} prefill T={T} l*={l} kv {e.kv}", (ks, vs), y, A, alts)
    finally:
        case.clear()


# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def arenas():
    cur = {}

    def get(fmt):
        if fmt not in cur:
            cur.clear()
            torch.cuda.empty_cache()
            cur[fmt] = QArena(fmt)
        return cur[fmt]
    yield get
    cur.clear()
    torch.cuda.empty_cache()


def _ns(fmt):
    return PATH_A_N + (PATH_B_N if fmt == "fp8" else ())


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
def test_quant_decode_projections(arenas, fmt):
    """qkv, wo, FFN and mixed-position probes at l* = 0, 12, 23 (fp32 cache), the qkv probe with a bf16 cache, and the head,
    on path A (and fp8's path B at 9 and 12 slots)."""
    qa = arenas(fmt)
    ns = _ns(fmt)
    tally = Tally()
    e = QEngine(qa, "fp32", max(ns))
    try:
        for probe in ("qkv", "wo", "ffn", "mixed"):
            for l in LSTAR:
                run_probe(qa, e, probe, l, ns, tally)
        run_head(qa, lambda n: e, PATH_A_N, tally)
    finally:
        e.close()
    if fmt == "fp8":      # path B's head reads lm_head's q widened at create: run_head creates this engine after writing it
        holder = {}

        def e_get(n):
            if "e" not in holder:
                holder["e"] = QEngine(qa, "fp32", max(PATH_B_N))
            return holder["e"]
        try:
            run_head(qa, e_get, PATH_B_N, tally)
        finally:
            if "e" in holder:
                holder["e"].close()
    eb = QEngine(qa, "bf16", max(ns))
    try:
        for l in LSTAR:
            run_probe(qa, eb, "qkv", l, ns, tally)
    finally:
        eb.close()
    tally.report(f"{fmt} decode")
    print(f"  peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
def test_quant_prefill_path_b(arenas, fmt):
    """Prefill of T = 70 through path B (the per-layer widen / dequantise and k_tc_gemm with row scales) at l* = 0, 12,
    23, with an fp32 and a bf16 cache."""
    qa = arenas(fmt)
    tally = Tally()
    for kv in ("fp32", "bf16"):
        e = QEngine(qa, kv, 2)
        try:
            for l in LSTAR:
                run_prefill(qa, e, l, tally)
        finally:
            e.close()
    tally.report(f"{fmt} prefill")
