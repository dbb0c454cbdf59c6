"""GPU: the weight-streaming projections of one stage-1 decode step at production width (metavoice-1B: D = 2048, H = 16,
F = 5632, V = 2562, 24 layers) against a float64 computation that reproduces every rounding the kernels declare: every
phase of the persistent kernel (path C, all four <kv, NB> instances), the bf16 k_gemv of path A and the tensor-core
rows path B (k_prep_b, the QKV scatter, the SwiGLU instance, the head over V = 2562 with its ragged last tile).

PROBE MODEL.  The engine runs unchanged (mvb_s1_begin + mvb_s1_step_logits) on ONE all-zero bf16 arena packed by
pack_arena; every case writes its random tensors into the arena slices in place and zeroes them afterwards (path A / B
replay graphs that read the arena, path C's tensor maps point into it: no engine keeps a derived copy of a weight).
block_size = 256 keeps the KV cache under 2 GB.  Embeddings sit on a 1/32 grid (tok +-12, pos +-4, speaker +-4, |x| <=
20/32): x is exact in fp32 and every fp32 sum of squares of x is exact in any order, so the only difference left in an
RMSNorm scale is rsqrtf (2 ulp).  The speaker projection W_spk is 0.5 x a selection matrix and spk sits on the grid:
k_spk_proj is exact and the two CFG rows differ.  Every utterance has its own token, speaker and position.  Every layer
except the target l* in {0, 12, 23} is zero and adds exactly 0 to x (q = k = v = 0, attention output 0, g = u = 0,
silu(0) 0 = 0), so l* = 0 covers the operand staged straight from the embedding tables, l* = 12, 23 the layer stride
and the stat[2l] / stat[2l + 1] slots.  Probes (one phase random, observed):
  1 QKV: random ln_1 gain, W_qkv ~ N(0, 1/D).  k and v are read back from the cache at the current position; every
    other cache entry must be unchanged.  q is not observable at L = 1 (a single weight exp(0) = 1 whatever the score);
    the attention tests cover q through selection matrices.
  2 wo + residual: probe 1's QKV, wo ~ N(0, 1/D) with its PILOT rows (output dims h 128 + 127) zero, zero FFN,
    ln_f = 1, lm_head = [I_D; 0], position 0.  At L = 1 the attention output is exactly the read-back v in every path
    (one weight exp(0) = 1, running sum 1, the merge divides by 1; the fp32-cache loop multiplies v by pw = 1, the
    mma form by pc = 1 after rounding v to bf16 as stored).  Then logits[:D] = RMSNorm(x + wo v): the pilot logits
    give the kernel's own final scale r^ = mean(l / x) over the pilots (y = 0 there exactly) and y^ = l / r^ - x.
  3 FFN: wo = 0, random ln_2 gain, w1, w3 ~ N(0, 1/D), w2 ~ N(0, 1/F) with zero pilot rows; observed as in probe 2.
    Nine rows of w1 are rescaled so that rs g of utterance 0's conditioned row is -95 .. 90: the __expf overflow ->
    __fdividef = 0 corner and the growth of __expf's error with |g|.
  4 head: every layer zero, random ln_f gain, lm_head ~ N(0, 1/D) [V x D]; all 2562 logits observed, with the two
    rows of the ragged last row tile; rows of the caller's logits buffer outside the batch must stay untouched.
  5 mixed positions, three launches: probe 2 with W_q = 0 (every score exactly 0: attention is the mean of the L
    V rows).  Each utterance has its own position p_u; K / V are injected at [0, p_u), poison above (NaN; finite for
    the mma form, which reads whole 64-position boxes), and step_logits runs at p_u, p_u + 1, p_u + 2 (pos_emb rows,
    the multi-split merge of the wo staging, the launch-time zeroing of logits / stat / qkv / gu across launches).
    At H = 16 the persistent kernel cuts a row into at most floor(132 / (2 x 16)) = 4 splits, so the wo staging's
    nch > 4 branch is unreachable at production width; the attention tests cover it at H = 2.

OPERAND as staged (float64 of the exact fp32 / bf16 values; hilo(v) = bf16(v) + bf16(v - bf16(v))):
  path C  n^ = hilo(x g)  (x g is exact: a 5-bit times an 8-bit significand), the projection is scaled by rs after
          accumulation: y = fl(acc rs) (k, v, the head logits), g = fl(G rs) and u = fl(U rs) before the SiLU;
  path B  n^ = hilo(fl(fl(x rs) g)) (k_prep_b), no scale after;  path A  n^ = fl(fl(x rs) g) in fp32 (k_gemv).
rs = rsqrt(fl(ss / D + eps)) of the exact sum of squares; the reference takes path C's rs exactly in float64, and for
paths A / B torch's fp32 rsqrt of the same argument.

ELEMENTWISE BOUND.  For y = s W n^ (s = rs on path C, else 1) and A = s |W| |n^|:
    |y^ - y| <= (gamma + tau) A + 2 u |y|,      u = 2^-23,
  gamma (paths B, C) = (18 * 4 * 2 * ceil(KB / S) + S + 1) u: the m16n8k16 model of test_gemm_ops_gpu.py (each MMA
    moves the exact value by <= 18 u (|c| + sum |p|), 4 MMAs per 64-wide k-block for hi and again for lo).  Every split
    starts its accumulator at 0 and runs at most ceil(KB / S) of the KB = K / 64 k-blocks (pc_slice, k_tc_gemm), so its
    partial is off by <= 18 u 8 ceil(KB / S) times the sum of its |products|; summed over the splits that is the first
    term times A.  The S fp32 partials are then added (path C: red.add, S from a mirror of plan_pc on this device's SM
    count; path B: the split-K reduction, S from a mirror of plan_gemm), + 1 for the add onto the residual;
  gamma (path A) = (K / 32 + 5 + 1) u: one fma chain of K / 32 terms per lane, a 5-step butterfly, the residual add;
  tau: path C 2^-21 (rsqrtf's 2 ulp and the rounding of the rs product), path B 2^-20 + 2^-16 (the kernel's and the
    reference's fp32 rsqrt differ by <= 4 ulp, which moves v by 2^-21 and can flip lo by one bf16 ulp <= 2^-16 |v|),
    path A 2^-20 (the same rs difference through two fp32 products).
  A bf16 cache stores fl_bf16(y): + 2^-8 (|y| + bound) (the bf16 unit roundoff; one rounding).
Residual phases (wo, w2) add (S + 1) u |x| for the adds onto x.
FFN (a running error bound): e_g = (gamma_13 + tau) A_g + 2^-21 |g| (the rs product on path C), e_u alike;
    h = silu(g) u,  e_h = 1.1 e_g |u| + |silu(g)| e_u + 1.1 e_g e_u + (eps_s + u) |h| + [g < -80] |h|,
    eps_s = (2 + floor(1.17 |g|) + 4) u: __expf (2 + floor(1.17 |x|) ulp; only its share e / (1 + e) reaches the
    quotient), the 1 + e add, __fdividef (2 ulp) and the product with u; |silu'| <= 1.1; __fdividef returns 0 once the
    denominator passes 2^126 (g < -87.3) and so does IEEE division by expf's inf on paths A / B: there the reference's
    |h| < 1e-35 |u| counts in full.  Paths B, C restage h as hilo: + 2^-16 (|h| + e_h).  Then
    |y^ - y| <= gamma_2 |W2| (|h| + e_h) + |W2| e_h + (S + 1) u |x|.
Mixed positions: the mean of the L V rows is off by <= eps |mean|V||, the attention tests' eps at s = 0,
    eps = 2.02 * 2^-21 (n_resc + 3) + 2.02 rho_p + 2 n_acc u (n_resc, n_acc, rho_p per body as in
    test_attention_ops_gpu.py), and enters wo like e_h enters w2.
OBSERVATION (probes 2, 3, 5): the final RMSNorm and the [I; 0] head through the pilots add tau_obs (|x| + |y| + bound),
    tau_obs = 2^-15 for paths B, C and 2^-20 for path A (the derivation of test_attention_ops_gpu.py).
NORMWISE: ||y^ - y|| / ||y|| < 1e-4 for every observed vector; k, v in a bf16 cache against the reference rounded to
    bf16, < 1e-3 (a 1e-5-accurate value rounds to the other neighbour in a fraction ~1e-5 / 2^-8 of the elements).

SENSITIVITY: references that (a) drop the lo term of the head operand (paths B, C; two head rows, in the first and the
ragged last tile, have the signs of utterance 0's lo terms, so the dropped terms add up), (b) leave out the k-blocks of
split 0 of the engine's plan for QKV, w2 and the head (path C), (c) apply rs to u but not to g before the SiLU, (d) use
ln_1's gain where ln_2 belongs (in the FFN probe ln_1 is drawn from U(0.25, 1.75): with W_qkv = 0 the kernel does not
read it, and a gain within 10 % of ln_2 would hide under the FFN bound, which carries the w1 / w3 error through all
F = 5632 columns of w2 in absolute value), (e) read the two rows of the ragged last head tile one tile (128 rows) lower, must each
put elements over the bound of the true reference."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
D, H, F, V, NL = 2048, 16, 5632, 2562, 24
BLOCK = 256
SPK = 256
PILOT = 127
EPS = 1e-5
TAU = {"A": 2.0 ** -20, "B": 2.0 ** -20 + 2.0 ** -16, "C": 2.0 ** -21}
TAU_OBS = {"A": 2.0 ** -20, "B": 2.0 ** -15, "C": 2.0 ** -15}
HILO = 2.0 ** -16
BF16_U = 2.0 ** -8
NORMWISE = 1e-4
NORMWISE_BF16 = 1e-3
LSTAR = (0, 12, 23)
SENS_L = 12

# form -> kv dtype, tensor_core_path of setup_caches, body it must run, utterance counts
FORMS = {
    "C-fp32": ("fp32", None, "C", (1, 4, 5, 8)),     # <fp32, 16> at 1 and 4 utterances, <fp32, 32> at 5 and 8
    "C-bf16": ("bf16", None, "C", (1, 4, 5, 8)),     # the mma.sync attention form, <bf16, 16> / <bf16, 32>
    "A": ("fp32", "", "A", (1, 3)),
    "B": ("bf16", "B", "B", (2, 8, 9, 16)),
}
# kernel launches of one mvb_s1_step_logits (k_identity_slots included) for the 24-layer model:
# A (launch_body): embed + 5 per layer (QKV, attention, wo, w1|w3, w2) + head;
# B (launch_body_b): k_rows_decode + embed + per layer 4 linears x (k_prep_b + k_tc_gemm) + attention, + head (2);
# C: launch_persistent counts the persistent kernel once
LAUNCHES = {"A": 1 + 1 + 5 * NL + 1, "B": 1 + 1 + 1 + 9 * NL + 2, "C": 1 + 1}
PROBES = ["qkv", "wo", "ffn", "head", "mixed"]
POS = [17, 0, 255, 100, 64, 31, 200, 128, 3, 77, 190, 45, 250, 9, 160, 222]          # probes 1, 3, 4
MIXED = [200, 3, 63, 130, 31, 97, 253, 64, 1, 128, 190, 45, 222, 9, 160, 0]        # probe 5: p_u (+ 0, 1, 2)
W1_TARGETS = {5: -95.0, 700: -90.0, 1400: -88.6, 2100: -87.9, 2800: -60.0, 3500: -20.0, 4200: 20.0, 4900: 60.0,
              5600: 90.0}
MATS = {"qkv": (3 * D, D), "o": (D, D), "w13": (2 * F, D), "w2": (D, F), "head": (V, D)}


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def plan_pc(M, K, ctas, tile_rows=128):
    """Mirror of plan_pc (stage1_engine.cu): the K split count of one matrix in the persistent kernel."""
    T, KB = -(-M // tile_rows), K // 64
    best = None
    for S in range(1, min(KB, 32, ctas) + 1):
        tiles_per, kb_per = -(-T // (ctas // S)), -(-KB // S)
        if kb_per > 12:
            continue
        cost = tiles_per * (2 * kb_per + 5) + 4 * kb_per
        if best is None or cost < best[0]:
            best = (cost, S)
    return best[1] if best else 0     # 0: no split fits (the host then declines path C)


def plan_gemm_ksplit(M, K, n_sm):
    """Mirror of plan_gemm's automatic K split (tc_gemm_host.cuh) for path B."""
    tiles, nkb = -(-M // 128), K // 64
    ks = max(1, min(n_sm, 132) // tiles)
    if ks > nkb // 2:
        ks = max(1, nkb // 2)
    if nkb <= 8 or tiles > 128:
        ks = 1
    return min(ks, 16)


def n_split(body, mat, n_sm=None):
    """K splits whose fp32 partials are added for one output element (0 on path A), planned for n_sm SMs (default:
    this device's count)."""
    M, K = MATS[mat]
    n_sm = n_sm or _n_sm()
    if body == "C":
        return plan_pc(M, K, n_sm)
    if body == "B":
        return plan_gemm_ksplit(M // 2 if mat == "w13" else M, K, n_sm)   # the SwiGLU instance tiles w1 and w3 together
    return 0


def gamma(body, mat, n_sm=None):
    """gamma of the module docstring: MMAs of the longest split (ceil(KB / S) k-blocks, hi and lo) + the split adds + 1."""
    K = MATS[mat][1]
    if body == "A":
        return (K / 32 + 5 + 1) * U
    S = n_split(body, mat, n_sm)
    return (18 * 4 * 2 * -(-(K // 64) // S) + S + 1) * U


def split0_cols(mat, n_sm=None):
    """The columns of split 0 of path C's plan (pc_slice: kb1 = KB / S for split 0)."""
    M, K = MATS[mat]
    return 64 * ((K // 64) // plan_pc(M, K, n_sm or _n_sm()))


# ---------------------------------------------------------------------------------------------------------------------
class Arena:
    """One all-zero bf16 arena (pack_arena) with a view of every tensor, plus the static embedding tables."""

    def __init__(self):
        from mvb200.fast_model import _GLOBAL_KEYS, _LAYER_KEYS, pack_arena
        shapes = {"transformer.wtes.0.weight": (V, D), "transformer.wpe.weight": (BLOCK, D),
                  "speaker_cond_pos.weight": (D, SPK), "transformer.ln_f.weight": (D,), "lm_heads.0.weight": (V, D)}
        lshapes = {"ln_1.weight": (D,), "attn.c_attn.weight": (3 * D, D), "attn.c_proj.weight": (D, D),
                   "ln_2.weight": (D,), "mlp.swiglu.w1.weight": (F, D), "mlp.swiglu.w3.weight": (F, D),
                   "mlp.c_proj.weight": (D, F)}
        for i in range(NL):
            shapes.update({f"transformer.h.{i}.{k}": s for k, s in lshapes.items()})
        zero = torch.zeros((), dtype=torch.bfloat16)
        arena, self.offsets = pack_arena({k: zero.expand(*s) for k, s in shapes.items()}, NL)
        self.buf = arena.cuda()
        keys = list(_GLOBAL_KEYS) + [f"transformer.h.{i}.{k}" for i in range(NL) for k in _LAYER_KEYS]
        self.t = {}
        for k, o in zip(keys, self.offsets):
            s = shapes[k]
            self.t[k] = self.buf[o:o + 2 * math.prod(s)].view(torch.bfloat16).view(*s)
        g = torch.Generator().manual_seed(0)
        self.pil = torch.zeros(D, dtype=torch.bool)
        self.pil[PILOT::128] = True
        tok = torch.randint(-12, 13, (V, D), generator=g).float()
        mag = torch.randint(12, 21, (V, int(self.pil.sum())), generator=g).float()
        tok[:, self.pil] = mag * (torch.randint(0, 2, mag.shape, generator=g) * 2 - 1)
        pos = torch.randint(-4, 5, (BLOCK, D), generator=g).float()
        pos[:, self.pil] = 0
        wspk = torch.zeros(D, SPK)
        wspk[torch.arange(D), torch.arange(D) % SPK] = 0.5
        wspk[self.pil] = 0
        self.t["transformer.wtes.0.weight"].copy_(tok / 32)
        self.t["transformer.wpe.weight"].copy_(pos / 32)
        self.t["speaker_cond_pos.weight"].copy_(wspk)
        self.tok_d, self.pos_d, self.wspk_d = (tok / 32).double().cuda(), (pos / 32).double().cuda(), wspk.double().cuda()
        self.pil_d = self.pil.cuda()
        # utterance u: token TOKS[u], speaker embedding SPKS[u] (1/32 grid, |.| <= 8/32: projection |.| <= 4/32)
        self.toks = torch.randperm(V, generator=g)[:3 * 16].view(3, 16).tolist()     # [launch][utterance]
        self.spks = (torch.randint(-8, 9, (16, SPK), generator=g).float() / 32).cuda()

    def lw(self, l, name):
        return self.t[f"transformer.h.{l}.{name}"]


class Engine:
    def __init__(self, arena, form, n_sm=None):
        """n_sm: the SM count the engine is planned for (default: this device's)."""
        from mvb200.fast_model import ModelArgs, Transformer
        self.form, self.n_sm = form, n_sm or _n_sm()
        self.kv, tc, self.body, self.utts = FORMS[form]
        cfg = ModelArgs(block_size=BLOCK, vocab_size=V, n_layer=NL, n_head=H, dim=D, intermediate_size=F)
        self.m = Transformer(cfg, arena.buf, arena.offsets, device="cuda:0")
        self.m.setup_caches(2 * max(self.utts), BLOCK, kv_dtype=self.kv, tensor_core_path=tc)
        self.dt = torch.float32 if self.kv == "fp32" else torch.bfloat16
        self.cache = self.m._kv.view(self.dt).view(NL, 2, 2 * max(self.utts), H, BLOCK, 128)
        for u in range(max(self.utts)):
            self.m.set_speaker(u, arena.spks[u])
        torch.cuda.synchronize()

    def close(self):
        self.m.close()


def launches(e):
    return int(e.m._lib.mvb_s1_launch_count(e.m.handle))


def step(e, n, toks, poss):
    """begin every utterance at its (token, position), one mvb_s1_step_logits; returns logits [2 n, V]."""
    from mvb200 import _lib
    lib, h, st = e.m._lib, e.m.handle, e.m._stream()
    sp = _lib.Sampling(1.0, 1.0, 0.0, 0, 9999, 1)
    for u in range(n):
        _lib.check(lib.mvb_s1_begin(h, u, int(toks[u]), int(poss[u]), C.byref(sp), None, None, st))
    n0 = launches(e)
    lg = torch.full((2 * n + 3, V), float("nan"), device="cuda")
    _lib.check(lib.mvb_s1_step_logits(h, n, lg.data_ptr(), st))
    torch.cuda.synchronize()
    assert launches(e) - n0 == LAUNCHES[e.body], f"{e.form} n={n}: body {e.body} did not run"
    assert torch.isnan(lg[2 * n:]).all(), f"{e.form} n={n}: logits rows outside the batch were written"
    return lg[:2 * n].double()


def rows_x(a, n, toks, poss):
    """float64 x [2 n, D] of the batch: tok_emb + pos_emb (+ speaker projection on the conditioned row)."""
    x = a.tok_d[torch.tensor(toks[:n]).repeat_interleave(2).cuda()] + a.pos_d[torch.tensor(poss[:n]).repeat_interleave(2).cuda()]
    x[0::2] += a.spks[:n].double() @ a.wspk_d.t()
    return x


def hilo(v):
    hi = v.to(torch.bfloat16).float()
    lo = (v - hi).to(torch.bfloat16).float()
    return hi.double() + lo.double(), hi.double()


def operand(x, gain, body):
    """(n^, its hi term, scale s [R, 1]) of the RMSNorm-gained operand as the body stages it (module docstring)."""
    x32, g32 = x.float(), gain.float()
    arg = (x * x).sum(-1, keepdim=True).float() / D + EPS          # exact sum of squares, fp32 argument
    if body == "C":
        full, hi = hilo(x32 * g32)
        return full, hi, torch.rsqrt(arg.double())
    v = (x32 * torch.rsqrt(arg)) * g32
    one = torch.ones_like(arg, dtype=torch.float64)
    if body == "B":
        full, hi = hilo(v)
        return full, hi, one
    return v.double(), v.double(), one


def linear(W, nh, s):
    """y = s W n^ and A = s |W| |n^| (float64, rows of nh)."""
    return (nh @ W.t()) * s, (nh.abs() @ W.abs().t()) * s


def lin_bound(body, mat, y, A, n_sm=None):
    return (gamma(body, mat, n_sm) + TAU[body]) * A + 2 * U * y.abs() + 1e-30


def rs64(x):
    return torch.rsqrt(((x * x).sum(-1, keepdim=True).float() / D + EPS).double())


def recover(a, lg, x):
    """y^ from logits rows [R, V] and x [R, D] through the pilots (the kernel's own final RMSNorm scale)."""
    l = lg[:, :D]
    r = (l[:, PILOT::128] / x[:, PILOT::128]).mean(-1, keepdim=True)
    return l / r - x


def assess(label, got, ref, bound, mask=None, nw_ref=None, nw_limit=NORMWISE):
    """Elementwise bound and normwise error per row; returns (worst ratio, worst normwise)."""
    err = (got - ref).abs()
    if mask is not None:
        err = err * mask
    ratio = float((err / bound).max())
    bad = (err > bound).nonzero()
    assert bad.numel() == 0, (f"{label}: {bad.shape[0]} elements over the bound (max ratio {ratio:.2e}); first (row, column) "
                              f"{bad[0].tolist()}: got {float(got[tuple(bad[0])]):.9e}, want {float(ref[tuple(bad[0])]):.9e}, "
                              f"bound {float(bound[tuple(bad[0])]):.3e}")
    e2 = (got - (ref if nw_ref is None else nw_ref)).abs()
    if mask is not None:
        e2 = e2 * mask
    nw = float((e2.norm(dim=-1) / ref.norm(dim=-1).clamp_min(1e-30)).max())
    assert nw < nw_limit, f"{label}: normwise error {nw:.2e}"
    return ratio, nw


def n_over(got, alt, bound, mask=None):
    err = (got - alt).abs()
    if mask is not None:
        err = err * mask
    return int((err > bound).sum())


def check_cache_rest(e, n, poss, l, before=None):
    """Every cache entry other than the appended ones at (layer l, rows of the batch, their positions) is unchanged:
    zero layers hold zeros (their appended k = v = 0 included), layer l is byte-equal to `before` (or zero)."""
    for j in range(NL):
        if j != l:
            assert (e.cache[j] == 0).all(), f"{e.form}: zero layer {j} cache changed"
    cur = e.cache[l].clone()
    ref = before.clone() if before is not None else torch.zeros_like(cur)
    for u in range(n):
        cur[:, 2 * u:2 * u + 2, :, poss[u]] = 0
        ref[:, 2 * u:2 * u + 2, :, poss[u]] = 0
    assert torch.equal(cur.view(torch.uint8), ref.view(torch.uint8)), \
        f"{e.form}: layer {l} cache entries other than the appended ones changed"


def appended(e, n, poss, l):
    """k, v [2 n, D] appended by the step at each row's position (float64 of the stored values)."""
    ks, vs = [], []
    for u in range(n):
        for c in range(2):
            ks.append(e.cache[l, 0, 2 * u + c, :, poss[u]].reshape(D))
            vs.append(e.cache[l, 1, 2 * u + c, :, poss[u]].reshape(D))
    return torch.stack(ks).double(), torch.stack(vs).double()


def kv_bound(e, y, A, i):
    """reference and bound of the appended k (i = 0) or v (i = 1) from the QKV reference y, A [R, 3D]."""
    sl = slice((i + 1) * D, (i + 2) * D)
    ref, b = y[:, sl], lin_bound(e.body, "qkv", y[:, sl], A[:, sl], e.n_sm)
    if e.kv == "bf16":
        b = b + BF16_U * (ref.abs() + b)
    return ref, b


def check_kv(e, label, kv_got, y, A):
    """appended k / v against the QKV reference y [R, 3D]."""
    worst = nw = 0.0
    for i, got in enumerate(kv_got):
        ref, b = kv_bound(e, y, A, i)
        nw_ref, lim = None, NORMWISE
        if e.kv == "bf16":
            nw_ref, lim = ref.to(torch.bfloat16).double(), NORMWISE_BF16
        r, w = assess(f"{label} {'kv'[i]}", got, ref, b, nw_ref=nw_ref, nw_limit=lim)
        worst, nw = max(worst, r), max(nw, w)
    return worst, nw


def obs_bound(body, x, y, b):
    return b + TAU_OBS[body] * (x.abs() + y.abs() + b)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def arena():
    a = Arena()
    yield a
    del a.buf
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def engines(arena):
    cur = {}

    def get(form):
        if form not in cur:
            for k in list(cur):
                cur.pop(k).close()
            torch.cuda.empty_cache()
            cur[form] = Engine(arena, form)
        return cur[form]
    yield get
    for v in cur.values():
        v.close()


def _rand(shape, std, g):
    return torch.randn(*shape, generator=g, device="cuda") * std


def _gain(g):
    return (1 + 0.1 * torch.randn(D, generator=g, device="cuda")).to(torch.bfloat16)


class Case:
    """The random tensors one probe writes into the arena (bf16 in place; float64 copies for the reference)."""

    def __init__(self, a, l, seed):
        self.a, self.l, self.keys = a, l, []
        self.g = torch.Generator(device="cuda").manual_seed(seed)

    def put(self, key, val):
        t = self.a.t[key] if key in self.a.t else self.a.lw(self.l, key)
        t.copy_(val)
        self.keys.append(t)
        return t.double()

    def clear(self):
        for t in self.keys:
            t.zero_()
        torch.cuda.synchronize()


def _qkv(case, wq_zero=False):
    g1 = case.put("ln_1.weight", _gain(case.g))
    W = _rand((3 * D, D), D ** -0.5, case.g)
    if wq_zero:
        W[:D] = 0
    return g1, case.put("attn.c_attn.weight", W)


def _observe_head(case):
    case.put("transformer.ln_f.weight", torch.ones(D, device="cuda"))
    case.put("lm_heads.0.weight", torch.cat([torch.eye(D, device="cuda"), torch.zeros(V - D, D, device="cuda")]))


def _wo_pilot_zero(case, std, shape):
    W = _rand(shape, std, case.g)
    W[PILOT::128] = 0
    return W


def run_probe(a, e, probe, l):
    body, label0 = e.body, f"{e.form} {probe} l*={l}"
    case = Case(a, l, seed=1000 * l + PROBES.index(probe) * 17 + len(e.form))
    worst = nw = 0.0
    sens = {}
    mask = (~a.pil_d).double()
    try:
        if probe in ("qkv", "wo"):
            g1, Wqkv = _qkv(case)
            if probe == "wo":
                Wo = case.put("attn.c_proj.weight", _wo_pilot_zero(case, D ** -0.5, (D, D))).double()
                _observe_head(case)
        elif probe == "mixed":
            g1, Wqkv = _qkv(case, wq_zero=True)
            Wo = case.put("attn.c_proj.weight", _wo_pilot_zero(case, D ** -0.5, (D, D))).double()
            _observe_head(case)
        elif probe == "ffn":
            # not read by the kernel here (W_qkv = 0): the gain of the wrong-gain reference
            g1 = case.put("ln_1.weight", 0.25 + 1.5 * torch.rand(D, generator=case.g, device="cuda"))
            g2 = case.put("ln_2.weight", _gain(case.g))
            W1 = _rand((F, D), D ** -0.5, case.g).double()
            # rescale rows of w1 so that rs g of utterance 0's conditioned row hits the targets
            x0 = rows_x(a, 1, a.toks[0], POS)[:1]
            nh0, _, s0 = operand(x0, g2, body)
            rows = torch.tensor(list(W1_TARGETS), device="cuda")
            g0 = (nh0 @ W1[rows].t() * s0)[0]
            W1[rows] *= (torch.tensor(list(W1_TARGETS.values()), device="cuda", dtype=torch.float64) / g0)[:, None]
            W1 = case.put("mlp.swiglu.w1.weight", W1.float())
            W3 = case.put("mlp.swiglu.w3.weight", _rand((F, D), D ** -0.5, case.g))
            W2 = case.put("mlp.c_proj.weight", _wo_pilot_zero(case, F ** -0.5, (D, F)))
            _observe_head(case)
        else:   # head
            gf = case.put("transformer.ln_f.weight", _gain(case.g))
            Wh = _rand((V, D), D ** -0.5, case.g)
            # rows 0 and V - 1 (first / ragged last tile) carry the signs of utterance 0's lo terms
            x0 = rows_x(a, 1, a.toks[0], POS)[:1]
            nh0, hi0, _ = operand(x0, gf, body)
            sg = torch.sign(nh0 - hi0)[0].float()
            for j in (0, V - 1):
                Wh[j] = Wh[j].abs() * sg
            Wh = case.put("lm_heads.0.weight", Wh)
        torch.cuda.synchronize()

        for n in e.utts:
            sens_case = l == SENS_L and n == e.utts[0]
            label = f"{label0} n={n}"
            if probe == "mixed":
                r, w = _run_mixed(a, e, case, label, n, g1, Wqkv, Wo, mask, sens if sens_case else None)
                worst, nw = max(worst, r), max(nw, w)
                continue
            e.m._kv.zero_()
            poss = [0] * n if probe == "wo" else POS[:n]
            toks = a.toks[0][:n]
            x = rows_x(a, n, toks, poss)
            lg = step(e, n, toks, poss)
            if probe in ("qkv", "wo"):
                check_cache_rest(e, n, poss, l)
                nh, _, s = operand(x, g1, body)
                y, A = linear(Wqkv, nh, s)
                kv_got = appended(e, n, poss, l)
                r, w = check_kv(e, label, kv_got, y, A)
                worst, nw = max(worst, r), max(nw, w)
                if sens_case and body == "C" and probe == "qkv":
                    c = split0_cols("qkv", e.n_sm)
                    y_d = linear(Wqkv[:, c:], nh[:, c:], s)[0]
                    sens["qkv without split 0"] = sum(
                        n_over(kv_got[i], y_d[:, (i + 1) * D:(i + 2) * D], kv_bound(e, y, A, i)[1]) for i in range(2))
                if probe == "wo":
                    v = kv_got[1]
                    op = v if body == "A" else hilo(v.float())[0]
                    yo, Ao = linear(Wo, op, 1.0)
                    b = gamma(body, "o", e.n_sm) * Ao + (n_split(body, "o", e.n_sm) + 1) * U * x.abs() + 1e-30
                    yh = recover(a, lg, x)
                    r, w = assess(label + " y", yh, yo, obs_bound(body, x, yo, b), mask)
                    worst, nw = max(worst, r), max(nw, w)
            elif probe == "ffn":
                check_cache_rest(e, n, poss, l)
                yh = recover(a, lg, x)
                yr, b, parts = _ffn_ref(body, x, g2, W1, W3, W2, n_sm=e.n_sm)
                r, w = assess(label + " y", yh, yr, obs_bound(body, x, yr, b), mask)
                worst, nw = max(worst, r), max(nw, w)
                if sens_case:
                    bo = obs_bound(body, x, yr, b)
                    sens["u scaled by rs, g not"] = n_over(yh, _ffn_ref(body, x, g2, W1, W3, W2, g_unscaled=True, n_sm=e.n_sm)[0],
                                                           bo, mask)
                    sens["ln_1 gain in the FFN"] = n_over(yh, _ffn_ref(body, x, g1, W1, W3, W2, n_sm=e.n_sm)[0], bo, mask)
                    if body == "C":
                        c = split0_cols("w2", e.n_sm)
                        h = parts["h"]
                        sens["w2 without split 0"] = n_over(yh, h[:, c:] @ W2[:, c:].t(), bo, mask)
            else:   # head
                check_cache_rest(e, n, poss, l)
                nh, hi, s = operand(x, gf, body)
                y, A = linear(Wh, nh, s)
                b = lin_bound(body, "head", y, A, e.n_sm)
                r, w = assess(label + " logits", lg, y, b)
                worst, nw = max(worst, r), max(nw, w)
                if sens_case:
                    Wsh = Wh.clone()
                    Wsh[V - 2:] = Wh[V - 2 - 128:V - 128]
                    sens["ragged head tile shifted by 128 rows"] = n_over(lg, linear(Wsh, nh, s)[0], b)
                    if body != "A":
                        sens["head operand hi only"] = n_over(lg[:1], linear(Wh, hi, s)[0][:1], b[:1])
                    if body == "C":
                        c = split0_cols("head", e.n_sm)
                        sens["head without split 0"] = n_over(lg, linear(Wh[:, c:], nh[:, c:], s)[0], b)
    finally:
        case.clear()
    for k, v in sens.items():
        print(f"  sensitivity {label0}: reference with {k}: {v} elements over the bound")
        assert v > 0, f"{label0}: a reference with {k} satisfies the bound"
    return worst, nw, sens


def _ffn_ref(body, x, gain, W1, W3, W2, g_unscaled=False, n_sm=None):
    """float64 FFN of the module docstring: (y, elementwise bound before the observation chain, parts)."""
    nh, _, s = operand(x, gain, body)
    G, AG = linear(W1, nh, s)
    Uu, AU = linear(W3, nh, s)
    gam, tau = gamma(body, "w13", n_sm), TAU[body]
    eg = (gam + tau) * AG + 2.0 ** -21 * G.abs()
    eu = (gam + tau) * AU + 2.0 ** -21 * Uu.abs()
    if g_unscaled:
        G = G / rs64(x)
    sil = G * torch.sigmoid(G)
    h = sil * Uu
    eps_s = (6 + torch.floor(1.17 * G.abs())) * U
    eh = 1.1 * eg * Uu.abs() + sil.abs() * eu + 1.1 * eg * eu + (eps_s + U) * h.abs() + (G < -80) * h.abs()
    if body != "A":
        eh = eh + HILO * (h.abs() + eh)
    y = h @ W2.t()
    b = (gamma(body, "w2", n_sm) * ((h.abs() + eh) @ W2.abs().t()) + eh @ W2.abs().t()
         + (n_split(body, "w2", n_sm) + 1) * U * x.abs())
    return y, b + 1e-30, {"h": h}


def _att_eps(e, L):
    """eps of the attention tests at s = 0 for the body and cache form that ran."""
    if e.body in ("A", "B"):
        n_resc, n_acc, rho = L / 64 + 2, L / 32 + 40, 0.0
    elif e.kv == "bf16":
        n_resc, n_acc, rho = L / 64 + 2, 2.5 * L + 160, 2.0 ** -17
    else:
        n_resc, n_acc, rho = L / 16 + 2, 3 * L / 16 + 160, 0.0
    return 2.02 * (2.0 ** -21 * (n_resc + 3) + rho) + 2 * n_acc * U


def _run_mixed(a, e, case, label, n, g1, Wqkv, Wo, mask, sens):
    """Probe 5: injected K / V below p_u, poison above, three launches at p_u, p_u + 1, p_u + 2."""
    body, l = e.body, case.l
    gi = torch.Generator(device="cuda").manual_seed(n + 7 * l)
    e.m._kv.zero_()
    base = MIXED[:n]
    lay = e.cache[l]
    if e.kv == "bf16" and body == "C":
        i = torch.arange(BLOCK, device="cuda")[:, None] + torch.arange(128, device="cuda")[None]
        poison = ((i % 2) * 2 - 1).to(e.dt) * 8192 * (1 + (i % 5).to(e.dt) / 8)
    else:
        poison = torch.full((BLOCK, 128), float("nan"), dtype=e.dt, device="cuda")
    for u in range(n):
        for cr in (2 * u, 2 * u + 1):
            lay[:, cr] = poison
            p = base[u]
            lay[0, cr, :, :p] = (torch.randn(H, p, 128, generator=gi, device="cuda") * 0.7).to(e.dt)
            lay[1, cr, :, :p] = torch.randn(H, p, 128, generator=gi, device="cuda").to(e.dt)
    worst = nw = 0.0
    for it in range(3):
        poss = [p + it for p in base]
        toks = a.toks[it][:n]
        x = rows_x(a, n, toks, poss)
        before = lay.clone()
        lg = step(e, n, toks, poss)
        check_cache_rest(e, n, poss, l, before)
        nh, _, s = operand(x, g1, body)
        y, A = linear(Wqkv, nh, s)
        r, w = check_kv(e, f"{label} launch {it}", appended(e, n, poss, l), y, A)
        worst, nw = max(worst, r), max(nw, w)
        # reference attention output: the mean of the L V rows read back from the cache
        mean, em = [], []
        for u in range(n):
            L = poss[u] + 1
            for c in range(2):
                Vr = lay[1, 2 * u + c, :, :L].double()                      # [H, L, 128]
                mean.append(Vr.mean(1).reshape(D))
                em.append(_att_eps(e, L) * Vr.abs().mean(1).reshape(D))
        m, em = torch.stack(mean), torch.stack(em)
        eop = em + (0.0 if body == "A" else HILO * (m.abs() + em))
        yo = m @ Wo.t()
        b = (gamma(body, "o", e.n_sm) * ((m.abs() + eop) @ Wo.abs().t()) + eop @ Wo.abs().t()
             + (n_split(body, "o", e.n_sm) + 1) * U * x.abs() + 1e-30)
        yh = recover(a, lg, x)
        r, w = assess(f"{label} launch {it} y", yh, yo, obs_bound(body, x, yo, b), mask)
        worst, nw = max(worst, r), max(nw, w)
    return worst, nw


CASES = [(f, p) for f in FORMS for p in PROBES]


@pytest.mark.parametrize("form,probe", CASES, ids=[f"{f}-{p}" for f, p in CASES])
def test_decode_projection(arena, engines, form, probe):
    e = engines(form)
    inst = ""
    if e.body == "C":
        inst = " instances " + ", ".join(f"<{e.kv}, {32 if n > 4 else 16}> n={n}" for n in e.utts)
        inst += "; K splits " + ", ".join(f"{m} {n_split('C', m)}" for m in MATS)
    for l in LSTAR:
        worst, nw, _ = run_probe(arena, e, probe, l)
        print(f"{form} [body {e.body}, {LAUNCHES[e.body]} launches] {probe} l*={l} n_utts={list(e.utts)}{inst}: "
              f"max |err|/bound {worst:.2e}, normwise {nw:.2e}")
    print(f"  peak device memory so far: {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
