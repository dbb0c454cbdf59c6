"""GPU: every attention kernel against a float64 softmax(q K^T / sqrt(128)) V, up to the full 2048-position context.

Stage 1 (k_attn_decode / k_attn_rows over attn_core, and the attention phase of k_decode_persistent in its fp32-cache
and bf16 mma.sync forms) is fused into engine launches whose merged output never reaches global memory, so it
is observed through a PROBE MODEL that the engine runs unchanged: one layer, attn_norm = ffn_norm = ln_f = 1,
w1 = w3 = w2 = 0 (the FFN adds exactly 0), wo = I, lm_head = [I_D; 0], speaker projection 0.  Then
    logits[:, :D] = RMSNorm(x + y^)        (y^ = the merged attention output, x = tok_emb[tok] + pos_emb[pos])
wqkv is a selection matrix (one 1 per row): q, k and v of the current token are coordinates of n = RMSNorm(x), so every
path computes them with a single product.  The rows of W_v for head dimension 127 are zero and so is dimension 127 of
every injected V: y^ is exactly 0 there in every path (sums of exact zeros), hence logit h*128+127 = x_j * r with the
kernel's own final RMSNorm scale r, and r^ = mean_h(logit / x) recovers it; y^ = logit / r^ - x inverts the norm in
float64.  Embeddings sit on a 1/32 grid (|x| <= 20/32) so x is exact in bf16 and its fp32 sum of squares is exact.

The KV cache is caller memory ([layer][K|V][row = 2 utt + cfg][head][pos][128]): random K / V are written at positions
[0, L - 1), every other entry is poisoned (NaN; for the mma form, which reads whole 64-position boxes, a large finite
pattern), the position is set with mvb_s1_begin(pos = L - 1) and mvb_s1_step_logits runs one body.  Afterwards every
byte of the cache except the appended entries at L - 1 is unchanged (poison included), the appended k / v match
n_sel within 2^-15 relative (+ 2^-8 for the bf16 rounding), and the reference attends over the injected entries plus
the appended ones READ BACK from the cache.  Which body ran is taken from the launch-count delta.

Elementwise bound.  For one (row, head) with float64 scores s_i, probabilities P_i and A_i = sum_j |q_j k_ij| / sqrt(128):
    |y^ - y| <= eps * sum_i P_i |v_i| + tau_obs * (|x| + |y| + eps * sum_i P_i |v_i|)
    eps = 2.02 * dw + 2 * n_acc * u,   u = 2^-23,
    dw  = kappa * max_i A_i + 2^-21 * (n_resc + 3 + max|s|) + 3 * 2^-23 * (max s - min s) + rho_p.
Derivation.  Every weight the kernel forms is exp(s^_i - m^) (times merge factors common to a split); the shift cancels
in the normalisation, so each weight is off by exp(d_i) with |d_i| <= dw, and normalised probabilities by at most
(e^(2 dw) - 1) P_i <= 2.02 dw P_i.  dw collects:
  * the score error kappa * A_i, kappa = 2^-15: q is within 2^-17 + 4u per element of n_sel / sqrt(128) (the hi/lo
    split of RMSNorm(x) in k_prep_b; the other paths form it with one fp32 product), the mma form splits q into hi/lo
    bf16 again (2^-17), and the 128-term fp32 dot product adds at most 12u (8 fma + 4 butterfly adds) on the CUDA cores
    or 4 chains x 18u (m16n8k16 model of test_gemm_ops_gpu.py) on the tensor cores: 2^-17 + 2^-17 + 80u < 2^-15;
  * the exponentials: ex2.approx.ftz / __expf are within 2^-21 relative, the argument (s - m) * log2 e is rounded
    (|s - m| * 2^-23 each for the weight, the running-max rescales and the split merge: <= 3 * spread * 2^-23), each
    weight passes through at most n_resc running-max rescales plus 3 merge factors, and the 1/sqrt(128) and RMSNorm
    scale factors common to all scores move them by <= |s| * 2^-21;
  * rho_p = 2^-17 for the mma form, which multiplies V by p as hi + lo bf16 while the row sum uses fp32 p.
n_resc: rescales of one accumulator.  attn_core (paths A, B): a half-warp visits ceil(L/8)/8 positions, L/64 + 2;
persistent fp32-cache loop: one per 2-position trip of a half-warp, L/16 + 2; mma: one per 64-position tile, L/64 + 2.
n_acc: fp32 roundings along one output sum (and, separately, along the row sum; hence the factor 2): attn_core 2 per
visited position + 8 half-warp and 8 split merges (x 2): L/32 + 40; fp32-cache loop 3 per trip + 8 half-warp merges +
<= 64 split merges (x 2) + current token: 3 L/16 + 160; mma: per tile 4 hi + 4 lo m16n8k16 into two accumulators at
18u each plus the rescale and the add, i.e. <= 150u per 64 positions: 2.5 L + 160.
Observation chain (tau_obs = 2^-15 for paths B and C, 2^-20 for path A): paths B and C carry y^ into wo as hi + lo bf16
(2^-17 |y^|), the wo = I product has one nonzero term and the residual add rounds once (u |x + y^|); the FFN adds exact
zeros; the final RMSNorm and the head (one nonzero term) make each logit = (x + y^)_j * r (1 + 2^-17 + 3u), the same for
the pilot logits that give r^, so l / r^ - x is off by <= (2^-16 + 8u) |x + y^| + 2^-17 |y^| <= 2^-15 (|x| + |y^|).
Path A keeps everything in fp32 (k_gemv stages fp32 activations; wo and the head multiply by exact 1s): one rounding
each in the residual add and in (x * rs) * g, two ulp in r^, so the error is <= 4 u |x + y^| <= 2^-20 (|x| + |y^|).
Normwise: ||y^ - y|| / ||y|| < 1e-4 per call.

Stage 2 (k_s2_attn<64|128>) is called directly through mvb_s2_attn_test with the same bound: kappa = (hs/4 + 4) u
(hs/4 serial fma + 2 shuffle adds + the q * rsqrtf(hs) product), n_resc = t/4 + 2 (one rescale per 4-key trip),
n_acc = 5 t/4 + 8 (o * corr + 4 fma per trip; 1/l and the product), rho_p = 0, no observation chain.

Sensitivity: references that drop position 0, the first position of a KV tile or L - 2 (needle cases), that leave the
current token's k / v unrounded in bf16 mode (L = 1, 2), or that scale the scores by 1/sqrt(64) must violate the bound."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
KAPPA_S1 = 2.0 ** -15
TAU_OBS = 2.0 ** -15
TAU_OBS_A = 2.0 ** -20
NORMWISE = 1e-4
BLOCK = 2048
PILOT = 127
EPS = 1e-5

# the context lengths L = pos + 1 of every decode case, each for a boundary of one of the kernels
L_CASES = [
    1, 2,              # only the current token / one cached position (7 of attn_core's 8 splits empty)
    8, 9,              # attn_core's split length ceil(L/8) rounded up to 8: one split, then two
    16, 17,            # the mma form's 16-position warp slice; one past it
    31, 32, 33,        # fp32 tiles of 32 positions: last tile holds only the current token at 33 (npos = 0)
    63, 64, 65, 66,    # bf16 tiles of 64: npos = 0 tile at 65, one cached position in the second tile at 66
    96,                # 1.5 bf16 tiles, 3 fp32 tiles
    127, 128, 129, 130,  # two bf16 tiles: full / current only / one position in the third
    1000, 1025,        # ragged long context; 1025 = 16 bf16 tiles + a current-token-only tile
    2047, 2048,        # the last two cache slots (2048 = every slot of the context)
]
MIXED_8 = [1, 2048, 33, 65, 129, 1000, 2, 1025]     # 8 utterances in one step, mixed L including 1 and 2048

# body -> kernel launches of one mvb_s1_step_logits on the one-layer probe (k_identity_slots included):
# A: embed + 5 per layer + head = 7;  B: k_rows_decode + embed + (4 linears x 2 + attention) + head (2) = 13;
# C: the persistent kernel
BODY_LAUNCHES = {"A": 1 + 7, "B": 1 + 13, "C": 1 + 1}

# path form -> (kv dtype, tensor_core_path, body it must run); on path C the bf16 cache runs the mma.sync form
FORMS = {
    "A-fp32": ("fp32", "", "A"),
    "A-bf16": ("bf16", "", "A"),
    "B-fp32": ("fp32", "B", "B"),
    "B-bf16": ("bf16", "B", "B"),
    "C-fp32": ("fp32", None, "C"),
    "C-mma": ("bf16", None, "C"),
}


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pc_fits(n_utts, H, kv, n_sm=None):
    """Mirror of pc_att_fits (stage1_engine.cu): the persistent kernel's per-CTA attention tile table (<= 128 tiles) and
    split count (<= 64) hold for n_utts utterances at every position of the 2048-slot context on a part with n_sm SMs
    (default: this one)."""
    from test_sm_count_cpu import att_fits
    return att_fits(n_sm or _n_sm(), n_utts, H, kv, BLOCK)


def expected_body(p, n_utts):
    """The body mvb_s1_step_logits / mvb_s1_decode runs for n_utts utterances of probe p: the persistent kernel where the
    host's rule (use_path_c, mirrored in test_sm_count_cpu.py) takes the batch, else the per-layer path (tensor-core rows
    path from 2 utterances up)."""
    from test_sm_count_cpu import path_c
    if p.body == "C" and not path_c((p.D, p.H, 256, p.V), p.n_sm, n_utts, p.kv, BLOCK):
        return "B" if n_utts >= 2 else "A"
    return p.body


def _params(form, L, body):
    """(n_resc, n_acc, rho_p) of the docstring for the body that ran."""
    kv = FORMS[form][0]
    if body in ("A", "B"):
        return L / 64 + 2, L / 32 + 40, 0.0
    if kv == "bf16":
        return L / 64 + 2, 2.5 * L + 160, 2.0 ** -17
    return L / 16 + 2, 3 * L / 16 + 160, 0.0


def softmax_eps(s, A, n_resc, n_acc, kappa, rho_p):
    """eps of the docstring; s, A: [..., L] float64 -> [..., 1]."""
    spread = s.amax(-1, keepdim=True) - s.amin(-1, keepdim=True)
    dw = (kappa * A.amax(-1, keepdim=True) + 2.0 ** -21 * (n_resc + 3 + s.abs().amax(-1, keepdim=True))
          + 3 * U * spread + rho_p)
    return 2.02 * dw + 2 * n_acc * U


# ---------------------------------------------------------------------------------------------------------------------
# stage-1 probe model
class Probe:
    def __init__(self, H, form, utts, seed=0, n_layer=1, n_sm=None):
        """n_sm: the SM count the engine is planned for (default: this device's)."""
        from mvb200.fast_model import ModelArgs, Transformer
        kv, tc, body = FORMS[form]
        self.n_sm = n_sm or _n_sm()
        self.H, self.D, self.form, self.body, self.kv = H, 128 * H, form, body, kv
        D = self.D
        self.V = 512 if D <= 256 else 2562
        g = torch.Generator().manual_seed(seed)
        pil = torch.zeros(D, dtype=torch.bool)
        pil[PILOT::128] = True
        tok = torch.randint(-12, 13, (self.V, D), generator=g).float()
        mag = torch.randint(12, 21, (self.V, int(pil.sum())), generator=g).float()
        tok[:, pil] = mag * (torch.randint(0, 2, mag.shape, generator=g) * 2 - 1)
        pos = torch.randint(-4, 5, (BLOCK, D), generator=g).float()
        pos[:, pil] = 0
        self.tok, self.pos = tok / 32, pos / 32                   # exact in bf16; |x| <= 20/32
        self.perm = [torch.randperm(D, generator=g) for _ in range(3)]   # q, k, v selections
        wqkv = torch.zeros(3 * D, D)
        for i, p in enumerate(self.perm):
            wqkv[i * D + torch.arange(D), p] = 1.0
        wqkv[2 * D + PILOT::128] = 0                                # v[..., 127] == 0
        F = 256
        sd = {"transformer.wtes.0.weight": self.tok, "transformer.wpe.weight": self.pos,
              "speaker_cond_pos.weight": torch.zeros(D, 256), "transformer.ln_f.weight": torch.ones(D),
              "lm_heads.0.weight": torch.cat([torch.eye(D), torch.zeros(self.V - D, D)]),
              "transformer.h.0.ln_1.weight": torch.ones(D), "transformer.h.0.attn.c_attn.weight": wqkv,
              "transformer.h.0.attn.c_proj.weight": torch.eye(D), "transformer.h.0.ln_2.weight": torch.ones(D),
              "transformer.h.0.mlp.swiglu.w1.weight": torch.zeros(F, D),
              "transformer.h.0.mlp.swiglu.w3.weight": torch.zeros(F, D),
              "transformer.h.0.mlp.c_proj.weight": torch.zeros(D, F)}
        if n_layer == 2:
            # layer 1 appends k = RMSNorm(x + y^_0) (W_k = I, q = v = 0) and adds exactly 0 to the residual stream
            wqkv1 = torch.zeros(3 * D, D)
            wqkv1[D:2 * D] = torch.eye(D)
            sd.update({"transformer.h.1.ln_1.weight": torch.ones(D), "transformer.h.1.attn.c_attn.weight": wqkv1,
                       "transformer.h.1.attn.c_proj.weight": torch.zeros(D, D), "transformer.h.1.ln_2.weight": torch.ones(D),
                       "transformer.h.1.mlp.swiglu.w1.weight": torch.zeros(F, D),
                       "transformer.h.1.mlp.swiglu.w3.weight": torch.zeros(F, D),
                       "transformer.h.1.mlp.c_proj.weight": torch.zeros(D, F)})
        sd = {k: v.to(torch.bfloat16) for k, v in sd.items()}
        cfg = ModelArgs(block_size=BLOCK, vocab_size=self.V, n_layer=n_layer, n_head=H, dim=D, intermediate_size=F)
        self.m = Transformer.from_state_dict(sd, cfg, device="cuda:0")
        self.m.setup_caches(2 * utts, BLOCK, kv_dtype=kv, tensor_core_path=tc)
        dt = torch.float32 if kv == "fp32" else torch.bfloat16
        self.kv_all = self.m._kv.view(dt).view(n_layer, 2, 2 * utts, H, BLOCK, 128)   # [layer][K|V][row][head][pos][128]
        self.cache = self.kv_all[0]
        self.tok_d, self.pos_d = self.tok.double().cuda(), self.pos.double().cuda()
        self.perm_d = [p.cuda() for p in self.perm]
        if kv == "bf16" and body == "C":
            i = torch.arange(BLOCK, device="cuda")[:, None] + torch.arange(128, device="cuda")[None]
            self.poison = ((i % 2) * 2 - 1).to(dt) * 8192 * (1 + (i % 5).to(dt) / 8)   # finite: the mma form reads whole boxes
        else:
            self.poison = torch.full((BLOCK, 128), float("nan"), dtype=dt, device="cuda")

    def close(self):
        self.m.close()

    def x(self, tok, pos):
        """float64 [..., D]: the fp32 sum tok_emb + pos_emb (exact on the 1/32 grid)."""
        return self.tok_d[tok] + self.pos_d[pos]

    def sel(self, x):
        """float64 n = RMSNorm(x) and its q / k / v selections [..., H, 128] (q unscaled)."""
        n = x / torch.sqrt((x * x).mean(-1, keepdim=True) + EPS)
        q, k, v = (n[..., p].reshape(*x.shape[:-1], self.H, 128) for p in self.perm_d)
        v = v.clone()
        v[..., PILOT] = 0
        return q, k, v

    def recover(self, logits, x):
        """y^ from the logits rows [..., V] and x [..., D] (float64)."""
        l = logits[..., :self.D].double()
        r = (l[..., PILOT::128] / x[..., PILOT::128]).mean(-1, keepdim=True)
        return l / r - x


def _launches(p):
    return int(p.m._lib.mvb_s1_launch_count(p.m.handle))


def make_kv(p, q, L, regime, g, needle=None):
    """Injected K, V [H, L - 1, 128] (float64 of the stored dtype) for one cache row whose query is q [H, 128]."""
    H, n = p.H, L - 1
    dt = p.cache.dtype
    rnd = lambda *s: torch.randn(*s, generator=g, device="cuda", dtype=torch.float64)  # noqa: E731
    qhat = q * math.sqrt(128) / (q * q).sum(-1, keepdim=True)          # k = t * qhat scores t
    if regime == "flat":
        K = rnd(H, n, 128) * 0.7
    elif regime == "wide":
        t = (torch.rand(H, n, 1, generator=g, device="cuda", dtype=torch.float64) * 2 - 1) * 40
        K = t * qhat[:, None] + rnd(H, n, 128) * 0.05
    elif regime == "ties":
        K = (rnd(H, 1, 128) * 0.7).expand(H, n, 128)
    elif regime == "needle":
        K = rnd(H, n, 128) * 0.3
        if needle == "cur":
            K = K - 30 * qhat[:, None]
        else:
            K[:, needle] += 25 * qhat
    else:
        raise ValueError(regime)
    Vv = rnd(H, n, 128)
    Vv[..., PILOT] = 0
    return K.to(dt).double(), Vv.to(dt).double()


def run_decode(p, Ls, regime, seed, needles=None, tok=None):
    """One mvb_s1_step_logits for utterances with context lengths Ls on an injected, poisoned cache.  Returns the
    per-row data the checks need: list of dicts with y^, q, K_all, V_all (float64, appended entries read back)."""
    from mvb200 import _lib
    n = len(Ls)
    g = torch.Generator(device="cuda").manual_seed(seed)
    gt = torch.Generator().manual_seed(seed)
    toks = tok if tok is not None else torch.randint(0, p.V, (n,), generator=gt).tolist()
    cache = p.cache
    cache[:] = p.poison
    rows = []
    for u, L in enumerate(Ls):
        x = p.x(torch.tensor(toks[u], device="cuda"), torch.tensor(L - 1, device="cuda"))
        q, kc, vc = p.sel(x)
        for c in range(2):
            K, Vv = make_kv(p, q, L, regime, g, None if needles is None else needles[u])
            cache[0, 2 * u + c, :, :L - 1] = K.to(cache.dtype)
            cache[1, 2 * u + c, :, :L - 1] = Vv.to(cache.dtype)
            rows.append(dict(u=u, c=c, L=L, x=x, q=q, kc=kc, vc=vc, K=K, V=Vv))
    before = p.m._kv.clone()
    lib, h, st = p.m._lib, p.m.handle, p.m._stream()
    sp = _lib.Sampling(1.0, 1.0, 0.0, 0, 9999, 1)
    for u, L in enumerate(Ls):
        _lib.check(lib.mvb_s1_begin(h, u, int(toks[u]), L - 1, C.byref(sp), None, None, st))
    n0 = _launches(p)
    lg = torch.empty(2 * n, p.V, device="cuda")
    _lib.check(lib.mvb_s1_step_logits(h, n, lg.data_ptr(), st))
    torch.cuda.synchronize()
    body = expected_body(p, n)
    assert _launches(p) - n0 == BODY_LAUNCHES[body], f"{p.form}: body {body} did not run"
    # only the appended entries changed
    want = before.view(cache.dtype).view(cache.shape)
    for r in rows:
        cr, L = 2 * r["u"] + r["c"], r["L"]
        want[:, cr, :, L - 1] = cache[:, cr, :, L - 1]
    assert torch.equal(p.m._kv, before), f"{p.form}: the step changed cache entries other than the appended ones"
    for r in rows:
        cr, L = 2 * r["u"] + r["c"], r["L"]
        ka, va = cache[0, cr, :, L - 1].double(), cache[1, cr, :, L - 1].double()
        rel = 2.0 ** -15 + (2.0 ** -8 if p.kv == "bf16" else 0.0)
        for got, ref, what in ((ka, r["kc"], "k"), (va, r["vc"], "v")):
            assert ((got - ref).abs() <= rel * ref.abs() + 1e-30).all(), f"{p.form} L={L}: appended {what} off"
        r["K_all"] = torch.cat([r["K"], ka[:, None]], 1)
        r["V_all"] = torch.cat([r["V"], va[:, None]], 1)
        r["y_hat"] = p.recover(lg[cr], r["x"]).view(p.H, 128)
        r["body"], r["logits"] = body, lg[cr]
    return rows


def reference(r, scale=1 / math.sqrt(128), drop=None, k_cur=None, v_cur=None):
    """float64 attention of one row; drop: a position left out; k_cur / v_cur: replace the appended entries."""
    K, Vv = r["K_all"].clone(), r["V_all"].clone()
    if k_cur is not None:
        K[:, -1], Vv[:, -1] = k_cur, v_cur
    q = r["q"]
    s = torch.einsum("hd,hld->hl", q, K) * scale
    A = torch.einsum("hd,hld->hl", q.abs(), K.abs()) * scale
    if drop is not None:
        s[:, drop] = -math.inf
    P = torch.softmax(s, -1)
    return torch.einsum("hl,hld->hd", P, Vv), s, A, torch.einsum("hl,hld->hd", P, Vv.abs())


def _bound(p, r):
    """The reference output and the elementwise bound of the docstring for one row."""
    y, s, A, PV = reference(r)
    n_resc, n_acc, rho = _params(p.form, r["L"], r["body"])
    eps = softmax_eps(s, A, n_resc, n_acc, KAPPA_S1, rho) * PV
    tau = TAU_OBS_A if r["body"] == "A" else TAU_OBS
    return y, eps + tau * (r["x"].view(p.H, 128).abs() + y.abs() + eps) + 1e-30


def check_rows(p, rows, label):
    """Assert the bound for every row; returns (worst ratio, worst normwise)."""
    worst = nw_worst = 0.0
    for r in rows:
        y, bound = _bound(p, r)
        err = (r["y_hat"] - y).abs()
        err[:, PILOT] = 0
        ratio = float((err / bound).max())
        nw = float(err.norm() / y.norm())
        worst, nw_worst = max(worst, ratio), max(nw_worst, nw)
        bad = (err > bound).nonzero()
        assert bad.numel() == 0, (f"{label} utt {r['u']} row {r['c']} L={r['L']}: {bad.shape[0]} elements over the bound "
                                  f"(max ratio {ratio:.2e}), first (head, dim) {bad[0].tolist()}")
        assert nw < NORMWISE, f"{label} L={r['L']}: normwise {nw:.2e}"
    return worst, nw_worst


def violations(p, rows, **ref_kw):
    """Sensitivity: the kernel's output against an altered reference, under the bound of the true one: (elements over,
    max ratio)."""
    n_over, worst = 0, 0.0
    for r in rows:
        _, bound = _bound(p, r)
        y = reference(r, **ref_kw)[0]
        err = (r["y_hat"] - y).abs()
        err[:, PILOT] = 0
        n_over += int((err > bound).sum())
        worst = max(worst, float((err / bound).max()))
    return n_over, worst


@pytest.fixture(scope="module")
def probes():
    cache = {}

    def get(H, form, utts, n_layer=1):
        key = (H, form, utts, n_layer)
        if key not in cache:
            for k in list(cache):
                cache.pop(k).close()
            torch.cuda.empty_cache()
            cache[key] = Probe(H, form, utts, seed=H, n_layer=n_layer)
        return cache[key]
    yield get
    for v in cache.values():
        v.close()


@pytest.mark.parametrize("H", [2, 16])
@pytest.mark.parametrize("form", list(FORMS))
def test_decode_every_length(probes, form, H):
    """Every L of L_CASES alone (the <., 16> persistent instance: 1 utterance; paths A / B: 2 utterances at the same L)
    and 8 utterances in one step with mixed L (the <., 32> instance), flat / wide / tied scores."""
    utts = 8
    p = probes(H, form, utts)
    single = 2 if p.body == "B" else 1
    worst = nw = 0.0
    for regime in ("flat", "wide", "ties"):
        for i, L in enumerate(L_CASES):
            w, n = check_rows(p, run_decode(p, [L] * single, regime, seed=1000 * H + 10 * i), f"{form} H={H} {regime}")
            worst, nw = max(worst, w), max(nw, n)
        w, n = check_rows(p, run_decode(p, MIXED_8, regime, seed=7 + H), f"{form} H={H} {regime} mixed-8")
        worst, nw = max(worst, w), max(nw, n)
    print(f"decode {form} H={H} [body {p.body}]: every L in {L_CASES[0]}..{L_CASES[-1]} + mixed batch of 8: "
          f"max |err|/bound {worst:.2e}, normwise {nw:.2e}")


NEEDLE_LS = [2, 34, 66, 130, 1025, 2048]


def _needles(L):
    """needle positions for context length L: 0, the last / first positions of the first fp32 and bf16 tiles, the first
    position of the last tile, L - 2, and the current token."""
    cand = [0, 31, 32, 63, 64, (L - 2) // 64 * 64, (L - 2) // 32 * 32, L - 2]
    return sorted({c for c in cand if 0 <= c < L - 1}) + ["cur"]


@pytest.mark.parametrize("form", list(FORMS))
def test_decode_needles(probes, form):
    p = probes(2, form, 8)
    worst = 0.0
    for L in NEEDLE_LS:
        for nd in _needles(L):
            w, _ = check_rows(p, run_decode(p, [L] * (2 if p.body == "B" else 1), "needle", seed=L, needles=[nd] * 2),
                              f"{form} needle {nd} L={L}")
            worst = max(worst, w)
    print(f"needles {form} [body {p.body}]: max |err|/bound {worst:.2e}")


def test_persistent_tile_table_at_capacity(probes):
    """fp32 cache, H = 16, 8 utterances all at L = 2048: on 132 SMs every CTA owns up to PC_MAX_TILES = 128 tiles (and
    the split merge reads nz = 1 partial per (row, head)); path C must still run it.  Parts with fewer SMs route this
    batch to the per-layer path (pc_att_fits), which the other cases cover."""
    if not _pc_fits(8, 16, "fp32"):
        pytest.skip(f"on {_n_sm()} SMs the tile table of this batch exceeds 128 tiles; the host check picks the per-layer path")
    p = probes(16, "C-fp32", 8)
    assert expected_body(p, 8) == "C"
    for regime in ("flat", "wide"):
        w, nw = check_rows(p, run_decode(p, [2048] * 8, regime, seed=5), f"C-fp32 capacity {regime}")
        print(f"C-fp32 H=16, 8 x L=2048 ({_n_sm()} SMs) {regime} [body C]: max |err|/bound {w:.2e}, normwise {nw:.2e}")


def test_split_merge_above_four_splits(probes):
    """H = 2, one utterance: zmax = n_sm / 4, so long rows are cut into more than 4 splits and the wo staging takes its
    nch > 4 merge branch (fp32: up to 64 tiles -> min(zmax, 64) splits)."""
    split_merge(probes)


def split_merge(probes):
    """test_split_merge_above_four_splits on the SM count the probes are planned for."""
    for form, ppc in (("C-fp32", 32), ("C-mma", 64)):
        p = probes(2, form, 8)
        n_sm = p.n_sm
        for L in (1000, 2048):
            tt = (L + ppc - 1) // ppc
            zr = min(n_sm // 4, tt)
            tps = (tt + zr - 1) // zr
            nz = (tt + tps - 1) // tps
            assert nz > 4
            w, nw = check_rows(p, run_decode(p, [L], "wide", seed=L), f"{form} nz={nz}")
            print(f"{form} L={L}: {nz} splits merged [body {expected_body(p, 1)}]: max |err|/bound {w:.2e}, normwise {nw:.2e}")


@pytest.mark.parametrize("n", [12, 40])
@pytest.mark.parametrize("kv", ["fp32", "bf16"])
def test_path_b_many_utterances(probes, n, kv):
    p = probes(2, f"B-{kv}", n)
    Ls = [L_CASES[(5 * i) % len(L_CASES)] for i in range(n - 2)] + [1, 2048]
    for regime in ("flat", "wide"):
        w, nw = check_rows(p, run_decode(p, Ls, regime, seed=n), f"B-{kv} n={n} {regime}")
        print(f"path B, {n} utterances (R = {2 * n}), L up to 2048, {regime}: max |err|/bound {w:.2e}, normwise {nw:.2e}")


# ---- prefill: 70 positions on an injected cache ------------------------------------------------------------------
@pytest.mark.parametrize("pos0", [0, 1000, 1978])
@pytest.mark.parametrize("form", ["A-fp32", "B-fp32", "B-bf16"])
def test_prefill_every_position(probes, form, pos0):
    """mvb_s1_forward, S = 70 from pos0 (path A: one position at a time; path B: 64-token chunks, causal inside the
    chunk): every position's output against float64 attention over the injected [0, pos0) plus the entries the prefill
    appended, read back.  Positions >= pos0 + 70 stay NaN and untouched."""
    from mvb200 import _lib
    p = probes(2, form, 1)
    S = 70
    g = torch.Generator(device="cuda").manual_seed(pos0)
    gt = torch.Generator().manual_seed(pos0)
    idx = torch.randint(0, p.V, (2, S), generator=gt, dtype=torch.int32)
    pos = torch.arange(pos0, pos0 + S, device="cuda")
    cache = p.cache
    cache[:] = float("nan")
    x = p.x(idx.cuda().long(), pos[None].expand(2, S))              # [2, S, D]
    q, kc, vc = p.sel(x)                                            # [2, S, H, 128]
    inj = []
    for c in range(2):
        K, Vv = make_kv(p, q[c, 0], pos0 + 1, "flat", g)
        cache[0, c, :, :pos0] = K.to(cache.dtype)
        cache[1, c, :, :pos0] = Vv.to(cache.dtype)
        inj.append((K, Vv))
    before = p.m._kv.clone()
    lg = torch.empty(2, S, p.V, device="cuda")
    n0 = _launches(p)
    _lib.check(p.m._lib.mvb_s1_forward(p.m.handle, 0, idx.cuda().contiguous().data_ptr(), S, pos0, lg.data_ptr(), 1,
                                       p.m._stream()))
    torch.cuda.synchronize()
    # path A: k_set_input + the one-position body (7 launches) per position; path B per 64-token chunk: k_rows_prefill +
    # embed + (4 linears x 2 + attention) + head (2), then k_gather_last + the last position's head (2) + k_set_input
    want_launches = S * (1 + 7) if p.body == "A" else -(-S // 64) * (1 + 1 + 9 + 2) + 4
    assert _launches(p) - n0 == want_launches, f"prefill {form}: body {p.body} did not run"
    want = before.view(cache.dtype).view(cache.shape)
    want[:, :2, :, pos0:pos0 + S] = cache[:, :2, :, pos0:pos0 + S]
    assert torch.equal(p.m._kv, before), "the prefill changed cache entries outside [pos0, pos0 + S)"
    worst = nw = 0.0
    for c in range(2):
        Ka = cache[0, c, :, pos0:pos0 + S].double()                 # [H, S, 128]
        Va = cache[1, c, :, pos0:pos0 + S].double()
        rel = 2.0 ** -15 + (2.0 ** -8 if p.kv == "bf16" else 0.0)
        assert ((Ka - kc[c].transpose(0, 1)).abs() <= rel * kc[c].transpose(0, 1).abs() + 1e-30).all()
        assert ((Va - vc[c].transpose(0, 1)).abs() <= rel * vc[c].transpose(0, 1).abs() + 1e-30).all()
        Kall, Vall = torch.cat([inj[c][0], Ka], 1), torch.cat([inj[c][1], Va], 1)
        for i in range(S):
            L = pos0 + i + 1
            r = dict(u=0, c=c, L=L, x=x[c, i], q=q[c, i], K_all=Kall[:, :L], V_all=Vall[:, :L], body=p.body,
                     y_hat=p.recover(lg[c, i], x[c, i]).view(p.H, 128))
            w, n = check_rows(p, [r], f"prefill {form} pos0={pos0} i={i}")
            worst, nw = max(worst, w), max(nw, n)
    print(f"prefill {form} pos0={pos0}, 70 positions: max |err|/bound {worst:.2e}, normwise {nw:.2e}")


# ---- the fused multi-step burst ------------------------------------------------------------------------------------
# (form, first position, last position): bursts that cross fp32 (32) and bf16 (64) tile boundaries, and the context end
BURSTS = [("C-fp32", 28, 40), ("C-mma", 60, 70), ("C-fp32", 2030, 2047), ("C-mma", 2030, 2047)]


@pytest.mark.parametrize("n_utts", [1, 8])
@pytest.mark.parametrize("form,first,last", BURSTS)
def test_fused_burst_reads_back_its_own_appends(probes, form, first, last, n_utts):
    """mvb_s1_decode with forced tokens and top_k = 0 runs the whole burst in ONE persistent launch: the K / V of position
    t are stored with generic stores + fence.proxy.async and fetched by TMA at t + 1 inside the same launch.  Two-layer
    probe: layer 1 has W_k = I, so the layer-1 k it appends at t is RMSNorm(x_t + y^_0(t)) = the layer-0 attention output
    at t, which attends over every entry appended earlier in the burst.  Checked at every position against float64
    teacher-forced attention over the layer-0 cache read back: the layer-0 k / v (2^-15, + 2^-8 bf16) and the layer-1 k,
    whose bound is the attention bound b propagated through the RMSNorm (first order, |z| = |x + y|, r = rsqrt(mean z^2
    + eps)):  r b + |n1| r^2 sum(|z| b) / D, plus 2^-15 |n1| for the layer-1 QKV (hi/lo staging, 256-term fp32 sum of
    squares, rsqrtf) and 2^-8 |n1| for the bf16 rounding.  No other cache byte changes.  With the fp32 cache, a reference
    that misses the entry appended one step earlier (a stale read) must violate the bound."""
    p = probes(2, form, 8, n_layer=2)
    if expected_body(p, n_utts) != "C":
        pytest.skip(f"on {_n_sm()} SMs the persistent kernel does not take this batch")
    fused_burst(probes, form, first, last, n_utts)


def fused_burst(probes, form, first, last, n_utts):
    """test_fused_burst_reads_back_its_own_appends on the SM count the probes are planned for; path C must take the
    batch with the fused sampler."""
    from mvb200 import _lib
    p = probes(2, form, 8, n_layer=2)
    n_steps, D = last - first + 1, p.D
    g = torch.Generator(device="cuda").manual_seed(first + n_utts)
    toks = torch.randint(0, p.V, (n_utts, n_steps), generator=torch.Generator().manual_seed(first + n_utts))
    kv = p.kv_all
    kv[:] = p.poison
    for u in range(n_utts):
        for cr in (2 * u, 2 * u + 1):
            for l in range(2):
                kv[l, 0, cr, :, :first] = (torch.randn(p.H, first, 128, generator=g, device="cuda", dtype=torch.float64) * 0.7).to(kv.dtype)
                Vv = torch.randn(p.H, first, 128, generator=g, device="cuda", dtype=torch.float64)
                Vv[..., PILOT] = 0
                kv[l, 1, cr, :, :first] = Vv.to(kv.dtype)
    before = p.m._kv.clone()
    # token of position first + i: toks[:, i]; the sampler feeds back forced[n] after its n-th draw
    forced = [torch.cat([toks[u, 1:], toks[u, :1]]).to(torch.int32).cuda().contiguous() for u in range(n_utts)]
    lib, h, st = p.m._lib, p.m.handle, p.m._stream()
    sp = _lib.Sampling(1.0, 1.0, 0.0, 0, 9999, 1)          # top_k = 0: the fused single-launch path
    for u in range(n_utts):
        _lib.check(lib.mvb_s1_begin(h, u, int(toks[u, 0]), first, C.byref(sp), None, forced[u].data_ptr(), st))
    n0 = _launches(p)
    _lib.check(lib.mvb_s1_decode(h, n_utts, n_steps, st))
    torch.cuda.synchronize()
    # k_identity_slots + ONE persistent launch (per-step launches would be 1 + 2 n_steps)
    assert _launches(p) - n0 == 2, f"{form}: the burst did not run as one fused launch"
    want = before.view(kv.dtype).view(kv.shape)
    for u in range(n_utts):
        want[:, :, 2 * u:2 * u + 2, :, first:last + 1] = kv[:, :, 2 * u:2 * u + 2, :, first:last + 1]
    assert torch.equal(p.m._kv, before), f"{form}: the burst changed cache entries outside positions [{first}, {last}]"
    rel = 2.0 ** -15 + (2.0 ** -8 if p.kv == "bf16" else 0.0)
    worst = nw = 0.0
    stale_over = 0
    for u in range(n_utts):
        x = p.x(toks[u].cuda(), torch.arange(first, last + 1, device="cuda"))      # [n_steps, D]
        q, kc, vc = p.sel(x)
        for cr in (2 * u, 2 * u + 1):
            K0, V0 = kv[0, 0, cr, :, :last + 1].double(), kv[0, 1, cr, :, :last + 1].double()
            for got, ref, what in ((K0[:, first:], kc, "k"), (V0[:, first:], vc, "v")):
                ref = ref.transpose(0, 1)
                assert ((got - ref).abs() <= rel * ref.abs() + 1e-30).all(), f"{form}: layer-0 {what} appended in the burst off"
            for i in range(n_steps):
                L = first + i + 1
                r = dict(u=u, c=cr & 1, L=L, x=x[i], q=q[i], K_all=K0[:, :L], V_all=V0[:, :L], body="C")
                y, b = _bound(p, r)
                z = x[i] + y.reshape(D)
                r1 = 1 / torch.sqrt((z * z).mean() + EPS)
                n1 = z * r1
                bf = b.reshape(D)
                bound = 1.01 * (r1 * bf + n1.abs() * r1 ** 2 * (z.abs() * bf).sum() / D) + rel * n1.abs() + 1e-30
                k1 = kv[1, 0, cr, :, first + i].double().reshape(D)
                err = (k1 - n1).abs()
                bad = (err > bound).nonzero()
                assert bad.numel() == 0, (f"{form} burst {first}->{last} utt {u} row {cr & 1} position {first + i}: layer-1 k "
                                          f"{bad.shape[0]} elements over, max ratio {float((err / bound).max()):.2e}")
                worst = max(worst, float((err / bound).max()))
                nw = max(nw, float(err.norm() / n1.norm()))
                if i > 0:            # the reference without the entry position first + i - 1 appended one step earlier
                    ys = reference(r, drop=L - 2)[0]
                    zs = x[i] + ys.reshape(D)
                    ns = zs / torch.sqrt((zs * zs).mean() + EPS)
                    stale_over += int(((k1 - ns).abs() > bound).sum())
    if p.kv == "fp32":
        assert nw < NORMWISE, f"{form}: layer-1 k normwise {nw:.2e}"
        if first < 100:      # (at L ~ 2040 one flat position moves y^ by less than the bound)
            assert stale_over > 0, "a reference that misses the previous step's append satisfies the bound"
    print(f"fused burst {form} {first}->{last}, {n_utts} utterance(s) [one launch]: layer-1 k max |err|/bound {worst:.2e}, "
          f"normwise {nw:.2e}; stale-read reference: {stale_over} elements over")


# ---- sensitivity -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", ["A-bf16", "B-fp32", "C-fp32", "C-mma"])
def test_altered_references_violate_the_bound(probes, form):
    p = probes(2, form, 8)
    nb = 2 if p.body == "B" else 1
    L = 2048
    ppc = 32 if p.kv == "fp32" else 64
    for drop, L in ((0, L), (ppc * 5, L), (L - 2, L)):
        rows = run_decode(p, [L] * nb, "needle", seed=3, needles=[drop] * nb)
        check_rows(p, rows, f"{form} needle {drop}")
        n_over, ratio = violations(p, rows, drop=drop)
        print(f"{form} L={L}: reference without position {drop}: {n_over} elements over, max ratio {ratio:.1e}")
        assert n_over > 0
    rows = run_decode(p, [130] * nb, "wide", seed=4)
    n_over, ratio = violations(p, rows, scale=1 / math.sqrt(64))
    print(f"{form} L=130 wide: scores scaled by 1/sqrt(64): {n_over} elements over, max ratio {ratio:.1e}")
    assert n_over > 0
    if p.kv == "bf16":
        for L in (1, 2):
            rows = run_decode(p, [L] * nb, "flat", seed=L)
            n_over = 0
            for r in rows:
                k_cur, v_cur = r["kc"], r["vc"]
                n, ratio = violations(p, [r], k_cur=k_cur, v_cur=v_cur)
                n_over += n
            print(f"{form} L={L}: unrounded current-token k / v: {n_over} elements over, max ratio {ratio:.1e}")
            assert n_over > 0


# ---------------------------------------------------------------------------------------------------------------------
# stage 2: k_s2_attn<64|128>
S2_T = [1, 3, 4, 5, 31, 32, 33, 63, 64, 65, 256, 1023, 1024]


def _s2_qkv(B, t, E, nh, regime, g):
    hs = E // nh
    rnd = lambda *s: torch.randn(*s, generator=g, device="cuda", dtype=torch.float64)  # noqa: E731
    q = rnd(B, t, nh, hs)
    if regime == "flat":
        k = rnd(B, t, nh, hs) * 0.1
    elif regime == "wide":
        d = rnd(1, 1, nh, hs)
        d = d / d.norm(dim=-1, keepdim=True)
        q = q * 0.05 + d * (torch.rand(B, t, nh, 1, generator=g, device="cuda", dtype=torch.float64) * 2 - 1) * math.sqrt(hs)
        k = d * (torch.rand(B, t, nh, 1, generator=g, device="cuda", dtype=torch.float64) * 2 - 1) * 40 + rnd(B, t, nh, hs) * 0.05
    elif regime == "ties":
        k = (rnd(B, 1, nh, hs) * 0.3).expand(B, t, nh, hs)
    elif regime == "needle":       # one key per (batch, head) scores ~ +12..25 for every query, the rest ~ 0
        d = rnd(1, 1, nh, hs)
        d = d / d.norm(dim=-1, keepdim=True)
        q = q * 0.3 + d * math.sqrt(hs) * (0.5 + 0.5 * torch.rand(B, t, nh, 1, generator=g, device="cuda", dtype=torch.float64))
        j = torch.randint(0, t, (B, 1, nh, 1), generator=g, device="cuda")
        hot = torch.zeros(B, t, nh, 1, device="cuda", dtype=torch.float64).scatter_(1, j, 1.0)
        k = rnd(B, t, nh, hs) * 0.05 + hot * d * 25
    else:
        raise ValueError(regime)
    v = rnd(B, t, nh, hs)
    return torch.cat([z.reshape(B * t, E) for z in (q, k, v)], 1).float()


def _s2_run(qkv, B, t, E, nh, guard=5):
    from mvb200 import _lib as L
    lib = L.load()
    out = torch.full((B * t + guard, E), float("nan"), device="cuda")
    L.check(lib.mvb_s2_attn_test(qkv.data_ptr(), B, t, E, nh, out.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    assert not torch.isnan(out[:B * t]).any(), "output rows left unwritten"
    assert torch.isnan(out[B * t:]).all(), "the kernel wrote past [B * t, E)"
    return out[:B * t]


def _s2_ref(qkv, B, t, E, nh, scale=None):
    hs = E // nh
    z = qkv.double().view(B, t, 3, nh, hs)
    q, k, v = (z[:, :, i].transpose(1, 2) for i in range(3))     # [B, nh, t, hs]
    sc = scale if scale is not None else 1 / math.sqrt(hs)
    s = q @ k.transpose(-1, -2) * sc
    A = q.abs() @ k.abs().transpose(-1, -2) * sc
    P = torch.softmax(s, -1)
    y = P @ v
    eps = softmax_eps(s, A, t / 4 + 2, 1.25 * t + 8, (hs / 4 + 4) * U, 0.0) * (P @ v.abs())
    back = lambda a: a.transpose(1, 2).reshape(B * t, E)  # noqa: E731
    return back(y), back(eps + 1e-30)


@pytest.mark.parametrize("hs", [64, 128])
@pytest.mark.parametrize("B", [1, 3])
def test_stage2_attention(hs, B):
    nh = 2
    E = nh * hs
    worst = nw = 0.0
    for regime in ("flat", "wide", "ties", "needle"):
        for t in S2_T:
            g = torch.Generator(device="cuda").manual_seed(t + 7 * B + hs)
            qkv = _s2_qkv(B, t, E, nh, regime, g)
            got = _s2_run(qkv, B, t, E, nh).double()
            y, bound = _s2_ref(qkv, B, t, E, nh)
            err = (got - y).abs()
            bad = (err > bound).nonzero()
            assert bad.numel() == 0, f"hs={hs} B={B} t={t} {regime}: {bad.shape[0]} over, first {bad[0].tolist()}"
            n = float(err.norm() / y.norm())
            assert n < NORMWISE, f"hs={hs} B={B} t={t} {regime}: normwise {n:.2e}"
            worst, nw = max(worst, float((err / bound).max())), max(nw, n)
    print(f"k_s2_attn<{hs}> B={B}, t in {S2_T[0]}..{S2_T[-1]}, 4 regimes: max |err|/bound {worst:.2e}, normwise {nw:.2e}")


@pytest.mark.parametrize("hs", [64, 128])
def test_stage2_scale_sensitivity(hs):
    """A reference that scales the scores by 1/sqrt(hs/2) violates the bound."""
    nh, B, t = 2, 1, 65
    E = nh * hs
    qkv = _s2_qkv(B, t, E, nh, "wide", torch.Generator(device="cuda").manual_seed(1))
    got = _s2_run(qkv, B, t, E, nh).double()
    y, bound = _s2_ref(qkv, B, t, E, nh, scale=1 / math.sqrt(hs / 2))
    n_over = int(((got - y).abs() > bound).sum())
    print(f"k_s2_attn<{hs}>: reference scaled by 1/sqrt({hs // 2}): {n_over} of {got.numel()} elements over")
    assert n_over > 0
