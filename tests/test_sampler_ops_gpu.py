"""GPU: every token sampler against a float64 restatement of its semantics: k_sample (API and decode mode), the
grid-distributed sampler inside k_decode_persistent (the fused burst) and k_s2_sample, with supplied Exp(1) noise and
with the on-device Philox streams.

Reference.  It starts from the exact fp32 keys a kernel forms (numpy float32, same rounding order):
    stage 1: k = fdiv_rn(fadd_rn(fmul_rn(g, l_c), fmul_rn(1 - g, l_u)), max(T, 1e-5));   stage 2: k = fdiv_rn(l, T)
and then works in float64: stable ascending order (ties by ascending index); top-k sets entries < the k-th largest key
to -inf (top_k >= V keeps everything); e = exp(k - max), cum = inclusive cumulative sum / total in that order; top-p
drops cum <= fp32(1 - top_p) except the last entry of the order; p = e / sum of kept e; token = argmax(p / q), lowest
index on ties.  Philox noise is recomputed on the host (Philox4x32-10, the kernels' counters and keys; the uniform is
formed in numpy float32 exactly as on the device, the one word that rounds it to 1.0 clamped to 1 - 2^-24 as the kernels
do) and q = -log(uni) in float64.

Bounds (u = 2^-24, the fp32 unit roundoff; every bound carries a factor 1.01 for second-order terms).
  * Each exponential: e_i = expf(fsub_rn(k_i, m)); the subtraction is off by <= u |k_i - m| in the argument and expf by
    <= 2 ulp, so e_i is within a_i = 2^-22 + u |k_i - m| relative.  Entries with k_i - m < -87 (e below 2^-126) may
    flush or lose relative accuracy: they carry an absolute 2^-126 each instead.  a = max a_i over the other entries.
  * Cumulative mass (kept-set decisions).  k_sample: the scan sums 4 entries per thread, 5 warp-scan levels, 5 levels over
    the 32 warp totals, forms the exclusive prefix as incl - loc (a cancellation: its error is relative to the warp
    total, not to the prefix) and adds <= 4 own entries; every rounding is bounded by u times a partial sum <= total, at
    most 44 of them feed one cum (30 the numerator, 13 the total, 1 the division):
        delta_cum = 1.01 (2 a + 44 u) + V 2^-126.
    Fused sampler: a lane sums V/32 entries in sequence, then 5 shuffle levels; Z sums V/128 per thread, 5 + 2 levels;
    all terms are positive, so the error is relative to cum <= 1:  delta_cum = 1.01 (2 a + (V/32 + V/128 + 13) u) + V 2^-126.
    Every entry whose float64 cum lies more than delta_cum from fp32(1 - top_p) must be kept or dropped exactly as in
    the reference; entries inside that band are excused and counted (the token check then accepts either decision).
    When every key is equal, every e is exactly 1 and every partial sum is an integer < 2^24, so the kernels' cum is
    exact: delta_cum = 0 and the kept set must match exactly (the tie-order cases).
  * Probabilities (probs_out of mvb_s1_sample): p^_i = fdiv(e^_i, K^), K^ the kept sum (k_sample: 4 per thread + two
    5-level warp sums, 13 roundings of a positive sum), on the kernel's own kept set:
        |p^ - p| <= beta_i p + 2^-125,   beta_i = 1.01 (a_i + a + 14 u).
  * Token: score^_i = fdiv(p^_i, q_i) is within rho = 1.01 (2 a + (n_K + 2) u + eps_q) of p_i / q_i, n_K = 13
    (k_sample), PC_SAMP_OWN + 10 = 42 (fused: own entries, CTA partials, block sum), 19 (k_s2_sample: 8 per thread,
    5 shuffle levels, 8 warp totals), eps_q = 2^-23 for Philox (logf, 1 ulp) and 0 for supplied noise.  The token must
    equal the float64 arg-max j unless score_tok >= score_j (1 - rho) / (1 + rho) (a certified near-tie: either
    candidate passes).  Every case set has draws that are not near-ties.
Goodness of fit of the Philox streams: Pearson chi-square against the float64 probabilities with bins of expected count
< 5 merged, rejected below p = 1e-6; the same statistic must reject the tokens against a slightly wrong distribution.

Decode mode is observed through a PROBE MODEL the engine runs unchanged: D = 256, H = 2, one layer with every weight
zero (each layer adds exactly 0), pos_emb = 0, tok_emb[t] = one-hot at column t mod 255, the speaker projection reads
spk_emb[0] into column 255, lm_head entries on the 1/256 grid (bf16-exact).  Each logit is then one product or an exact
sum of two, so split-K order cannot change it, and mvb_s1_step_logits returns bit for bit the normalised logits both
stage-1 samplers consume (asserted: two calls agree).  The fed token selects the distribution; forced tokens set the
sequence.  Which body and sampler ran is taken from the launch-count delta."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy import stats

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

U = 2.0 ** -24
EXP_REL = 2.0 ** -22
LOGF_REL = 2.0 ** -23
ABS_UF = 2.0 ** -126
N_K = {"k_sample": 13, "fused": 42, "s2": 19}
ALPHA = 1e-6
BLOCK = 2048
D, H, F = 256, 2, 256
N_COL = 255                     # token t selects lm_head column t mod 255; column 255 carries the speaker value
FLAT_COL, EOA_COL = 0, 1        # column 0: every logit equal; column 1: token V - 1 certain
CHAIN = (250, 251, 252)         # token 250 -> 251 -> 252 -> 1 -> V - 1, each certain
GEN_BURST = 32


# ---------------------------------------------------------------------------------------------------------------------
# float64 reference
def keys_s1(lc, lu, g, T):
    g32 = np.float32(g)
    omg = np.float32(1.0) - g32
    t = max(np.float32(T), np.float32(1e-5))
    return ((g32 * np.asarray(lc, np.float32)) + (omg * np.asarray(lu, np.float32))) / t


def keys_s2(l, T):
    return np.asarray(l, np.float32) / np.float32(T)


def philox_x(v, c1, c2, c3, seed):
    """First output word of Philox4x32-10 for counters (v, c1, c2, c3) (broadcast) and key (seed lo, seed hi)."""
    M = np.uint64(0xFFFFFFFF)
    c0, c1, c2, c3 = (np.asarray(c, np.uint64) & M for c in np.broadcast_arrays(*(np.asarray(c, np.int64) for c in (v, c1, c2, c3))))
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M, (k1 + np.uint64(0xBB67AE85)) & M
    return c0


def philox_q(V, c1, c2, c3, seed):
    """The Exp(1) draws of sampler calls (counters c1..c3 broadcast against the entry index on the last axis):
    uni = ((x >> 8) + 0.5) * 2^-24 in fp32, q = -log(uni) in float64."""
    x = philox_x(np.arange(V), c1, c2, c3, seed)
    uni = ((x >> np.uint64(8)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -24)
    return -np.log(np.minimum(uni, np.float32(1 - 2.0 ** -24)).astype(np.float64))


def reference(k, top_p=None, top_k=None, q=None, flip=(), kept_override=None, strict=False, desc_ties=False,
              topk_drop_ties=False, no_keep_last=False):
    """float64 semantics from the fp32 keys k [V].  flip: entries whose top-p decision is inverted (band variants);
    kept_override: use this kept set for p / token.  The remaining flags are the altered references of the sensitivity
    checks."""
    V = k.size
    kd = k.astype(np.float64)
    idx = np.arange(V)
    order = np.lexsort((-idx if desc_ties else idx, kd))
    alive = np.ones(V, bool)
    if top_k is not None and top_k > 0:
        kk = min(int(top_k), V)
        if topk_drop_ties:
            alive = np.zeros(V, bool)
            alive[order[V - kk:]] = True
        else:
            alive = kd >= np.sort(kd)[V - kk]
    m = kd.max()
    with np.errstate(invalid="ignore"):
        e = np.where(alive, np.exp(kd - m), 0.0)
    cs = np.cumsum(e[order])
    cum = np.empty(V)
    cum[order] = cs / cs[-1]
    thr = None
    kept = alive.copy()
    if top_p is not None and top_p > 0:
        thr = float(np.float32(1.0) - np.float32(top_p))
        drop = (cum < thr) if strict else (cum <= thr)
        if not no_keep_last:
            drop[order[-1]] = False
        drop[list(flip)] = ~drop[list(flip)]
        kept = alive & ~drop
    if kept_override is not None:
        kept = kept_override & alive
    ek = np.where(kept, e, 0.0)
    tot = ek.sum()
    p = ek / tot if tot > 0 else np.zeros(V)
    r = dict(k=kd, m=m, e=e, cum=cum, thr=thr, kept=kept, alive=alive, p=p, order=order)
    if q is not None:
        s = p / np.asarray(q, np.float64)
        r["score"] = s
        r["token"] = int(np.argmax(s))
    return r


def a_terms(r):
    """(a_i per entry, a = max over entries with normal e)."""
    d = r["k"] - r["m"]
    a_i = EXP_REL + U * np.abs(d)
    ok = r["alive"] & (d >= -87)
    return a_i, float(a_i[ok].max()) if ok.any() else EXP_REL


def delta_cum(r, sampler, V):
    if np.all(r["k"][r["alive"]] == r["m"]):
        return 0.0                          # all keys equal: every partial sum is an exact integer
    _, a = a_terms(r)
    n = 44 if sampler != "fused" else V / 32 + V / 128 + 13
    return 1.01 * (2 * a + n * U) + V * ABS_UF


def band(r, delta):
    """Entries whose top-p decision the kernel may take either way (and which are alive with a normal e)."""
    if r["thr"] is None or r["thr"] == 0.0 or delta == 0.0:
        return np.zeros(0, int)        # thr = 0: every kept cum is > 0 in the kernels too; delta = 0: exact
    b = (np.abs(r["cum"] - r["thr"]) <= delta) & r["alive"] & (r["k"] - r["m"] >= -87)
    b[r["order"][-1]] = False           # never dropped
    return np.nonzero(b)[0]


def rho(r, sampler, philox):
    _, a = a_terms(r)
    return 1.01 * (2 * a + (N_K[sampler] + 2) * U + (LOGF_REL if philox else 0.0))


def prepare(k, sampler, philox=False, **kw):
    """The reference variants of one key vector: the float64 kept set and every inversion of the top-p decisions in the
    band, each with its probabilities and near-tie factor (1 - rho) / (1 + rho).  Returns (variants, n_band)."""
    r0 = reference(k, **kw)
    b = band(r0, delta_cum(r0, sampler, k.size))
    assert b.size <= 6, f"{b.size} entries in the top-p band"
    out = []
    for mask in range(2 ** b.size):
        r = r0 if mask == 0 else reference(k, flip=[int(b[i]) for i in range(b.size) if mask >> i & 1], **kw)
        rh = rho(r, sampler, philox)
        out.append((r["p"], (1 - rh) / (1 + rh)))
    return out, int(b.size)


def judge(tok, q, variants):
    """(ok, near_tie): the kernel's token is the float64 arg-max of p / q for some variant, or within its certified
    margin of it."""
    ok = near = False
    for p, lim in variants:
        s = p / np.asarray(q, np.float64)
        j = int(np.argmax(s))
        if s.size > 1:
            top2 = np.partition(s, s.size - 2)[-2:]
            near = near or bool(top2[0] >= top2[1] * lim and top2[1] > 0)
        ok = ok or tok == j or bool(s[tok] >= s[j] * lim and s[tok] > 0)
    return ok, near


def token_ok(tok, k, q, sampler, philox=False, **kw):
    """(ok, near_tie, n_band) for one draw."""
    variants, nb = prepare(k, sampler, philox, **kw)
    return (*judge(tok, q, variants), nb)


def check_api_draw(tok, probs, k, q, top_p, top_k, label, philox=False):
    """k_sample API mode: kept set, probabilities and token.  Returns (worst |err|/bound, n_band, near_tie)."""
    V = k.size
    r = reference(k, top_p=top_p, top_k=top_k, q=q)
    dc = delta_cum(r, "k_sample", V)
    b = band(r, dc)
    normal = ~r["alive"] | (r["k"] - r["m"] >= -80)
    got_kept = probs > 0
    mism = (got_kept != r["kept"]) & normal
    mism[b] = False
    assert not mism.any(), f"{label}: kept set differs outside the band at {np.nonzero(mism)[0][:8].tolist()}"
    r2 = reference(k, top_p=top_p, top_k=top_k, q=q, kept_override=got_kept | (r["kept"] & ~normal))
    a_i, a = a_terms(r2)
    beta = 1.01 * (a_i + a + 14 * U)
    if dc == 0.0:
        beta = np.full(V, U)
    err = np.abs(probs.astype(np.float64) - r2["p"])
    bound = beta * r2["p"] + 2.0 ** -125
    bad = np.nonzero(err > bound)[0]
    assert bad.size == 0, f"{label}: probs over the bound at {bad[:8].tolist()} (max ratio {float((err / bound).max()):.2e})"
    ok, near, nb = token_ok(int(tok), k, q, "k_sample", philox, top_p=top_p, top_k=top_k)
    assert ok, f"{label}: token {int(tok)} vs float64 {r['token']} (not a certified near-tie)"
    return float((err / bound).max()), nb, near


def chi2(counts, p):
    """Pearson chi-square p-value of observed counts against probabilities p, bins of expected count < 5 merged."""
    n = counts.sum()
    exp_ = p * n
    big = exp_ >= 5
    obs = np.append(counts[big], counts[~big].sum())
    ex = np.append(exp_[big], exp_[~big].sum())
    keep = ex > 0
    if (obs[~keep] > 0).any():
        return 0.0, len(obs) - 1
    obs, ex = obs[keep], ex[keep]
    stat = float(((obs - ex) ** 2 / ex).sum())
    dof = len(obs) - 1
    return float(stats.chi2.sf(stat, dof)), dof


# ---------------------------------------------------------------------------------------------------------------------
# engines
def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Probe:
    """The probe model of the module docstring at vocabulary V for `utts` utterance slots; tc and mode are
    setup_caches' tensor_core_path and from_state_dict's quantisation_mode."""

    def __init__(self, V, utts, fused=True, seed=0, tc=None, mode=None, n_sm=None):
        """n_sm: the SM count the engine is planned for (default: this device's)."""
        from mvb200.fast_model import ModelArgs, Transformer
        self.V, self.n_sm = V, n_sm or _n_sm()
        rng = np.random.default_rng(seed + V)
        tok = np.zeros((V, D), np.float32)
        tok[np.arange(V), np.arange(V) % N_COL] = 1.0
        sig = rng.uniform(0.04, 0.3, N_COL)          # normalised logit ~ 14 W: sigma ~ 0.6 .. 4
        W = np.zeros((V, D), np.float32)
        W[:, :N_COL] = np.clip(np.round(rng.standard_normal((V, N_COL)) * sig * 256), -255, 255) / 256
        W[:, FLAT_COL] = 0.25
        W[:, EOA_COL] = 0.0
        W[V - 1, EOA_COL] = 8.0
        if V > CHAIN[-1]:
            for c, nxt in zip(CHAIN, CHAIN[1:] + (EOA_COL,)):
                W[:, c] = 0.0
                W[nxt, c] = 8.0
        W[:, N_COL] = np.clip(np.round(rng.standard_normal(V) * 0.1 * 256), -255, 255) / 256
        wspk = np.zeros((D, 256), np.float32)
        wspk[N_COL, 0] = 1.0
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a))  # noqa: E731
        sd = {"transformer.wtes.0.weight": t(tok), "transformer.wpe.weight": torch.zeros(BLOCK, D),
              "speaker_cond_pos.weight": t(wspk), "transformer.ln_f.weight": torch.ones(D), "lm_heads.0.weight": t(W),
              "transformer.h.0.ln_1.weight": torch.ones(D), "transformer.h.0.attn.c_attn.weight": torch.zeros(3 * D, D),
              "transformer.h.0.attn.c_proj.weight": torch.zeros(D, D), "transformer.h.0.ln_2.weight": torch.ones(D),
              "transformer.h.0.mlp.swiglu.w1.weight": torch.zeros(F, D),
              "transformer.h.0.mlp.swiglu.w3.weight": torch.zeros(F, D),
              "transformer.h.0.mlp.c_proj.weight": torch.zeros(D, F)}
        sd = {k: v.to(torch.bfloat16) for k, v in sd.items()}
        cfg = ModelArgs(block_size=BLOCK, vocab_size=V, n_layer=1, n_head=H, dim=D, intermediate_size=F)
        self.m = Transformer.from_state_dict(sd, cfg, device="cuda:0", quantisation_mode=mode)
        self.m.setup_caches(2 * utts, BLOCK, tensor_core_path=tc, unfused_sampler=not fused)
        self.fused, self.utts = fused, utts
        self.lib, self.h = self.m._lib, self.m.handle
        self._keep = []

    def close(self):
        self.m.close()

    def st(self):
        return self.m._stream()

    def launches(self):
        return int(self.lib.mvb_s1_launch_count(self.h))

    def set_speakers(self, vals):
        for u, c in enumerate(vals):
            e = torch.zeros(256)
            e[0] = float(c)
            self.m.set_speaker(u, e)

    def begin(self, u, first, sp, noise=None, forced=None):
        from mvb200 import _lib
        _lib.check(self.lib.mvb_s1_begin(self.h, u, int(first), 0, C.byref(sp), noise, forced, self.st()))

    def logits(self, toks):
        """Normalised logits [2 n, V] (fp32 numpy) of step_logits with slot u fed toks[u]; two calls must agree."""
        from mvb200 import _lib
        n = len(toks)
        outs = []
        for _ in range(2):
            for u, t in enumerate(toks):
                self.begin(u, t, _lib.Sampling(1.0, 1.0, 0.0, 0, 9999, 1))
            lg = torch.empty(2 * n, self.V, device="cuda")
            _lib.check(self.lib.mvb_s1_step_logits(self.h, n, lg.data_ptr(), self.st()))
            torch.cuda.synchronize()
            outs.append(lg.cpu().numpy())
        assert np.array_equal(outs[0], outs[1]), "step_logits is not bit-reproducible on the probe"
        return outs[0]

    def table(self, n, tokens):
        """{token: [2 n, V]} for every token in `tokens` (all n slots fed that token)."""
        return {t: self.logits([t] * n) for t in sorted(set(int(x) for x in tokens))}

    def body(self, n, top_k_any=False):
        """(sampler, per-step launches) mvb_s1_decode must run for n utterances, and whether it is one fused launch."""
        from test_sm_count_cpu import fused_ok, path_c
        if path_c((D, H, F, self.V), self.n_sm, n, "bf16", BLOCK):
            if self.fused and not top_k_any and fused_ok(self.n_sm, self.V):
                return "fused"
            return "C+k_sample"
        return "B+k_sample" if n >= 2 else "A+k_sample"


LAUNCHES_PER_STEP = {"C+k_sample": 2, "B+k_sample": 14, "A+k_sample": 8}


def run_decode(p, slots, n_steps, seed):
    """One mvb_s1_decode burst.  slots: list of dicts g, T, top_p, top_k, fed (n_steps + 1 tokens; None = no forcing,
    fed[0] only), noise (True: supplied Exp(1) [n_steps, V]; False: Philox), seed, eoa.  Returns (sampled [n, n_steps],
    noise per slot, sampler that ran)."""
    from mvb200 import _lib
    n, V = len(slots), p.V
    rng = np.random.default_rng(seed)
    keep, noises = [], []
    top_k_any = any((s.get("top_k") or 0) > 0 for s in slots)
    for u, s in enumerate(slots):
        sp = _lib.Sampling(s["g"], s["T"], s.get("top_p") or 0.0, s.get("top_k") or 0, s.get("eoa", 9999), s.get("seed", 1))
        q = None
        if s.get("noise", True):
            q = rng.exponential(size=(n_steps, V)).astype(np.float32)
            if "design" in s:
                q = s["design"](q)
            qd = torch.from_numpy(q).cuda()
            keep.append(qd)
        noises.append(q)
        fd = None
        if s["fed"] is not None and len(s["fed"]) > 1:
            f = np.zeros(BLOCK, np.int32)
            f[:len(s["fed"]) - 1] = s["fed"][1:]
            fd = torch.from_numpy(f).cuda()
            keep.append(fd)
        p.begin(u, s["fed"][0], sp, None if q is None else qd.data_ptr(), None if fd is None else fd.data_ptr())
    n0 = p.launches()
    _lib.check(p.lib.mvb_s1_decode(p.h, n, n_steps, p.st()))
    torch.cuda.synchronize()
    body = p.body(n, top_k_any)
    want = 2 if body == "fused" else 1 + n_steps * LAUNCHES_PER_STEP[body]
    assert p.launches() - n0 == want, f"V={V} n={n}: expected {body} ({want} launches), got {p.launches() - n0}"
    out = np.zeros((n, n_steps), np.int32)
    for u in range(n):
        buf = (C.c_int32 * n_steps)()
        _lib.check(p.lib.mvb_s1_fetch_sampled(p.h, u, buf, n_steps, p.st()))
        out[u] = np.frombuffer(buf, np.int32)
    del keep
    return out, noises, body


def check_decode(p, slots, sampled, noises, table, body, label, skip=()):
    """Every draw of every slot (except `skip`) against the float64 reference; returns (draws, near-ties, band)."""
    sampler = "fused" if body == "fused" else "k_sample"
    n = len(slots)
    draws = near = nb = 0
    for u, s in enumerate(slots):
        if u in skip:
            continue
        philox = noises[u] is None
        n_steps = sampled.shape[1]
        Q = philox_q(p.V, np.arange(n_steps)[:, None], 0, u, s.get("seed", 1)) if philox else noises[u]
        prep = {}
        for i in range(n_steps):
            t = int(s["fed"][i])
            if t not in prep:
                lg = table[t]
                k = keys_s1(lg[2 * u], lg[2 * u + 1], s["g"], s["T"])
                prep[t] = prepare(k, sampler, philox, top_p=s.get("top_p"), top_k=s.get("top_k"))
            ok, nt = judge(int(sampled[u, i]), Q[i], prep[t][0])
            assert ok, f"{label} [{body}] slot {u} step {i}: token {int(sampled[u, i])} is not the float64 draw"
            draws, near, nb = draws + 1, near + int(nt), nb + prep[t][1]
    assert draws > near, f"{label}: every draw is a near-tie"
    return draws, near, nb


@pytest.fixture(scope="module")
def probes():
    cache = {}

    def get(V, utts, fused=True):
        key = (V, utts, fused)
        if key not in cache:
            for k in list(cache):
                cache.pop(k).close()
            torch.cuda.empty_cache()
            cache[key] = Probe(V, utts, fused)
        return cache[key]
    yield get
    for v in cache.values():
        v.close()


# ---------------------------------------------------------------------------------------------------------------------
# stage 1, API mode (mvb_s1_sample)
V_API = [2, 130, 2562, 4096]        # 2: the smallest even vocabulary mvb_s1_create accepts
GUID = [3.0, 1.0, 0.0]
TEMP = [1.0, 0.7, 1e-6]
TOP_P = [None, 0.95, 0.5, 1e-3, 1.0, 1e-9]
REGIMES = ["gauss1", "gauss5", "gauss40", "bf16", "needle", "equal", "plateau"]


def _top_k(V):
    return [None, 1, 200, V - 1, V, V + 5]


def api_logits(V, regime, rng):
    n = lambda s: rng.standard_normal(V) * s  # noqa: E731
    if regime.startswith("gauss"):
        s = float(regime[5:])
        lc = n(s)
        lu = lc + n(s / 4)
    elif regime == "bf16":
        grid = np.arange(-8, 9) / 4.0
        lc, lu = rng.choice(grid, V), rng.choice(grid[::2], V)
    elif regime == "needle":
        lc, lu = n(1), n(1)
        lc[rng.integers(V)] += 30
    elif regime == "equal":
        lc, lu = np.full(V, 0.75), np.full(V, -0.25)
    elif regime == "plateau":       # two tie groups; the top-p boundary falls inside the upper one
        hi = rng.permutation(V) < (V + 1) // 2
        lc = np.where(hi, 0.0, -3.0)
        lu = lc.copy()
    return np.stack([lc, lu]).astype(np.float32)


def run_api(p, lg, q, combos, step=0, noise=True):
    """mvb_s1_sample for every (g, T, top_p, top_k) combo on logits lg [2, V]: tokens [n], probs [n, V]."""
    from mvb200 import _lib
    V, n = p.V, len(combos)
    lgd = torch.from_numpy(lg).cuda()
    qd = torch.from_numpy(q).cuda() if noise else None
    tok = torch.empty(n, dtype=torch.int32, device="cuda")
    probs = torch.empty(n, V, device="cuda")
    n0 = p.launches()
    for i, (g, T, tp, tk) in enumerate(combos):
        sp = _lib.Sampling(g, T, tp or 0.0, tk or 0, 9999, 7)
        _lib.check(p.lib.mvb_s1_sample(p.h, lgd.data_ptr(), C.byref(sp), None if qd is None else qd.data_ptr(),
                                       step + i if not noise else step, tok[i:].data_ptr(), probs[i].data_ptr(), p.st()))
    torch.cuda.synchronize()
    assert p.launches() - n0 == n
    return tok.cpu().numpy(), probs.cpu().numpy()


@pytest.mark.parametrize("V", V_API)
def test_api_sampler_grid(probes, V):
    """Every (guidance, temperature, top_p, top_k) of the grid on seven logit regimes: probs_out (exact zeros where an
    entry is dropped), the kept set and the token under supplied noise."""
    p = probes(V, 1)
    rng = np.random.default_rng(V)
    combos = [(g, T, tp, tk) for g in GUID for T in TEMP for tp in TOP_P for tk in _top_k(V)]
    worst = 0.0
    nb = near = draws = 0
    band_plain = 0
    for regime in REGIMES:
        lg = api_logits(V, regime, rng)
        q = rng.exponential(size=V).astype(np.float32)
        toks, probs = run_api(p, lg, q, combos)
        for i, (g, T, tp, tk) in enumerate(combos):
            k = keys_s1(lg[0], lg[1], g, T)
            w, b, nt = check_api_draw(toks[i], probs[i], k, q, tp, tk, f"V={V} {regime} g={g} T={T} top_p={tp} top_k={tk}")
            worst, nb, near, draws = max(worst, w), nb + b, near + int(nt), draws + 1
            if regime in ("equal", "needle"):
                band_plain += b
    assert draws > near
    assert band_plain == 0, f"{band_plain} band entries in the equal / needle regimes"
    print(f"k_sample API V={V}: {draws} draws (7 regimes x {len(combos)} parameter sets): max |err|/bound {worst:.2e}, "
          f"{nb} entries in the top-p band, {near} certified near-ties")


def test_api_flat_tie_order_exact(probes):
    """V = 4096, all keys equal, top_p = 0.5: cum is exactly i / 4096, so the kept set is exactly 2048 ... 4095 with
    probability 1/2048 each; top_p = 1e-9 keeps only 4095; top_k = 200 keeps every tie at the pivot."""
    p = probes(4096, 1)
    lg = api_logits(4096, "equal", np.random.default_rng(0))
    q = np.random.default_rng(1).exponential(size=4096).astype(np.float32)
    toks, probs = run_api(p, lg, q, [(3.0, 1.0, 0.5, None), (3.0, 1.0, 1e-9, None), (3.0, 1.0, None, 200)])
    want = np.zeros(4096, np.float32)
    want[2048:] = 1 / 2048
    assert np.array_equal(probs[0], want)
    assert int(toks[0]) == 2048 + int(np.argmin(q[2048:]))
    assert np.array_equal(np.nonzero(probs[1])[0], [4095]) and probs[1][4095] == 1.0 and toks[1] == 4095
    assert np.all(probs[2] == np.float32(1 / 4096))


def test_api_reference_matches_oracle_and_golden(golden_dir):
    """The float64 restatement against oracle/stage1_port.sample and tests/golden/sampler.npz (tie-free cases)."""
    from oracle import stage1_port as P
    g = np.load(f"{golden_dir}/sampler.npz")
    for c in range(g["idx"].shape[0]):
        gs, temp, tp, tk = [float(v) for v in g["params"][c]]
        tp, tk = (None if tp < 0 else tp), (None if tk == 0 else int(tk))
        lg = g["logits"][c]
        k = keys_s1(lg[0], lg[1], gs, temp)
        r = reference(k, top_p=tp, top_k=tk, q=g["noise"][c])
        assert r["token"] == int(g["idx"][c])
        assert np.array_equal(r["p"] > 0, g["probs"][c] > 0)
        np.testing.assert_allclose(r["p"], g["probs"][c], rtol=2e-5, atol=1e-9)
    rng = np.random.default_rng(3)
    for i in range(40):
        V = [130, 2562][i % 2]
        lg = rng.standard_normal((2, V)).astype(np.float32) * [1, 3, 8, 0.5][i % 4]
        gs, temp, tp, tk = [3.0, 1.0, 0.0][i % 3], [1.0, 0.7][i % 2], [None, 0.9, 0.5][i % 3], [None, 50][i % 2]
        q = rng.exponential(size=V).astype(np.float32)
        t = lambda a: torch.from_numpy(np.asarray(a, np.float32))  # noqa: E731
        idx, probs, kept = P.sample(t(lg)[:, None, :], t(gs), t(temp), None if tp is None else t(tp), tk, q=t(q),
                                    return_kept=True)
        r = reference(keys_s1(lg[0], lg[1], gs, temp), top_p=tp, top_k=tk, q=q)
        differ = r["kept"] != kept.numpy()
        differ[band(r, 1e-5)] = False                     # torch forms cum in fp32
        assert not differ.any()
        np.testing.assert_allclose(r["p"], probs.double().numpy(), rtol=1e-5, atol=1e-12)
        assert r["token"] == int(idx)


# ---------------------------------------------------------------------------------------------------------------------
# stage 1 in the decode loop
SLOT_PARAMS = [(3.0, 1.0, 0.95), (1.0, 0.7, None), (0.0, 1.0, 0.5), (2.0, 1.3, 0.9),
               (3.0, 1e-6, 0.95), (1.5, 1.0, 1e-3), (3.0, 0.5, 1.0), (-1.0, 1.0, 0.8)]
SPK = [0.5, 1.0, 0.25, 0.5, 0.75, 0.5, 1.0, 0.25]


def _slots(n, V, n_steps, rng, top_k=None):
    hi = min(V, N_COL)
    out = []
    for u in range(n):
        g, T, tp = SLOT_PARAMS[u % 8]
        fed = rng.integers(2, hi, n_steps + 1)
        fed = fed[(fed < CHAIN[0]) | (fed > CHAIN[-1])] if V > CHAIN[-1] else fed
        fed = np.resize(fed, n_steps + 1)
        out.append(dict(g=g, T=T, top_p=tp, top_k=(top_k if u % 2 == 0 else None) if top_k else None, fed=fed))
    return out


DECODE_CASES = [  # (V, utterances, fused engine, top_k on even slots)
    (130, 1, True, None), (130, 8, True, None), (2562, 1, True, None), (2562, 8, True, None),
    (4096, 1, True, None), (4096, 8, True, None),
    (2562, 8, False, None), (4096, 8, False, None), (2562, 8, True, 40), (130, 8, True, 200),
    (2562, 12, True, None), (4096, 12, True, 40),
]


@pytest.mark.parametrize("V,n,fused,top_k", DECODE_CASES)
def test_decode_burst_supplied_noise(probes, V, n, fused, top_k):
    """A 40-step mvb_s1_decode burst, every slot with its own guidance / temperature / top_p (and top_k > 0 on even
    slots, which forces k_sample), forced tokens, supplied noise: every draw against the float64 reference.  The body
    (one fused launch; persistent + k_sample per step; path B + k_sample) is asserted from the launch count."""
    burst_supplied_noise(probes(V, 12 if n > 8 else 8, fused), n, top_k)


def burst_supplied_noise(p, n, top_k):
    """test_decode_burst_supplied_noise on probe p; returns the sampler that ran."""
    V, fused = p.V, p.fused
    rng = np.random.default_rng(V + n + (top_k or 0))
    n_steps = 40
    slots = _slots(n, V, n_steps, rng, top_k)
    p.set_speakers([SPK[u % 8] for u in range(n)])
    table = p.table(n, np.concatenate([s["fed"] for s in slots]))
    sampled, noises, body = run_decode(p, slots, n_steps, seed=V + n)
    if fused and top_k is None and n <= 8:
        assert body == "fused" or -(-V // p.n_sm) > 32
    draws, near, nb = check_decode(p, slots, sampled, noises, table, body, f"V={V} n={n}")
    print(f"decode V={V}, {n} utterances [{body}] on {p.n_sm} SMs: {draws} draws, {near} certified near-ties, {nb} band entries")
    return body


def test_decode_eoa_latch_leaves_other_slots_alone(probes):
    """Slot 3 is fed token 250 and not forced: its draws are certain (250 -> 251 -> 252 -> 1 -> V - 1 = EOA), it latches
    at step 3 and stops; the seven other slots draw every one of their 30 steps as the reference says."""
    from mvb200 import _lib
    V, n, n_steps = 2562, 8, 30
    p = probes(V, 8)
    rng = np.random.default_rng(11)
    slots = _slots(n, V, n_steps, rng)
    slots[3] = dict(g=3.0, T=1.0, top_p=0.95, fed=np.array([CHAIN[0]]), eoa=V - 1)
    p.set_speakers(SPK)
    table = p.table(n, np.concatenate([s["fed"] for i, s in enumerate(slots) if i != 3]))
    sampled, noises, body = run_decode(p, slots, n_steps, seed=12)
    assert body == "fused"
    assert sampled[3, :4].tolist() == [CHAIN[1], CHAIN[2], EOA_COL, V - 1]
    n_out, done = C.c_int32(), C.c_int32()
    _lib.check(p.lib.mvb_s1_fetch(p.h, 3, None, 0, C.byref(n_out), C.byref(done), p.st()))
    assert (n_out.value, done.value) == (4, 1)
    check_decode(p, slots, sampled, noises, table, body, "EOA batch", skip=(3,))


def test_generate_host_noise_across_bursts(probes):
    """mvb_s1_generate with HOST noise for 110 tokens (the first from k_sample after the prefill, then bursts of 32, 32,
    32, 13 with the draws staged per burst and noise_base moving): every step of both utterances vs the reference."""
    from mvb200 import _lib
    V, n, n_new = 2562, 2, 3 * GEN_BURST + 14     # GEN_BURST: decode steps per staged chunk in mvb_s1_generate
    p = probes(V, 8)
    rng = np.random.default_rng(5)
    prompts = np.array([7, 9], np.int32)
    spk = np.zeros((n, 256), np.float32)
    spk[:, 0] = [0.5, 1.0]
    params = (_lib.Sampling * n)(_lib.Sampling(3.0, 1.0, 0.95, 0, 9999, 1), _lib.Sampling(1.5, 0.8, 0.5, 0, 9999, 2))
    forced = rng.integers(2, CHAIN[0], (n, n_new)).astype(np.int32)
    noise = rng.exponential(size=(n, n_new, V)).astype(np.float32)
    out = np.zeros((n, n_new), np.int32)
    lens = np.zeros(n, np.int32)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    plens = np.ones(n, np.int32)
    _lib.check(p.lib.mvb_s1_generate(p.h, n, ptr(prompts), ptr(plens), ptr(spk), params, n_new,
                                     ptr(noise), 0, ptr(forced), ptr(out), ptr(lens), p.st()))
    assert lens.tolist() == [n_new] * n and np.array_equal(out, forced)
    sampled = np.zeros((n, n_new), np.int32)
    for u in range(n):
        buf = (C.c_int32 * n_new)()
        _lib.check(p.lib.mvb_s1_fetch_sampled(p.h, u, buf, n_new, p.st()))
        sampled[u] = np.frombuffer(buf, np.int32)
    # step 0 reads the prefill's logits rows (path A, one position); steps >= 1 the decode body's
    pre = []
    for u in range(n):
        p.set_speakers([spk[0, 0], spk[1, 0]])
        idx = torch.tensor([[prompts[u]], [prompts[u]]], dtype=torch.int32, device="cuda")
        lg = torch.empty(2, V, device="cuda")
        _lib.check(p.lib.mvb_s1_forward(p.h, u, idx.data_ptr(), 1, 0, lg.data_ptr(), 0, p.st()))
        torch.cuda.synchronize()
        pre.append(lg.cpu().numpy())
    table = p.table(n, forced.ravel())
    draws = near = 0
    for u in range(n):
        sp = params[u]
        for i in range(n_new):
            lg = pre[u] if i == 0 else table[int(forced[u, i - 1])][2 * u:2 * u + 2]
            k = keys_s1(lg[0], lg[1], sp.guidance_scale, sp.temperature)
            ok, nt, _ = token_ok(int(sampled[u, i]), k, noise[u, i], "fused" if i else "k_sample", top_p=sp.top_p)
            assert ok, f"generate utt {u} step {i}: token {int(sampled[u, i])} is not the float64 draw"
            draws, near = draws + 1, near + int(nt)
    assert draws > near
    print(f"generate, host noise, {n_new} tokens x {n} (4 staged bursts): {draws} draws, {near} certified near-ties")


def _flat_design(q):
    q = 1.0 + 0.5 * q / q.max()
    for i, js in enumerate([(2047, 2048), (2048,), (4095,), (0, 3000), (2046, 2047, 2049), (2047, 0, 4095)]):
        for r, j in enumerate(js):
            q[i, j] = 0.01 * (r + 1)
    return q.astype(np.float32)


@pytest.mark.parametrize("fused", [True, False])
def test_decode_flat_tie_order_exact(probes, fused):
    """V = 4096, every logit equal, top_p = 0.5: the kept set is exactly 2048 ... 4095 in the fused ranking and in
    k_sample's sort.  Designed noise puts the smallest q on 2047 / 2048 / 4095 / 0: the tokens must be 2048, 2048,
    4095, 3000, 2049, 4095, and the remaining steps the argmin of q over 2048 ... 4095."""
    flat_tie_order(probes(4096, 8, fused))


def flat_tie_order(p):
    """test_decode_flat_tie_order_exact on probe p (V = 4096); returns the sampler that ran."""
    n_steps = 12
    slot = dict(g=3.0, T=1.0, top_p=0.5, fed=np.zeros(n_steps + 1, int), design=_flat_design)
    p.set_speakers([0.0])
    table = p.table(1, [0])
    lg = table[0]
    assert np.all(lg == lg[0, 0]), "the flat column does not give equal logits"
    sampled, noises, body = run_decode(p, [slot], n_steps, seed=3)
    assert body == ("fused" if p.fused and -(-4096 // p.n_sm) <= 32 else "C+k_sample")
    want = [2048 + int(np.argmin(noises[0][i, 2048:])) for i in range(n_steps)]
    assert want[:6] == [2048, 2048, 4095, 3000, 2049, 4095]
    assert sampled[0].tolist() == want
    return body


# ---------------------------------------------------------------------------------------------------------------------
# Philox streams
def _gof_slots(n, seed, top_p=0.9):
    return [dict(g=3.0, T=1.0, top_p=top_p, fed=np.full(2001, 5), noise=False, seed=seed) for _ in range(n)]


def test_philox_fused_vs_unfused_goodness_of_fit(probes):
    """8 slots x 2000 steps of one distribution (constant forced token), noise = NULL, all slots sharing one seed:
    every draw equals the float64 draw on the host-recomputed Philox stream (certified near-ties excepted); the pooled
    counts fit the float64 probabilities, pairs of consecutive tokens fit the product distribution, slots draw different
    streams, a rerun reproduces the tokens, the unfused engine draws the same tokens, and the same chi-square rejects
    temperature 1.1 and top_p off."""
    V, n, n_steps = 2562, 8, 2000
    res, tables = {}, {}
    for fused in (True, False):
        p = probes(V, 8, fused)
        p.set_speakers([0.5] * n)
        tables[fused] = p.table(n, [5])[5]
        runs = [run_decode(p, _gof_slots(n, 77), n_steps, seed=0) for _ in range(2 if fused else 1)]
        if fused:
            assert np.array_equal(runs[0][0], runs[1][0]), "a rerun with the same seed drew different tokens"
        res[fused] = (runs[0][0], runs[0][2])
    assert np.array_equal(tables[True], tables[False]), "the fused and unfused engines' step_logits differ"
    tf, body = res[True]
    tu, body_u = res[False]
    assert body == "fused" and body_u == "C+k_sample"
    lg = tables[True]
    k = keys_s1(lg[0], lg[1], 3.0, 1.0)
    r = reference(k, top_p=0.9)
    # every Philox draw of both samplers against the reference; disagreements only at certified near-ties
    prep = {smp: prepare(k, smp, True, top_p=0.9)[0] for smp in ("fused", "k_sample")}
    near = diff = 0
    for u in range(n):
        Q = philox_q(V, np.arange(n_steps)[:, None], 0, u, 77)
        for i in range(n_steps):
            for tok, smp in ((tf[u, i], "fused"), (tu[u, i], "k_sample")):
                ok, nt = judge(int(tok), Q[i], prep[smp])
                assert ok, f"Philox draw slot {u} step {i} ({smp}): token {int(tok)} is not the float64 draw"
            near += int(nt)
            if tf[u, i] != tu[u, i]:
                assert nt, f"fused and unfused disagree at slot {u} step {i} without a near-tie"
                diff += 1
    counts = np.bincount(tf.ravel(), minlength=V).astype(np.float64)
    pv, dof = chi2(counts, r["p"])
    assert pv > ALPHA, f"fused Philox tokens do not fit the float64 probabilities (p = {pv:.2e}, {dof} dof)"
    # independence: pairs of consecutive tokens on the 4 most probable tokens + the rest
    top = np.argsort(r["p"])[-4:]
    st = np.sort(top)
    pc = np.append(r["p"][st], 1 - r["p"][st].sum())
    c = np.where(np.isin(tf, st), np.searchsorted(st, tf), 4)
    pairs = (c[:, :-1] * 5 + c[:, 1:]).ravel()
    pv2, dof2 = chi2(np.bincount(pairs, minlength=25).astype(np.float64), np.outer(pc, pc).ravel())
    assert pv2 > ALPHA, f"consecutive Philox tokens are not independent (p = {pv2:.2e})"
    same = np.mean([np.mean(tf[a] == tf[b]) for a in range(n) for b in range(a)])
    assert same < (r["p"] ** 2).sum() + 0.05, f"slots sharing a seed draw the same stream ({same:.2f} agreement)"
    # power
    pv_t, _ = chi2(counts, reference(keys_s1(lg[0], lg[1], 3.0, 1.1), top_p=0.9)["p"])
    pv_p, _ = chi2(counts, reference(k)["p"])
    assert pv_t < ALPHA and pv_p < ALPHA, f"the chi-square does not see a biased stream (T 1.1: {pv_t:.1e}, top_p off: {pv_p:.1e})"
    print(f"Philox fused / unfused, {n} x {n_steps} draws: chi-square p = {pv:.3f} ({dof} dof), pairs p = {pv2:.3f} "
          f"({dof2} dof), cross-slot agreement {same:.3f} (sum p^2 = {(r['p'] ** 2).sum():.3f}), {near} near-ties, "
          f"{diff} fused/unfused differences; power: T = 1.1 p = {pv_t:.1e}, top_p off p = {pv_p:.1e}")


def test_philox_top_word_never_draws_a_dropped_entry(probes):
    """Seed 7 gives the Philox word x >> 8 = 2^24 - 1 at (entry 3094, step 35, slot 0): (x >> 8) + 0.5 rounds to 2^24 in
    fp32, so without the clamp uni = 1, q = -0 and the score of that entry (-inf, or NaN when its probability is 0)
    wins the arg-max.  k_sample API mode with top_k = 1, and both decode samplers on token 1 (only V - 1 has a nonzero
    probability), must not draw entry 3094 at step 35."""
    assert int(philox_x(np.array([3094]), 35, 0, 0, 7)[0] >> np.uint64(8)) == 0xFFFFFF
    p = probes(4096, 1)
    lg = api_logits(4096, "needle", np.random.default_rng(2))
    toks, probs = run_api(p, lg, None, [(3.0, 1.0, None, 1)], step=35, noise=False)
    assert int(toks[0]) == int(np.argmax(keys_s1(lg[0], lg[1], 3.0, 1.0))) != 3094
    for fused in (True, False):
        pp = probes(4096, 8, fused)
        pp.set_speakers([0.5])
        slot = dict(g=3.0, T=1.0, top_p=None, fed=np.full(37, EOA_COL), noise=False, seed=7)
        sampled, _, body = run_decode(pp, [slot], 36, seed=0)
        assert body == ("fused" if fused else "C+k_sample")
        assert np.all(sampled[0] == 4095), f"{body}: drew {sorted(set(sampled[0].tolist()) - {4095})}"


def test_philox_api_mode_goodness_of_fit(probes):
    """k_sample API mode, noise = NULL, steps 0 ... 2999: every draw vs the host Philox stream (slot 0), counts vs the
    float64 probabilities, and the power check."""
    V, N = 2562, 3000
    p = probes(V, 1)
    rng = np.random.default_rng(9)
    lg = api_logits(V, "gauss5", rng)
    combos = [(3.0, 1.0, 0.9, None)] * N
    toks, _ = run_api(p, lg, None, combos, step=0, noise=False)
    k = keys_s1(lg[0], lg[1], 3.0, 1.0)
    r = reference(k, top_p=0.9)
    near = 0
    prep = prepare(k, "k_sample", True, top_p=0.9)[0]
    Q = philox_q(V, np.arange(N)[:, None], 0, 0, 7)
    for i in range(N):
        ok, nt = judge(int(toks[i]), Q[i], prep)
        assert ok, f"API Philox step {i}: token {int(toks[i])} is not the float64 draw"
        near += int(nt)
    counts = np.bincount(toks, minlength=V).astype(np.float64)
    pv, dof = chi2(counts, r["p"])
    assert pv > ALPHA
    pv_t, _ = chi2(counts, reference(keys_s1(lg[0], lg[1], 3.0, 1.1), top_p=0.9)["p"])
    assert pv_t < ALPHA
    print(f"Philox k_sample API, {N} steps: chi-square p = {pv:.3f} ({dof} dof), {near} near-ties; T = 1.1: p = {pv_t:.1e}")


# ---------------------------------------------------------------------------------------------------------------------
# stage 2: k_s2_sample through mvb_s2_sample_test
def s2_sample(logits, T, top_k, noise=None, seed=0):
    """logits [n_hier, n_rows, V] fp32 numpy -> tokens [n_hier, n_rows]."""
    from mvb200 import _lib
    lib = _lib.load()
    nh, nr, V = logits.shape
    prm = np.zeros(4, np.uint32)
    prm[0] = np.float32(T).view(np.uint32)
    prm[1] = np.int32(top_k).view(np.uint32)
    prm[2], prm[3] = seed & 0xFFFFFFFF, seed >> 32
    prm_d = torch.from_numpy(prm.view(np.int32)).cuda()
    lg = torch.from_numpy(np.ascontiguousarray(logits)).cuda()
    nz = torch.from_numpy(np.ascontiguousarray(noise)).cuda() if noise is not None else None
    out = torch.full((nh * nr + 8,), -1, dtype=torch.int32, device="cuda")
    _lib.check(lib.mvb_s2_sample_test(lg.data_ptr(), nh, nr, V, prm_d.data_ptr(), None if nz is None else nz.data_ptr(),
                                      out.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    o = out.cpu().numpy()
    assert np.all(o[nh * nr:] == -1), "the sampler wrote past [n_hier, n_rows]"
    return o[:nh * nr].reshape(nh, nr)


def s2_logits(V, nh, nr, rng):
    """Half the rows Gaussian (sigma 2), half on a coarse grid (ties at every top-k pivot)."""
    g = rng.standard_normal((nh, nr, V)) * 2
    t = rng.integers(-6, 7, (nh, nr, V)) / 2.0
    return np.where(np.arange(nr)[None, :, None] % 2 == 0, g, t).astype(np.float32)


@pytest.mark.parametrize("V", [2, 1025, 2048])
def test_stage2_sampler(V):
    """top_k in {0, 1, 200, V - 1, V, V + 1} x temperature {0.5, 1, 3}, 2 hierarchies x 64 rows, supplied noise."""
    rng = np.random.default_rng(V)
    nh, nr = 2, 64
    draws = near = 0
    for top_k in [0, 1, 200, V - 1, V, V + 1]:
        for T in [0.5, 1.0, 3.0]:
            lg = s2_logits(V, nh, nr, rng)
            q = rng.exponential(size=lg.shape).astype(np.float32)
            tok = s2_sample(lg, T, top_k, q)
            for h in range(nh):
                for r_ in range(nr):
                    k = keys_s2(lg[h, r_], T)
                    ok, nt, _ = token_ok(int(tok[h, r_]), k, q[h, r_], "s2", top_k=top_k or None)
                    assert ok, f"k_s2_sample V={V} top_k={top_k} T={T} ({h}, {r_}): token {int(tok[h, r_])}"
                    draws, near = draws + 1, near + int(nt)
    assert draws > near
    print(f"k_s2_sample V={V}: {draws} draws, {near} certified near-ties")


def test_stage2_philox_goodness_of_fit():
    """One call, 6 hierarchies x 2048 identical rows, noise = NULL: every draw vs the host Philox stream (counters
    (entry, row, hierarchy, 0x5eed2)), counts vs the float64 probabilities; the chi-square rejects temperature 1.1."""
    V, nh, nr, seed = 1025, 6, 2048, 0x1234567890
    rng = np.random.default_rng(4)
    row = (rng.standard_normal(V) * 2).astype(np.float32)
    lg = np.broadcast_to(row, (nh, nr, V)).copy()
    tok = s2_sample(lg, 1.0, 200, None, seed)
    k = keys_s2(row, 1.0)
    r = reference(k, top_k=200)
    near = 0
    prep = prepare(k, "s2", True, top_k=200)[0]
    for h in range(nh):
        Q = philox_q(V, np.arange(nr)[:, None], h, 0x5eed2, seed)
        for i in range(nr):
            ok, nt = judge(int(tok[h, i]), Q[i], prep)
            assert ok, f"k_s2_sample Philox ({h}, {i}): token {int(tok[h, i])} is not the float64 draw"
            near += int(nt)
    counts = np.bincount(tok.ravel(), minlength=V).astype(np.float64)
    pv, dof = chi2(counts, r["p"])
    assert pv > ALPHA
    pv_t, _ = chi2(counts, reference(keys_s2(row, 1.1), top_k=200)["p"])
    assert pv_t < ALPHA
    assert len({tuple(tok[h]) for h in range(nh)}) == nh, "hierarchies drew identical streams"
    print(f"k_s2_sample Philox, {nh * nr} draws: chi-square p = {pv:.3f} ({dof} dof), {near} near-ties; "
          f"T = 1.1: p = {pv_t:.1e}")


def test_stage2_forward_tokens_follow_its_logits(golden_dir):
    """mvb_s2_forward with d_logits_out and supplied noise: every token matches the float64 reference on the returned
    logits (top_k = 200, certified-margin rule)."""
    from mvb200 import synth
    from mvb200.second_stage import SecondStage
    dims = synth.S2_TINY
    g = np.load(f"{golden_dir}/stage2.npz")
    m = SecondStage(synth.stage2_checkpoint(dims, 1), device="cuda:0")
    idx = torch.from_numpy(g["tiny_idx"])
    spk = torch.from_numpy(g["tiny_spk"])
    gen = torch.Generator().manual_seed(4242)
    noise = torch.stack([torch.empty(dims.block_size, v).exponential_(1, generator=gen) for v in dims.target_vocab_sizes])
    toks, lg = m.forward_tokens(idx, spk, 1.0, 200, noise=noise, return_logits=True)
    toks, lg, nz = toks[0].cpu().numpy(), lg.cpu().numpy(), noise.numpy()
    draws = near = 0
    for h in range(lg.shape[0]):
        for t in range(lg.shape[1]):
            k = keys_s2(lg[h, t], 1.0)
            ok, nt, _ = token_ok(int(toks[h, t]), k, nz[h, t], "s2", top_k=200)
            assert ok, f"stage-2 forward draw ({h}, {t}): token {int(toks[h, t])} is not the float64 draw"
            draws, near = draws + 1, near + int(nt)
    assert draws > near
    m.close()
    print(f"mvb_s2_forward: {draws} tokens vs the float64 reference on its own logits, {near} certified near-ties")


# ---------------------------------------------------------------------------------------------------------------------
# sensitivity: altered references must violate the checks
def _api_violations(tok, probs, k, q, top_p, top_k, **alt):
    """Kept-set mismatches (outside the true band) + probability-bound violations + a wrong token, against an altered
    reference."""
    V = k.size
    r = reference(k, top_p=top_p, top_k=top_k, q=q)
    b = band(r, delta_cum(r, "k_sample", V))
    ra = reference(k, top_p=top_p, top_k=top_k, q=q, **alt)
    mism = (probs > 0) != ra["kept"]
    mism[b] = False
    a_i, a = a_terms(ra)
    bound = 1.01 * (a_i + a + 14 * U) * ra["p"] + 2.0 ** -125
    n = int(mism.sum()) + int((np.abs(probs - ra["p"]) > bound).sum())
    if "token" in ra:
        n += int(int(tok) != ra["token"])
    return n


def test_altered_references_violate(probes):
    p = probes(4096, 1)
    rng = np.random.default_rng(21)
    flat = api_logits(4096, "equal", rng)
    q = rng.exponential(size=4096).astype(np.float32)
    cases = [("'<' at the top-p threshold", flat, (3.0, 1.0, 0.5, None), dict(strict=True)),
             ("ties by descending index", flat, (3.0, 1.0, 0.5, None), dict(desc_ties=True)),
             ("top-k dropping ties at the pivot", flat, (3.0, 1.0, None, 200), dict(topk_drop_ties=True)),
             ("top-k dropping ties at the pivot (bf16 grid)", api_logits(4096, "bf16", rng), (1.0, 1.0, None, 200),
              dict(topk_drop_ties=True)),
             ("no keep-the-last rule", flat, (3.0, 1.0, 1e-9, None), dict(no_keep_last=True))]
    for name, lg, (g, T, tp, tk), alt in cases:
        toks, probs = run_api(p, lg, q, [(g, T, tp, tk)])
        k = keys_s1(lg[0], lg[1], g, T)
        check_api_draw(toks[0], probs[0], k, q, tp, tk, name)
        n = _api_violations(toks[0], probs[0], k, q, tp, tk, **alt)
        print(f"altered reference, {name}: {n} violations")
        assert n > 0, f"the altered reference ({name}) satisfies the checks"
    lg = api_logits(4096, "gauss5", rng)
    toks, probs = run_api(p, lg, q, [(3.0, 1.0, 0.95, None)])
    ks = keys_s1(lg[1], lg[0], 3.0, 1.0)                  # guidance applied to the swapped rows
    n = _api_violations(toks[0], probs[0], ks, q, 0.95, None)
    print(f"altered reference, guidance on swapped rows: {n} violations")
    assert n > 0
    # the decode samplers on the flat case: '<' and descending ties pick 2047 where the kernels drew 2048
    for fused in (True, False):
        pp = probes(4096, 8, fused)
        pp.set_speakers([0.0])
        slot = dict(g=3.0, T=1.0, top_p=0.5, fed=np.zeros(7, int), design=_flat_design)
        sampled, noises, _ = run_decode(pp, [slot], 6, seed=3)
        kf = np.full(4096, np.float32(1.0))
        for alt in (dict(strict=True), dict(desc_ties=True)):
            bad = sum(int(sampled[0, i]) != reference(kf, top_p=0.5, q=noises[0][i], **alt)["token"] for i in range(6))
            assert bad > 0, f"decode ({'fused' if fused else 'k_sample'}): altered reference {alt} reproduces every token"
