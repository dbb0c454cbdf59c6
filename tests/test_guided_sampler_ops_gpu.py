"""GPU: k_sample's prompt-guided path (guidance_scale = (s, p), causal.py:89-105) against a float64 restatement, in API
mode (mvb_s1_sample_guided) and in decode mode (a guided primary u and its companion slot c), with supplied Exp(1) noise
and with the Philox stream.

Reference.  The exact fp32 keys of the three-row mix, keys3 of tests/test_guided_sampler_cpu.py:
    k = fdiv_rn(fadd_rn(fadd_rn(fmul_rn(cb, l_c), fmul_rn(cs, l_u)), fmul_rn(cp, l_p)), max(T, 1e-5)),
    cb = fp32(s + p - 1), cs = fp32(1 - s), cp = fp32(1 - p) formed in double from the fp32 scales,
then the float64 tail of tests/test_sampler_ops_gpu.py (stable ascending order, top-k, top-p with keep-the-last, p, the
arg-max of p / q) with its bounds, unchanged, since the tail after the mix is the unguided kernel's:
  * kept set: exact outside the band |cum - fp32(1 - top_p)| <= delta_cum = 1.01 (2 a + 44 u) + V 2^-126, a the largest
    exponential's relative error 2^-22 + u |k_i - m|; exact everywhere when every key is equal (the tie-order cases);
  * probs_out: |p^ - p| <= 1.01 (a_i + a + 14 u) p + 2^-125 on the kernel's own kept set;
  * token: the float64 arg-max unless a certified near-tie, score ratio within (1 - rho) / (1 + rho),
    rho = 1.01 (2 a + 15 u + eps_q), eps_q = 2^-23 for Philox (logf) and 0 for supplied noise.
Each check prints its worst |err| / bound, the band entries it excused and the near-ties it accepted.

Decode mode runs the PROBE MODEL of tests/test_sampler_ops_gpu.py (one all-zero layer, one-hot token embeddings, lm_head
on the 1/256 grid, the speaker in column 255): each logit is one product or an exact sum of two, so mvb_s1_step_logits
returns the rows k_sample consumes bit for bit, and a token's rows depend only on its column (t mod 255) and its slot's
speaker.  mvb_s1_admit_guided gives the companion the primary's speaker; afterwards the companion gets another one, so
rows 2u, 2u + 1 and 2c are three distinct distributions.  With end_of_audio 2048 and end_of_text 2561 at V = 2562, a fed
text token (> 2048) reaches the companion as 2561, another lm_head column.  Text tokens are steered into the sequence
by supplied noise: the host predicts each draw from the float64 reference and, every third step, puts q = 1e-30 on the
most probable kept text token.  The admission's draw reads the prefill rows, taken from mvb_s1_forward on the same slots.

The decode state is read back after every burst with mvb_s1_poll, mvb_s1_fetch and mvb_s1_fetch_sampled, and field by
field from the engine's workspace (the layout of make_layout in csrc/stage1_engine.cu, checked against values set
through the API before use): the companion's sampled_tokens, gen_tokens (fed: text -> end_of_text, end_of_audio and
below passed through), row_tok, pos, n_gen and done equal the primary's; the link fields hold; and after every burst that samples in
k_sample every decoded slot's two logits rows are zero, which is what the persistent kernel's red.add accumulation
starts from at the next step.  Once the host has seen a primary done, the link is gone (both link fields 0, the
companion parked) and a burst without top-k is one fused launch again.

Philox: the stream is keyed by the primary's slot and n_gen[u].  Goodness of fit of non-stationary draws: each draw's
randomised probability integral transform under the float64 three-row probabilities (tokens ordered by decreasing
probability), Pearson chi-square on 20 equal bins, rejected below p = 1e-6.  The same statistic must reject the
two-row distribution; draws keyed by the companion's slot must fail the per-draw check (the probe's three-row
distributions are peaked, so many draws agree under either stream; any certified failure rejects it).

Sensitivity: a coefficient formed in fp32 (s + p - 1 rounded twice) and the mix evaluated as cb l_c + (cs l_u + cp l_p)
change the order of designed ties (every kernel key equal, exact kept set); the uncond-speaker and uncond-prompt rows
swapped put probabilities over their bound; the companion fed the raw text token mispredicts decode draws; p == 1
routed through three rows with a NaN third row predicts NaN where the kernel's two-row path is bit-identical to
mvb_s1_sample."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_guided_sampler_cpu import keys3, tie_rows
from test_sampler_ops_gpu import (ALPHA, BLOCK, N_COL, TEMP, TOP_P, U, V_API, Probe, _top_k, a_terms, api_logits, band,
                                  check_api_draw, chi2, delta_cum, judge, keys_s1, philox_q, prepare, reference)

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

F32 = np.float32
NEXT1 = float(np.nextafter(F32(1), F32(2)))         # the smallest p > 1: three rows with cp = -2^-23
GS_API = [(3.0, 2.0), (3.1, 1.7), (1.0, 3.0), (2.5, NEXT1)]
REGIMES = ["gauss1", "gauss5", "gauss40", "bf16", "needle", "equal", "plateau"]
V_DEC, EOA, EOT = 2562, 2048, 2561
TINY_Q = np.float32(1e-30)
KINDS = {"C": dict(tc=None), "B": dict(tc="B"), "A": dict(tc=""), "int8": dict(tc="", mode="int8"),
         "int4": dict(tc="", mode="int4")}
PER_STEP = {"C": 2, "B": 14}                        # launches per decode step: body + k_sample


def _lib():
    from mvb200 import _lib as L
    return L


# ---------------------------------------------------------------------------------------------------------------------
# API mode
def api_rows(V, regime, rng):
    """[3, V]: the two rows of the unguided sampler tests' regime and an uncond-prompt row of the same kind."""
    lc, lu = api_logits(V, regime, rng)
    if regime.startswith("gauss"):
        lp = lc + rng.standard_normal(V) * float(regime[5:]) / 4
    elif regime == "bf16":
        lp = rng.choice(np.arange(-8, 9) / 4.0, V)
    elif regime == "needle":
        lp = rng.standard_normal(V)
    elif regime == "equal":
        lp = np.full(V, 0.5)
    else:
        lp = lc.copy()
    return np.stack([lc, lu, lp]).astype(F32)


def run_api3(p, rows, q, combos, step=0):
    """mvb_s1_sample_guided for every (s, p, T, top_p, top_k) on rows [3, V]; q None: Philox at step + i."""
    L = _lib()
    V, n = p.V, len(combos)
    lg = torch.from_numpy(np.ascontiguousarray(rows)).cuda()
    qd = None if q is None else torch.from_numpy(q).cuda()
    tok = torch.empty(n, dtype=torch.int32, device="cuda")
    probs = torch.empty(n, V, device="cuda")
    n0 = p.launches()
    for i, (s, pg, T, tp, tk) in enumerate(combos):
        sp = L.Sampling(s, T, tp or 0.0, tk or 0, 9999, 7)
        L.check(p.lib.mvb_s1_sample_guided(p.h, lg.data_ptr(), C.byref(sp), pg, None if qd is None else qd.data_ptr(),
                                           step + i if qd is None else step, tok[i:].data_ptr(), probs[i].data_ptr(),
                                           p.st()))
    torch.cuda.synchronize()
    assert p.launches() - n0 == n
    return tok.cpu().numpy(), probs.cpu().numpy()


@pytest.fixture(scope="module")
def engines():
    cache = {}

    def get(V, utts, kind="C"):
        key = (V, utts, kind)
        if key not in cache:
            for k in list(cache):
                cache.pop(k).close()
            torch.cuda.empty_cache()
            cache[key] = Probe(V, utts, **KINDS[kind])
            if utts > 1:
                check_layout(cache[key])
        return cache[key]
    yield get
    for v in cache.values():
        v.close()


@pytest.mark.parametrize("V", V_API)
def test_api_guided_grid(engines, V):
    """Every (s, p) x temperature x top_p x top_k on seven regimes of three rows, supplied noise; then the gauss5 rows
    with the Philox stream (step = draw index)."""
    p = engines(V, 1)
    rng = np.random.default_rng(100 + V)
    combos = [(s, pg, T, tp, tk) for s, pg in GS_API for T in TEMP for tp in TOP_P for tk in _top_k(V)]
    worst, nb, near, draws = 0.0, 0, 0, 0
    for regime in REGIMES + ["philox"]:
        rows = api_rows(V, "gauss5" if regime == "philox" else regime, rng)
        philox = regime == "philox"
        q = None if philox else rng.exponential(size=V).astype(F32)
        toks, probs = run_api3(p, rows, q, combos)
        Q = philox_q(V, np.arange(len(combos))[:, None], 0, 0, 7) if philox else None
        for i, (s, pg, T, tp, tk) in enumerate(combos):
            k = keys3(rows[0], rows[1], rows[2], s, pg, T)
            w, b, nt = check_api_draw(toks[i], probs[i], k, Q[i] if philox else q, tp, tk,
                                      f"V={V} {regime} (s, p)=({s}, {pg}) T={T} top_p={tp} top_k={tk}", philox=philox)
            worst, nb, near, draws = max(worst, w), nb + b, near + int(nt), draws + 1
    assert draws > near
    print(f"k_sample guided API V={V}: {draws} draws (7 regimes + Philox x {len(combos)} parameter sets): max |err|/bound "
          f"{worst:.2e}, {nb} entries in the top-p band, {near} certified near-ties")


def test_api_guided_flat_tie_order_exact(engines):
    """V = 4096, each of the three rows constant: every key equal, so top_p = 0.5 keeps exactly 2048 ... 4095 at
    1/2048, top_p = 1e-9 keeps 4095 alone, top_k = 200 keeps every tie."""
    p = engines(4096, 1)
    rows = np.stack([np.full(4096, 0.75), np.full(4096, -0.25), np.full(4096, 0.5)]).astype(F32)
    q = np.random.default_rng(1).exponential(size=4096).astype(F32)
    for s, pg in [(3.0, 2.0), (3.1, 1.7), (1.0, 3.0)]:
        toks, probs = run_api3(p, rows, q, [(s, pg, 1.0, 0.5, None), (s, pg, 1.0, 1e-9, None), (s, pg, 1.0, None, 200)])
        want = np.zeros(4096, F32)
        want[2048:] = 1 / 2048
        assert np.array_equal(probs[0], want), (s, pg)
        assert int(toks[0]) == 2048 + int(np.argmin(q[2048:]))
        assert np.array_equal(np.nonzero(probs[1])[0], [4095]) and probs[1][4095] == 1.0 and toks[1] == 4095
        assert np.all(probs[2] == F32(1 / 4096)) and int(toks[2]) == int(np.argmin(q))


def _p_one_pairs(p, rows, q, combos, step=0):
    """(tokens, probs) of mvb_s1_sample_guided with p = 1 on rows [3, V] and of mvb_s1_sample on rows[:2]."""
    L = _lib()
    g = run_api3(p, rows, q, [(s, 1.0, T, tp, tk) for s, T, tp, tk in combos], step)
    lg = torch.from_numpy(np.ascontiguousarray(rows[:2])).cuda()
    qd = None if q is None else torch.from_numpy(q).cuda()
    tok = torch.empty(len(combos), dtype=torch.int32, device="cuda")
    probs = torch.empty(len(combos), p.V, device="cuda")
    for i, (s, T, tp, tk) in enumerate(combos):
        sp = L.Sampling(s, T, tp or 0.0, tk or 0, 9999, 7)
        L.check(p.lib.mvb_s1_sample(p.h, lg.data_ptr(), C.byref(sp), None if qd is None else qd.data_ptr(),
                                    step + i if qd is None else step, tok[i:].data_ptr(), probs[i].data_ptr(), p.st()))
    torch.cuda.synchronize()
    return g, (tok.cpu().numpy(), probs.cpu().numpy())


@pytest.mark.parametrize("V", [130, 4096])
def test_api_p_one_is_the_two_row_sampler(engines, V):
    """p == 1 is mvb_s1_sample bit for bit and never reads row 2 (NaN here), with supplied noise and with Philox."""
    p = engines(V, 1)
    rng = np.random.default_rng(7)
    combos = [(s, T, tp, tk) for s in (3.0, 1.0, 2.5) for T in TEMP for tp in (None, 0.95, 1e-3) for tk in (None, 40)]
    for noise in (True, False):
        rows = api_rows(V, "gauss5", rng)
        rows[2] = np.nan
        q = rng.exponential(size=V).astype(F32) if noise else None
        (tg, pg), (t2, p2) = _p_one_pairs(p, rows, q, combos)
        assert np.array_equal(tg, t2)
        assert np.array_equal(pg.view(np.int32), p2.view(np.int32))
        assert not np.isnan(pg).any()


# ---------------------------------------------------------------------------------------------------------------------
# decode-mode state, read from the engine's workspace
def _layout(p):
    """Byte offsets of the decode state in the stage-1 workspace (make_layout, csrc/stage1_engine.cu)."""
    Uu, V = p.utts, p.V
    R, D, F, H, max_new = 2 * Uu, 256, 256, 2, BLOCK
    sizes = [("x", R * D * 4), ("qkv", R * 3 * D * 4), ("att", R * D * 4), ("ffn", R * F * 4), ("logits", R * V * 4),
             ("spk", Uu * D * 4), ("part_o", R * H * 8 * 128 * 4), ("part_ml", R * H * 8 * 2 * 4), ("slot_map", Uu * 4),
             ("pos", Uu * 4), ("row_tok", R * 4), ("done", Uu * 4), ("n_gen", Uu * 4), ("gen_tokens", Uu * max_new * 4),
             ("sampled", Uu * max_new * 4), ("samp", Uu * 32)]
    off, out = 0, {}
    for name, n in sizes:
        out[name] = (off, n)
        off = (off + n + 255) // 256 * 256
    return out


def ws_state(p):
    """The decode state of every slot, from the workspace."""
    torch.cuda.synchronize()
    ws = p.m._ws[1]
    lay = _layout(p)
    end = lay["samp"][0] + lay["samp"][1]
    raw = ws[:end].cpu().numpy()
    get = lambda name, dt: raw[lay[name][0]:lay[name][0] + lay[name][1]].view(dt)  # noqa: E731
    samp = get("samp", np.int32).reshape(p.utts, 8)
    return dict(logits=get("logits", np.float32).reshape(2 * p.utts, p.V), pos=get("pos", np.int32).copy(),
                row_tok=get("row_tok", np.int32).copy(), done=get("done", np.int32).copy(),
                n_gen=get("n_gen", np.int32).copy(), gen=get("gen_tokens", np.int32).reshape(p.utts, BLOCK).copy(),
                sampled=get("sampled", np.int32).reshape(p.utts, BLOCK).copy(),
                guidance=samp[:, 0].view(np.float32).copy(), eoa=samp[:, 4].copy(), link=samp[:, 5].copy())


def check_layout(p):
    """The workspace reader against values installed through the C ABI: mvb_s1_begin's token, position and sampling
    entry, and the rows mvb_s1_forward leaves in the logits buffer."""
    L = _lib()
    n = p.utts
    for u in range(n):
        L.check(p.lib.mvb_s1_begin(p.h, u, 10 + u, 100 + u, C.byref(L.Sampling(1.5 + u, 1.0, 0.0, 0, 2000 + u, 1)),
                                   None, None, p.st()))
    st = ws_state(p)
    assert st["pos"].tolist() == [100 + u for u in range(n)], "workspace layout: pos"
    assert st["row_tok"].tolist() == [10 + u // 2 for u in range(2 * n)], "workspace layout: row_tok"
    assert st["done"].tolist() == [0] * n and st["n_gen"].tolist() == [0] * n, "workspace layout: done / n_gen"
    assert st["guidance"].tolist() == [1.5 + u for u in range(n)] and st["eoa"].tolist() == [2000 + u for u in range(n)]
    assert st["link"].tolist() == [0] * n, "workspace layout: SamplingDev"
    lg = prefill_rows(p, n - 1, np.array([7], np.int32))
    assert np.array_equal(ws_state(p)["logits"][2 * n - 2:], lg), "workspace layout: logits"


def prefill_rows(p, slot, prompt):
    """[2, V] logits of the last prompt position through mvb_s1_forward, as an admission's prefill leaves them."""
    L = _lib()
    idx = torch.from_numpy(np.concatenate([prompt, prompt]).astype(np.int32)).cuda()
    lg = torch.empty(2, p.V, device="cuda")
    L.check(p.lib.mvb_s1_forward(p.h, slot, idx.data_ptr(), len(prompt), 0, lg.data_ptr(), 0, p.st()))
    torch.cuda.synchronize()
    return lg.cpu().numpy()


def set_spk(p, u, val):
    e = torch.zeros(256)
    e[0] = float(val)
    p.m.set_speaker(u, e)


class Table:
    """Step logits [2 n, V] by lm_head column, every slot fed the same token (mvb_s1_begin: call it only while no link
    is live)."""

    def __init__(self, p, n):
        self.p, self.n, self.cols = p, n, {}

    def __call__(self, t):
        c = int(t) % N_COL
        if c not in self.cols:
            self.cols[c] = self.p.logits([c] * self.n)
        return self.cols[c]


# ---------------------------------------------------------------------------------------------------------------------
# decode mode
GUIDED = [dict(s=3.0, pg=2.0, T=1.0, top_p=0.95, top_k=None, spk=0.5, cspk=-0.75),
          dict(s=3.1, pg=1.7, T=0.7, top_p=None, top_k=40, spk=0.75, cspk=1.0),
          dict(s=1.0, pg=3.0, T=1.0, top_p=0.5, top_k=None, spk=-0.5, cspk=0.25),
          dict(s=2.5, pg=NEXT1, T=1e-6, top_p=0.9, top_k=None, spk=1.0, cspk=-1.0)]
UNGUIDED = [dict(s=3.0, pg=None, T=1.0, top_p=0.9, top_k=None, spk=0.25), dict(s=1.5, pg=None, T=0.8, top_p=None, top_k=40, spk=-0.25)]
ARRANGE = {"above": ([(0, 1)], []), "below": ([(1, 0)], []), "apart": ([(0, 3)], [1, 2]),
           "two_pairs": ([(0, 4), (5, 2)], [1, 3])}


def fc_of(t):
    return EOT if t > EOA else t


def slot_keys(sl, rows, lp):
    if sl["pg"] is None:
        return keys_s1(rows[0], rows[1], sl["s"], sl["T"])
    return keys3(rows[0], rows[1], lp, sl["s"], sl["pg"], sl["T"])


class Run:
    """One decode scenario: guided pairs and unguided slots admitted into slots [0, n), bursts of mvb_s1_decode, the
    state after every burst, and the float64 check of every draw."""

    def __init__(self, p, pairs, unguided, seed, prompt_len=1, max_new=64, noise=True, force_text=True, eoa_at=None):
        self.p, self.pairs = p, pairs
        self.n = 1 + max([x for pr in pairs for x in pr] + list(unguided))
        self.rng = np.random.default_rng(seed)
        self.slots = {}
        for i, (u, c) in enumerate(pairs):
            self.slots[u] = dict(GUIDED[(i + seed) % len(GUIDED)], comp=c)
        for i, u in enumerate(unguided):
            self.slots[u] = dict(UNGUIDED[i % len(UNGUIDED)], comp=None)
        self.companions = {c: u for u, c in pairs}
        self.noise, self.force_text, self.eoa_at = noise, force_text, eoa_at
        self.T, self.max_new = prompt_len, max_new
        self.room = min(prompt_len + max_new, BLOCK) - prompt_len
        L = _lib()
        for u in range(p.utts):
            L.check(p.lib.mvb_s1_release(p.h, u, p.st()))
        # prompts; prefill rows with the admission's speakers (a companion has its primary's), then the decode speakers
        for u, sl in self.slots.items():
            sl["prompt"] = self.rng.integers(2, EOA, prompt_len).astype(np.int32)
            if prompt_len == 1:
                sl["prompt"][0] = self.rng.integers(EOA + 1, V_DEC)     # a text token: the companion's is end_of_text
        for u, sl in self.slots.items():
            set_spk(p, u, sl["spk"])
            if sl["comp"] is not None:
                set_spk(p, sl["comp"], sl["spk"])
        for u, sl in self.slots.items():
            sl["pre"] = prefill_rows(p, u, sl["prompt"])
            if sl["comp"] is not None:
                sl["pre_c"] = prefill_rows(p, sl["comp"], np.array([fc_of(t) for t in sl["prompt"]], np.int32))
        for u in range(self.n):
            if u not in self.slots and u not in self.companions:
                set_spk(p, u, 0.0)
        for u, sl in self.slots.items():
            if sl["comp"] is not None:
                set_spk(p, sl["comp"], sl["cspk"])
        self.table = Table(p, self.n)

    def rows(self, u, i, fed):
        """(rows 2u, 2u + 1, row 2c) slot u's draw i reads, given the tokens fed before it."""
        sl = self.slots[u]
        if i == 0:
            return sl["pre"], (sl["pre_c"][0] if sl["comp"] is not None else None)
        t = int(fed[i - 1])
        lp = self.table(fc_of(t))[2 * sl["comp"]] if sl["comp"] is not None else None
        return self.table(t)[2 * u:2 * u + 2], lp

    def design(self, n_draws):
        """Supplied noise per slot (q = 1e-30 on a kept text token every third draw, on end_of_audio at eoa_at) and the
        predicted tokens."""
        for u, sl in self.slots.items():
            q = self.rng.exponential(size=(self.room, V_DEC)).astype(F32)
            fed = []
            for i in range(min(n_draws, self.room)):
                rows, lp = self.rows(u, i, fed)
                r = reference(slot_keys(sl, rows, lp), top_p=sl["top_p"], top_k=sl["top_k"])
                want = None
                if self.eoa_at is not None and i >= self.eoa_at and sl["comp"] is not None:
                    want = EOA if r["p"][EOA] > 1e-20 else None
                elif self.force_text and i % 3 == 1 and sl["comp"] is not None:
                    text = np.arange(EOA + 1, V_DEC)
                    text = text[r["kept"][text] & (r["p"][text] > 1e-20)]
                    want = int(text[np.argmax(r["p"][text])]) if text.size else None
                if want is not None and r["p"][want] > 1e-20:
                    q[i, want] = TINY_Q
                fed.append(int(np.argmax(r["p"] / q[i])))
                if fed[-1] == EOA:
                    sl["eoa_step"] = i
                    break
            sl["q"] = q
            sl["predicted"] = fed

    def admit(self):
        L = _lib()
        self.keep = []
        for u, sl in self.slots.items():
            sp = L.Sampling(sl["s"], sl["T"], sl["top_p"] or 0.0, sl["top_k"] or 0, EOA, 11 + u)
            qd = torch.from_numpy(sl["q"]).cuda() if self.noise else None
            self.keep.append(qd)
            spk = np.zeros(256, F32)
            spk[0] = sl["spk"]
            pr = sl["prompt"]
            vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
            if sl["comp"] is None:
                L.check(self.p.lib.mvb_s1_admit(self.p.h, u, vp(pr), pr.size, vp(spk), C.byref(sp), self.max_new,
                                                None if qd is None else qd.data_ptr(), self.p.st()))
            else:
                L.check(self.p.lib.mvb_s1_admit_guided(self.p.h, u, sl["comp"], vp(pr), pr.size, vp(spk), C.byref(sp),
                                                       sl["pg"], EOT, self.max_new, None if qd is None else qd.data_ptr(),
                                                       self.p.st()))
                set_spk(self.p, sl["comp"], sl["cspk"])
        self.states = [self.snapshot()]

    def burst(self, n_steps, kind):
        """One mvb_s1_decode burst.  While a link is live (its primary not yet seen done by a poll) the resident kernel
        leaves sampling to k_sample; once every link is gone and no slot has top_k, the burst is one fused launch."""
        p = self.p
        prev = self.states[-1]["poll"][0]
        live = any(not prev[u] for u, sl in self.slots.items() if sl["comp"] is not None)
        n0 = p.launches()
        _lib().check(p.lib.mvb_s1_decode(p.h, self.n, n_steps, p.st()))
        torch.cuda.synchronize()
        per = (p.launches() - n0 - 1) / n_steps
        fused = kind == "C" and not live and not any(sl["top_k"] for sl in self.slots.values())
        if fused:
            assert p.launches() - n0 == 2, f"{kind}: {p.launches() - n0} launches, not the fused burst"
        elif kind in PER_STEP:
            assert per == PER_STEP[kind], f"{kind}: {per} launches per step"
        else:
            assert per == int(per) and per >= 2, f"{kind}: {per} launches per step"
        self.states.append(dict(self.snapshot(), fused=fused))

    def snapshot(self):
        """Workspace state first (poll and fetch dissolve the link of a finished primary), then the C ABI's view."""
        L = _lib()
        st = ws_state(self.p)
        done, n_gen = np.zeros(self.n, np.int32), np.zeros(self.n, np.int32)
        L.check(self.p.lib.mvb_s1_poll(self.p.h, self.n, done.ctypes.data_as(C.c_void_p), n_gen.ctypes.data_as(C.c_void_p),
                                       self.p.st()))
        st["poll"] = (done, n_gen)
        st["fetch"], st["fetch_sampled"] = {}, {}
        for u in range(self.n):
            buf = np.zeros(BLOCK, np.int32)
            n_out, d = C.c_int32(), C.c_int32()
            L.check(self.p.lib.mvb_s1_fetch(self.p.h, u, buf.ctypes.data_as(C.c_void_p), BLOCK, C.byref(n_out),
                                            C.byref(d), self.p.st()))
            st["fetch"][u] = buf[:n_out.value].copy()
            sb = (C.c_int32 * BLOCK)()
            L.check(self.p.lib.mvb_s1_fetch_sampled(self.p.h, u, sb, BLOCK, self.p.st()))
            st["fetch_sampled"][u] = np.frombuffer(sb, np.int32)[:n_out.value].copy()
        return st

    def check_states(self):
        """Field by field after every burst.  Returns {primary: companion tokens fed as end_of_text}."""
        n_text = {}
        for b, st in enumerate(self.states):
            lab = f"after burst {b}"
            assert st.get("fused") or not st["logits"][:2 * self.n].any(), f"{lab}: logits rows left non-zero at " \
                f"{sorted(set(np.nonzero(st['logits'][:2 * self.n])[0].tolist()))}"
            done, n_gen = st["poll"]
            assert np.array_equal(done, st["done"][:self.n]) and np.array_equal(n_gen, st["n_gen"][:self.n])
            for u, sl in self.slots.items():
                n = int(st["n_gen"][u])
                assert np.array_equal(st["fetch"][u], st["gen"][u, :n]) and np.array_equal(st["fetch_sampled"][u],
                                                                                          st["sampled"][u, :n])
                fed = st["gen"][u, :n]
                assert np.array_equal(fed, st["sampled"][u, :n]), f"{lab}: slot {u} fed differs from sampled (no forcing)"
                last = int(fed[-1]) if n else int(sl["prompt"][-1])
                assert st["row_tok"][2 * u] == st["row_tok"][2 * u + 1] == last, f"{lab}: row_tok of slot {u}"
                assert st["pos"][u] == self.T - 1 + n - int(st["done"][u]), f"{lab}: pos of slot {u}"
                if sl["comp"] is None:
                    assert st["link"][u] == 0
                    continue
                c = sl["comp"]
                tag = f"{lab}: companion {c} of slot {u}"
                assert st["n_gen"][c] == n and st["done"][c] == st["done"][u] and st["pos"][c] == st["pos"][u], tag
                assert np.array_equal(st["sampled"][c, :n], st["sampled"][u, :n]), f"{tag}: sampled_tokens"
                assert st["gen"][c, :n].tolist() == [fc_of(int(t)) for t in fed], f"{tag}: fed tokens"
                assert st["row_tok"][2 * c] == st["row_tok"][2 * c + 1] == fc_of(last), f"{tag}: row_tok"
                if b and self.states[b - 1]["done"][u]:      # seen done by the poll: link dissolved, companion parked
                    assert st["link"][u] == st["link"][c] == 0 and st["done"][c] == 1, f"{tag}: dissolved link"
                else:
                    assert (st["link"][u], st["link"][c]) == (c + 1, -(u + 1)), f"{tag}: link"
                    assert st["guidance"][c] == F32(sl["pg"]) and st["eoa"][c] == EOT, f"{tag}: p / end_of_text"
                n_text[u] = int((st["gen"][c, :n] == EOT).sum())
        return n_text

    def check_draws(self, raw_text=False):
        """Every draw of every slot against the float64 reference.  raw_text: the altered reference that feeds the
        companion the raw text token; returns the draws it gets wrong instead of asserting."""
        st = self.states[-1]
        draws = near = nb = wrong = 0
        for u, sl in self.slots.items():
            n = int(st["n_gen"][u])
            fed = st["gen"][u, :n]
            Q = sl["q"] if self.noise else philox_q(V_DEC, np.arange(n)[:, None], 0, u, 11 + u)
            for i in range(n):
                rows, lp = self.rows(u, i, fed)
                if raw_text and sl["comp"] is not None and i > 0:
                    lp = self.table(int(fed[i - 1]))[2 * sl["comp"]]
                k = slot_keys(sl, rows, lp)
                variants, b = prepare(k, "k_sample", not self.noise, top_p=sl["top_p"], top_k=sl["top_k"])
                ok, nt = judge(int(st["sampled"][u, i]), Q[i], variants)
                if raw_text:
                    wrong += int(not ok)
                    continue
                assert ok, f"slot {u} draw {i}: token {int(st['sampled'][u, i])} is not the float64 draw"
                draws, near, nb = draws + 1, near + int(nt), nb + b
        if raw_text:
            return wrong
        assert draws > near
        return draws, near, nb


DECODE_CASES = [("C", "above"), ("C", "below"), ("C", "apart"), ("C", "two_pairs"), ("B", "apart"), ("B", "two_pairs"),
                ("A", "below"), ("int8", "apart"), ("int4", "two_pairs")]


@pytest.mark.parametrize("case", range(len(DECODE_CASES)), ids=[f"{k}-{a}" for k, a in DECODE_CASES])
def test_decode_guided_bursts(engines, case):
    """Bursts of 5, 7 and 6 steps after the admission; supplied noise steering text tokens into the sequence."""
    kind, arr = DECODE_CASES[case]
    p = engines(V_DEC, 8, kind)
    pairs, ung = ARRANGE[arr]
    run = Run(p, pairs, ung, seed=case)
    bursts = [5, 7, 6]
    run.design(1 + sum(bursts))
    run.admit()
    for b in bursts:
        run.burst(b, kind)
    n_text = run.check_states()
    draws, near, nb = run.check_draws()
    for u, sl in run.slots.items():
        if sl["comp"] is not None and sl["T"] >= 0.5:
            assert n_text[u] >= 2, f"only {n_text[u]} text tokens reached companion {sl['comp']}"
    print(f"guided decode [{kind}, {arr}]: {draws} draws, {near} certified near-ties, {nb} band entries, "
          f"{n_text} text tokens fed to companions as end_of_text")


@pytest.mark.parametrize("kind", ["C", "A"])
def test_decode_guided_latches(engines, kind):
    """The end-of-audio latch (drawn at step 4), the token budget (max_new_tokens 9) and the context end (a 2041-token
    prompt: 7 tokens fit) each reach the companion with the primary; then, with the link dissolved by the poll, further
    bursts leave the finished pair's rows zero and its state alone while the unguided slot keeps drawing."""
    p = engines(V_DEC, 8, kind)
    for name, kw, want_n in [("eoa", dict(eoa_at=4), None), ("budget", dict(max_new=9), 9),
                             ("context", dict(prompt_len=2041, max_new=64), 7)]:
        run = Run(p, [(2, 0)], [1], seed=3, force_text=name != "eoa", **kw)
        run.slots[2].update(s=3.0, pg=2.0, T=1.0, top_p=None, top_k=None)
        run.design(40)
        if name == "eoa":
            want_n = run.slots[2]["eoa_step"] + 1
        run.admit()
        for b in (6, 6):
            run.burst(b, kind)
        run.check_states()
        st = run.states[-1]
        assert st["n_gen"][2] == st["n_gen"][0] == want_n and st["done"][2] == st["done"][0] == 1, name
        if name == "eoa":
            assert st["gen"][2, want_n - 1] == st["gen"][0, want_n - 1] == EOA
        if name == "context":
            assert st["pos"][2] == st["pos"][0] == BLOCK - 2
        # the host has seen the primary done: the link is gone, the companion parked; the burst goes on
        run.burst(3, kind)
        after = run.states[-1]
        assert after["link"][0] == after["link"][2] == 0 and after["done"][0] == 1
        assert after["fused"] or not after["logits"][:2 * run.n].any()
        for f in ("n_gen", "pos", "row_tok"):
            assert np.array_equal(after[f][[0, 2]] if f != "row_tok" else after[f][[0, 1, 4, 5]],
                                  st[f][[0, 2]] if f != "row_tok" else st[f][[0, 1, 4, 5]]), f"{name}: {f} moved"
        assert after["n_gen"][1] > st["n_gen"][1] or st["done"][1]
        draws, near, nb = run.check_draws()
        print(f"guided latch [{kind}] {name}: both slots done at n_gen = {want_n}; {draws} draws, {near} near-ties, "
              f"{nb} band entries")


def test_philox_guided_goodness_of_fit(engines):
    """One guided pair (primary 0, companion 1), noise = NULL, 1500 draws: every draw against the float64 reference on
    the host Philox stream keyed (n_gen, primary slot); the randomised PIT chi-square passes for the three-row
    probabilities and rejects the two-row ones; the stream keyed by the companion's slot fails per-draw checks."""
    p = engines(V_DEC, 8, "C")
    N = 1500
    run = Run(p, [(0, 1)], [], seed=0, max_new=N, noise=False, force_text=False)
    sl = run.slots[0]
    run.slots[0] = sl = dict(sl, s=3.0, pg=2.0, T=1.0, top_p=None, top_k=None)
    run.design(0)
    run.admit()
    run.burst(N - 1, "C")
    run.check_states()
    st = run.states[-1]
    n = int(st["n_gen"][0])
    assert n == N or st["gen"][0, n - 1] == EOA
    fed = st["gen"][0, :n]
    Qu = philox_q(V_DEC, np.arange(n)[:, None], 0, 0, 11)
    Qc = philox_q(V_DEC, np.arange(n)[:, None], 0, 1, 11)
    prng = np.random.default_rng(1)
    pit3, pit2, near, wrong_c = [], [], 0, 0
    for i in range(n):
        rows, lp = run.rows(0, i, fed)
        k = slot_keys(sl, rows, lp)
        variants, _ = prepare(k, "k_sample", True)
        tok = int(st["sampled"][0, i])
        ok, nt = judge(tok, Qu[i], variants)
        assert ok, f"Philox draw {i}: token {tok} is not the float64 draw"
        near += int(nt)
        wrong_c += int(not judge(tok, Qc[i], variants)[0])
        v = prng.uniform()
        for P, acc in ((variants[0][0], pit3), (reference(keys_s1(rows[0], rows[1], 3.0, 1.0))["p"], pit2)):
            order = np.argsort(-P, kind="stable")
            cum = np.cumsum(P[order])
            j = int(np.nonzero(order == tok)[0][0])
            acc.append(cum[j] - P[tok] * (1 - v))
    bins = 20
    exp_ = np.full(bins, 1.0 / bins)
    pv3, _ = chi2(np.bincount(np.minimum((np.array(pit3) * bins).astype(int), bins - 1), minlength=bins).astype(float), exp_)
    pv2, _ = chi2(np.bincount(np.minimum((np.array(pit2) * bins).astype(int), bins - 1), minlength=bins).astype(float), exp_)
    print(f"guided Philox, {n} draws: PIT chi-square p = {pv3:.3f} (three rows), {pv2:.1e} (two rows); {near} near-ties; "
          f"companion-keyed stream wrong on {wrong_c} of {n} draws")
    assert pv3 > ALPHA, f"guided Philox tokens do not fit the three-row probabilities (p = {pv3:.2e})"
    assert pv2 < ALPHA, f"the chi-square does not reject the two-row distribution (p = {pv2:.2e})"
    assert wrong_c > 0, "draws keyed by the companion's slot pass every per-draw check"


# ---------------------------------------------------------------------------------------------------------------------
# sensitivity
def _violations(tok, probs, k, q, top_p, top_k):
    """Kept-set mismatches outside the band, probabilities not within their bound (NaN counts) and a wrong token,
    against the reference started from keys k."""
    with np.errstate(invalid="ignore"):
        r = reference(k, top_p=top_p, top_k=top_k, q=q)
        b = band(r, delta_cum(r, "k_sample", k.size)) if np.isfinite(k).all() else np.zeros(0, int)
        mism = (probs > 0) != r["kept"]
        mism[b] = False
        a_i, a = a_terms(r) if np.isfinite(k).all() else (np.zeros(k.size), 0.0)
        bound = 1.01 * (a_i + a + 14 * U) * r["p"] + 2.0 ** -125
        return int(mism.sum()) + int((~(np.abs(probs - r["p"]) <= bound)).sum()) + int(int(tok) != r.get("token", -1))


def test_altered_references_violate(engines):
    p = engines(4096, 1)
    rng = np.random.default_rng(31)
    q = rng.exponential(size=4096).astype(F32)
    out = {}
    for name, (s, pg), variant in [("coefficient s + p - 1 formed in fp32", (3.1, 1.7), "fp32_sum"),
                                   ("mix as cb l_c + (cs l_u + cp l_p)", (3.0, 2.0), "right_assoc")]:
        rows = tie_rows(s, pg, variant)
        toks, probs = run_api3(p, rows, q, [(s, pg, 1.0, 0.5, None)])
        want = np.zeros(4096, F32)
        want[2048:] = 1 / 2048
        assert np.array_equal(probs[0], want), f"{name}: the designed ties are not exact in the kernel"
        out[name] = _violations(toks[0], probs[0], keys3(*rows, s, pg, 1.0, **{variant: True}), q, 0.5, None)
    rows = api_rows(4096, "gauss1", rng)                  # no top-p: every probability is compared
    toks, probs = run_api3(p, rows, q, [(3.0, 2.0, 1.0, None, None)])
    check_api_draw(toks[0], probs[0], keys3(rows[0], rows[1], rows[2], 3.0, 2.0, 1.0), q, None, None, "unaltered")
    out["uncond-speaker and uncond-prompt rows swapped"] = _violations(
        toks[0], probs[0], keys3(rows[0], rows[2], rows[1], 3.0, 2.0, 1.0), q, None, None)
    rows[2] = np.nan
    toks, probs = run_api3(p, rows, q, [(3.0, 1.0, 1.0, 0.95, None)])
    check_api_draw(toks[0], probs[0], keys_s1(rows[0], rows[1], 3.0, 1.0), q, 0.95, None, "p == 1")
    out["p == 1 through three rows, NaN third row"] = _violations(
        toks[0], probs[0], keys3(rows[0], rows[1], rows[2], 3.0, 1.0, 1.0), q, 0.95, None)
    pd = engines(V_DEC, 8, "C")
    run = Run(pd, [(0, 3)], [1, 2], seed=5)
    run.design(19)
    run.admit()
    for b in (9, 9):
        run.burst(b, "C")
    run.check_draws()
    out["companion fed the raw text token"] = run.check_draws(raw_text=True)
    for name, n in out.items():
        print(f"altered reference, {name}: {n} violations -> {'caught' if n else 'NOT caught'}")
    assert all(n > 0 for n in out.values()), out
