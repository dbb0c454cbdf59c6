"""GPU: the stage-2 front end (k_s2_spk, then k_s2_embed) through the hook mvb_s2_embed_test, against float64 on the same
bf16 tables.

    spk_proj[b] = W_spk . spk[b]                                           [B, E]
    x[b*t + i]  = sum_h wte_h[idx[b, h, i]] + wpe[i] + spk_proj[b]         [B*t, E]   (no speaker term when spk is NULL)

Bounds, from the order the kernels declare (u = 2^-24, gamma_n = n u / (1 - n u)):
  * k_s2_spk: lane l runs an fmaf chain over k = l (mod 32), ceil(SD/32) roundings, then a 5-level butterfly adds five:
        |s^ - s| <= gamma_{ceil(SD/32)+5} * sum_k |W_ek spk_k|
  * k_s2_embed: one sequential fp32 sum of the n_in table entries, the wpe entry and s^ (bf16 -> fp32 is exact):
        |x^ - x| <= gamma_{n_in+2} * (sum_h |wte_h| + |wpe| + |s| + |s^ - s|_bound) + |s^ - s|_bound
Tables, wpe and the speaker are N(0, 1) and W_spk is N(0, 1/SD), so the speaker term is as large as a table entry.  Every
hierarchy has its own table (distinct sizes), every utterance its own speaker, and the indices include 0, vocab - 1 and the
pad 1024 of each hierarchy.  Outputs are NaN-filled with guard rows before and after: only [0, B*t) x [0, E) of x and
[0, B) x [0, E) of spk_proj may change, and all of it must (spk_proj not at all without a speaker).

Sensitivity: references with the speakers rotated by one utterance, wpe row i + 1 instead of i, hierarchy n_in - 1 dropped
and idx read as [n_in, B, t] instead of [B, n_in, t] must violate the bound."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
PAD = 1024
GUARD_ROWS = 2

# (B, t, E, spk_dim, n_in): every B in {1, 3, 64}, t in {1, 77, 1024}, E in {64, 320, 384, 2048} (320: the 128-thread
# stride loop ends on a partial pass), spk_dim in {1, 33, 256} and n_in in {1, 2, 8}
CASES = [
    (1, 1, 64, 1, 1),
    (1, 1024, 2048, 256, 8),
    (3, 77, 320, 33, 2),
    (3, 1024, 384, 256, 2),      # the production stage-2 shape, three utterances
    (3, 1, 2048, 33, 8),
    (64, 77, 320, 1, 8),
    (64, 1024, 384, 256, 2),     # the production shape at the engine's largest batch: 65,536 rows
    (64, 1, 64, 33, 1),
]


def gamma(n):
    return n * U / (1 - n * U)


class Inputs:
    """bf16 tables, wpe and W_spk, fp32 speakers and int32 indices on the device, and their float64 copies."""

    def __init__(self, B, t, E, SD, n_in, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        rnd = lambda *s: torch.randn(*s, generator=g, device="cuda")  # noqa: E731
        self.B, self.t, self.E, self.SD, self.n_in = B, t, E, SD, n_in
        self.vocab = [1025 + 3 * h for h in range(n_in)]
        self.wte = [rnd(v, E).to(torch.bfloat16) for v in self.vocab]
        self.wpe = rnd(t, E).to(torch.bfloat16)
        self.W = (rnd(E, SD) / math.sqrt(SD)).to(torch.bfloat16)
        self.spk = rnd(B, SD)
        idx = torch.stack([torch.randint(0, v, (B, t), generator=g, device="cuda") for v in self.vocab], 1)   # [B, n_in, t]
        for h, v in enumerate(self.vocab):
            flat = idx[:, h].reshape(-1).clone()
            special = [0, v - 1, PAD]
            for k in range(min(3, flat.numel())):
                flat[k] = special[(k + h) % 3]
                flat[-1 - k] = special[(k + h + 1) % 3]
            idx[:, h] = flat.view(B, t)
        self.idx = idx.to(torch.int32).contiguous()
        self.wte_ptrs = torch.tensor([w.data_ptr() for w in self.wte], dtype=torch.int64, device="cuda")
        self.wte_d = [w.double() for w in self.wte]
        self.wpe_d, self.W_d, self.spk_d = self.wpe.double(), self.W.double(), self.spk.double()

    def run(self, with_speaker=True):
        """One hook call on NaN-filled, guarded outputs; returns (x^ [B, t, E], s^ [B, E] or None), float64."""
        from mvb200 import _lib as L
        B, t, E = self.B, self.t, self.E
        gx = GUARD_ROWS * E
        xb = torch.full((B * t * E + 2 * gx,), float("nan"), device="cuda")
        sb = torch.full((B * E + 2 * gx,), float("nan"), device="cuda")
        L.check(L.load().mvb_s2_embed_test(self.idx.data_ptr(), B, self.n_in, t, self.wte_ptrs.data_ptr(), self.wpe.data_ptr(),
                                           self.W.data_ptr(), self.spk.data_ptr() if with_speaker else None, self.SD, E,
                                           sb[gx:].data_ptr(), xb[gx:].data_ptr(),
                                           C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        x, s = xb[gx:gx + B * t * E], sb[gx:gx + B * E]
        assert torch.isnan(xb[:gx]).all() and torch.isnan(xb[gx + B * t * E:]).all(), "k_s2_embed wrote outside [0, B*t) x [0, E)"
        assert not torch.isnan(x).any(), "k_s2_embed left elements of x unwritten"
        assert torch.isnan(sb[:gx]).all() and torch.isnan(sb[gx + B * E:]).all(), "k_s2_spk wrote outside [0, B) x [0, E)"
        if not with_speaker:
            assert torch.isnan(s).all(), "spk_proj written without a speaker"
            return x.double().view(B, t, E), None
        assert not torch.isnan(s).any(), "k_s2_spk left elements of spk_proj unwritten"
        return x.double().view(B, t, E), s.double().view(B, E)

    def speaker(self):
        """float64 s [B, E] and its bound."""
        s = self.spk_d @ self.W_d.t()
        bound = gamma(-(-self.SD // 32) + 5) * (self.spk_d.abs() @ self.W_d.abs().t())
        return s, bound

    def reference(self, with_speaker=True, spk_roll=0, wpe_shift=0, drop_last=False, idx_layout="b h t"):
        """float64 x [B, t, E] and its bound; the keyword arguments alter the reference for the sensitivity checks."""
        B, t, n_in = self.B, self.t, self.n_in
        idx = self.idx.long()
        if idx_layout == "h b t":      # the same buffer read as [n_in, B, t]; indices wrapped into the table they now address
            idx = idx.reshape(n_in, B, t).transpose(0, 1)
            idx = torch.stack([idx[:, h] % v for h, v in enumerate(self.vocab)], 1)
        hs = range(n_in - 1) if drop_last else range(n_in)
        x = sum((self.wte_d[h][idx[:, h]] for h in hs), torch.zeros(B, t, self.E, dtype=torch.float64, device="cuda"))
        ab = sum(self.wte_d[h][self.idx[:, h].long()].abs() for h in range(n_in))
        wpe = self.wpe_d.roll(-wpe_shift, 0)
        x = x + wpe[None]
        ab = ab + self.wpe_d.abs()[None]
        bound = 0.0
        if with_speaker:
            s, sb = self.speaker()
            x = x + s.roll(spk_roll, 0)[:, None]
            ab = ab + (s.abs() + sb)[:, None]
            bound = sb[:, None]
        return x, gamma(n_in + 2) * ab + bound + 1e-300


def _check(got, ref, bound, label):
    err = (got - ref).abs()
    bad = (err > bound).nonzero()
    ratio = float((err / bound).max())
    assert bad.numel() == 0, f"{label}: {bad.shape[0]} elements over the bound (max ratio {ratio:.2e}), first {bad[0].tolist()}"
    dims = tuple(range(1, err.dim()))
    nw = (err.pow(2).sum(dims).sqrt() / ref.pow(2).sum(dims).sqrt()).max()     # worst utterance
    return ratio, float(nw)


@pytest.mark.parametrize("with_speaker", [True, False], ids=["speaker", "no-speaker"])
@pytest.mark.parametrize("B,t,E,SD,n_in", CASES)
def test_s2_front_end_vs_float64(B, t, E, SD, n_in, with_speaker):
    inp = Inputs(B, t, E, SD, n_in, seed=B * 7919 + t * 31 + E + SD * 3 + n_in)
    x, s = inp.run(with_speaker)
    label = f"B={B} t={t} E={E} spk_dim={SD} n_in={n_in}"
    msg = ""
    if with_speaker:
        s_ref, s_bound = inp.speaker()
        rs, ns = _check(s, s_ref, s_bound + 1e-300, f"k_s2_spk {label}")
        msg = f"spk_proj max |err|/bound {rs:.2e}, normwise {ns:.2e}; "
    x_ref, x_bound = inp.reference(with_speaker)
    rx, nx = _check(x, x_ref, x_bound, f"k_s2_embed {label}")
    if not with_speaker:            # the speaker term, had it been added, would be visible
        with_spk, _ = inp.reference(True)
        n_over = int(((x - with_spk).abs() > x_bound).sum())
        assert n_over > 0, "a reference with the speaker term also satisfies the no-speaker bound"
        msg = f"reference with a speaker term: {n_over} elements over; "
    print(f"s2 front end {label} ({'speaker' if with_speaker else 'no speaker'}): {msg}x max |err|/bound {rx:.2e}, "
          f"worst per-utterance normwise {nx:.2e}")


@pytest.mark.parametrize("B,t,E,SD,n_in", [(3, 77, 320, 33, 2), (64, 77, 320, 1, 8), (3, 1024, 384, 256, 2)])
def test_s2_front_end_altered_references_violate_the_bound(B, t, E, SD, n_in):
    inp = Inputs(B, t, E, SD, n_in, seed=17 + B + n_in)
    x, s = inp.run(True)
    _, bound = inp.reference(True)
    s_ref, s_bound = inp.speaker()
    counts = {}
    spk_over = int(((s - s_ref.roll(1, 0)).abs() > s_bound).sum())
    for name, kw in (("speakers rotated by one utterance", dict(spk_roll=1)), ("wpe row i + 1", dict(wpe_shift=1)),
                     (f"hierarchy {n_in - 1} dropped", dict(drop_last=True)), ("idx read as [n_in, B, t]", dict(idx_layout="h b t"))):
        alt, _ = inp.reference(True, **kw)
        counts[name] = int(((x - alt).abs() > bound).sum())
    print(f"s2 front end B={B} t={t} E={E} spk_dim={SD} n_in={n_in}: elements of x over the bound per altered reference "
          f"{counts} (of {x.numel()}); spk_proj vs rotated speakers: {spk_over} of {s.numel()} over")
    assert spk_over > 0
    for name, n in counts.items():
        assert n > 0, f"a reference with {name} satisfies the bound"


def test_s2_embed_hook_rejects_bad_arguments():
    """MVB_ERR_ARG (nothing launched, outputs untouched) for null pointers, B, t, E or spk_dim < 1 and n_in outside 1..8."""
    from mvb200 import _lib as L
    lib = L.load()
    inp = Inputs(2, 5, 64, 33, 2, seed=5)
    x = torch.full((2 * 5 * 64,), float("nan"), device="cuda")
    s = torch.full((2 * 64,), float("nan"), device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    good = dict(idx=inp.idx.data_ptr(), B=2, n_in=2, t=5, wte=inp.wte_ptrs.data_ptr(), wpe=inp.wpe.data_ptr(), W=inp.W.data_ptr(),
                spk=inp.spk.data_ptr(), SD=33, E=64, sp=s.data_ptr(), x=x.data_ptr())
    call = lambda a: lib.mvb_s2_embed_test(a["idx"], a["B"], a["n_in"], a["t"], a["wte"], a["wpe"], a["W"], a["spk"], a["SD"],  # noqa: E731
                                           a["E"], a["sp"], a["x"], st)
    for key, bad in (("idx", None), ("wte", None), ("wpe", None), ("x", None), ("W", None), ("sp", None), ("B", 0), ("t", 0),
                     ("E", 0), ("SD", 0), ("n_in", 0), ("n_in", 9), ("B", -1)):
        assert call({**good, key: bad}) == L.MVB_ERR_ARG, (key, bad)
        assert b"mvb_s2_embed_test" in lib.mvb_last_error()
    torch.cuda.synchronize()
    assert torch.isnan(x).all() and torch.isnan(s).all()
    # without a speaker, W_spk and spk_proj are not read and may be NULL
    assert call({**good, "spk": None, "W": None, "sp": None}) == L.MVB_OK
    assert not torch.isnan(x).any()
