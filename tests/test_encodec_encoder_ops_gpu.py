"""GPU: the EnCodec encoder kernels one at a time (hook `mvb_enc_op_test`, the launch helpers `mvb_enc_encode` uses)
against float64 references on the kernels' own fp32 inputs.  u = 2^-23 (a conservative unit roundoff).

k_conv1d_down<S>  ELU, then EncodecConv1d(k = 2S, stride S) over the V valid input samples: reflect padding of S on the
                  left and ceil(V / S) S - V on the right, with _pad1d's zero extension when V <= S (the float64
                  reference is the oracle's literal restatement, test_encodec_encoder_cpu.pad1d_reflect).  One fmaf chain
                  of Cin 2S products from 0, then + bias:
                    |err| <= (Cin 2S + 2) u (conv(|e|, |W|) + |b|) + conv(|de|, |W|),   de = u |e| on the ELU branch.
k_conv1d<K>       the same with stride 1, valid length V < block length T (the zero extension for V <= K - 1), the bound
                  of test_vocoder_ops_gpu.py.
                  Inputs past V are NaN and the output buffer is NaN-filled with NaN guards: exactly the ceil(V / S) (or V)
                  valid columns of every row must be written, finite, and nothing else.
k_rvq_encode      per codebook, score s_j = |e_j|^2 - 2 r.e_j: |e_j|^2 rounded once from a double sum (u |e|^2), the
                  dot product one fmaf chain of dim products (dim u sum |r||e_j|), doubled exactly and subtracted (u |s|):
                    |ds_j| <= u |e_j|^2 + 2 dim u sum_d |r_d e_jd| + u |s_j|.
                  The kernel must return the float64 argmin of s over the residual it holds (lowest index on exact ties)
                  unless the float64 gap to its choice is within ds_best + ds_choice; such frames are counted.  The
                  residual after the last codebook is bit-identical to the fp32 chain r -= e_idx over the chosen rows.
                  Codebooks: the synthetic checkpoint's N(0, 1) rows (|e| ~ 11, where |e|^2 alone nearly decides), rows at
                  the embeddings' scale, exact duplicate rows, and rows one ulp apart.
Sensitivity: zero instead of reflect right padding, no zero extension (numpy's repeated reflection instead), the highest
index on ties and a residual that is never updated must each break their bound or differ."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_encodec_encoder_cpu import pad1d_reflect

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
NORMWISE = 1e-4
GUARD = 1024
DEV = "cuda"


def _lib():
    from mvb200 import _lib as L
    return L, L.load()


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _elu(x):
    xd = x.double()
    e = torch.where(xd > 0, xd, torch.expm1(xd))
    return e, torch.where(xd > 0, torch.zeros_like(xd), U * e.abs())


def _op(op, x, Cin, T, V, w, b, Cout, k, elu, To, Vo):
    """One hook call on a NaN-filled guarded output [Cout, To]; checks that exactly the first Vo columns are written."""
    L, lib = _lib()
    buf = torch.full((2 * GUARD + Cout * To,), float("nan"), device=DEV)
    y = buf[GUARD:GUARD + Cout * To]
    L.check(lib.mvb_enc_op_test(op, x.data_ptr(), Cin, T, V, w.data_ptr(), None if b is None else b.data_ptr(), Cout, k, elu,
                                y.data_ptr(), None, _st()))
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + Cout * To:]).all(), "write outside the output"
    yv = y.view(Cout, To)
    assert not torch.isnan(yv[:, :Vo]).any(), "a valid output is missing or reads a sample past V"
    assert torch.isnan(yv[:, Vo:]).all(), "an output past the valid length was written"
    return yv[:, :Vo].double()


def _input(Cin, T, V, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(Cin, T, generator=g, device=DEV) * 0.8
    x[:, V:] = float("nan")              # the block tail past the valid length must never reach an output
    return x, g


def conv_ref(x, V, w, b, stride, mode="reflect", elu=True):
    """float64 (ref, bound) of (ELU +) EncodecConv1d over the first V samples.  mode: 'reflect' (the reference),
    'zero_right' (zero instead of reflect right padding), 'no_zero_ext' (numpy's repeated reflection)."""
    e, de = _elu(x[:, :V]) if elu else (x[:, :V].double(), torch.zeros_like(x[:, :V], dtype=torch.float64))
    K = w.shape[-1]
    left, right = K - stride, -(-V // stride) * stride - V

    def pad(v):
        if mode == "reflect":
            return pad1d_reflect(v[None], left, right)[0]
        if mode == "zero_right":
            return F.pad(pad1d_reflect(v[None], left, 0)[0], (0, right))
        return torch.from_numpy(np.pad(v.cpu().numpy(), ((0, 0), (left, right)), mode="reflect")).to(v.device)

    wd = w.double()
    ref = F.conv1d(pad(e)[None], wd, stride=stride)[0]
    A = F.conv1d(pad1d_reflect(e.abs()[None], left, right), wd.abs(), stride=stride)[0]
    dA = F.conv1d(pad1d_reflect(de[None], left, right), wd.abs(), stride=stride)[0]
    extra = torch.zeros_like(ref)
    if b is not None:
        ref = ref + b.double()[:, None]
        extra = extra + b.double().abs()[:, None]
    bound = (w.shape[1] * K + 2) * U * (A + extra) + dA + 1e-300
    return ref, bound


def _report(label, got, ref, bound):
    err = (got - ref).abs()
    nw = float(err.norm() / ref.norm().clamp_min(1e-300))
    print(f"{label}: max |err|/bound {float((err / bound).max()):.2e}, normwise {nw:.2e}")
    bad = (err > bound).nonzero()
    assert bad.numel() == 0, f"{label}: {bad.shape[0]} elements over the bound, first at {bad[0].tolist()}"
    assert nw < NORMWISE, f"{label}: normwise {nw:.2e}"


def _over(got, ref, bound):
    return int(((got - ref).abs() > bound).sum())


# ---- k_conv1d_down<S> ----------------------------------------------------------------------------------------------------
STAGES = ((2, 32, 64, 320), (4, 64, 128, 160), (5, 128, 256, 40), (8, 256, 512, 8))   # (S, Cin, Cout, samples per frame)


def _down_case(S, Cin, Cout, T, V, seed, mode="reflect"):
    x, g = _input(Cin, T, V, seed)
    w = torch.randn(Cout, Cin, 2 * S, generator=g, device=DEV) / (Cin * 2 * S) ** 0.5
    b = 0.1 * torch.randn(Cout, generator=g, device=DEV)
    Vo = -(-V // S)
    got = _op(0, x, Cin, T, V, w, b, Cout, S, 1, T // S, Vo)
    ref, bound = conv_ref(x, V, w, b, S)
    _report(f"k_conv1d_down<{S}> {Cin}->{Cout} T={T} V={V}", got, ref, bound)
    return x, w, b, got


@pytest.mark.parametrize("stage", range(4))
def test_conv_down_short_ragged_and_production(stage):
    S, Cin, Cout, m = STAGES[stage]
    for V in range(1, 3 * S + 2):                         # every valid length up to 3S + 1, zero extension included
        _down_case(S, Cin, Cout, 8 * S, V, seed=stage * 1000 + V)
    for V in (256 * S - 1, 256 * S, 256 * S + 1, 512 * S - 3, 512 * S + S - 1):   # around the 256-output tile seams
        T = -(-(V + 5) // (4 * S)) * 4 * S
        _down_case(S, Cin, Cout, T, V, seed=stage * 1000 + V)
    F30 = 2250                                           # 30 s: 2250 frames, at this stage's input rate
    _down_case(S, Cin, Cout, F30 * m, F30 * m - m // 2, seed=stage)


def test_conv_down_scalar_path_and_ragged_channels():
    """T % 4 != 0 (scalar loads) and channel counts that are not multiples of the pass / tile widths."""
    for S in (2, 4, 5, 8):
        _down_case(S, 17, 33, 75 * S, 75 * S - 2, seed=S)
        _down_case(S, 3, 1, 13 * S, 13 * S, seed=S + 1)


def test_conv_down_padding_sensitivity():
    for S in (4, 5):
        x, w, b, got = _down_case(S, 32, 32, 64 * S, 63 * S + 1, seed=11 * S)     # right padding of S - 1 samples
        V = 63 * S + 1
        _, bound = conv_ref(x, V, w, b, S)
        zr, _ = conv_ref(x, V, w, b, S, mode="zero_right")
        n = _over(got, zr, bound)
        print(f"S={S}: zero right padding: {n} elements over the bound")
        assert n > 0
        x, w, b, got = _down_case(S, 32, 32, 8 * S, 2, seed=13 * S)               # V = 2 <= S: zero extension
        _, bound = conv_ref(x, 2, w, b, S)
        nz, _ = conv_ref(x, 2, w, b, S, mode="no_zero_ext")
        n = _over(got, nz, bound)
        print(f"S={S}: no zero extension: {n} elements over the bound")
        assert n > 0


# ---- k_conv1d<K> with a valid length below the block length -------------------------------------------------------------
def _conv_case(K, Cin, Cout, T, V, elu, seed, bias=True):
    x, g = _input(Cin, T, V, seed)
    w = torch.randn(Cout, Cin, K, generator=g, device=DEV) / (Cin * K) ** 0.5
    b = 0.1 * torch.randn(Cout, generator=g, device=DEV) if bias else None
    got = _op(1, x, Cin, T, V, w, b, Cout, K, elu, T, V)
    ref, bound = conv_ref(x, V, w, b, 1, elu=bool(elu))
    _report(f"k_conv1d<{K}> {Cin}->{Cout} T={T} V={V} elu={elu}", got, ref, bound)
    return x, w, b, got


@pytest.mark.parametrize("K", [1, 3, 7])
def test_conv1d_valid_length_below_block(K):
    for V in range(1, 10):                      # V <= K - 1: zero extension; then reflection about V - 1
        _conv_case(K, 33, 33, 16, V, 1, seed=K * 100 + V)
    for T, V in ((512, 257), (520, 509), (1024, 767), (2250, 2250 - 3)):
        _conv_case(K, 33, 31, T, V, V % 2, seed=K * 100 + T)
    _conv_case(K, 512, 128, 16, 5, 1, seed=K)   # the final conv of a clip of 5 frames


def test_conv1d_zero_extension_sensitivity():
    x, w, b, got = _conv_case(7, 32, 32, 16, 3, 1, seed=5)
    _, bound = conv_ref(x, 3, w, b, 1)
    nz, _ = conv_ref(x, 3, w, b, 1, mode="no_zero_ext")
    n = _over(got, nz, bound)
    print(f"k7, V=3: no zero extension: {n} elements over the bound")
    assert n > 0


# ---- k_rvq_encode ----------------------------------------------------------------------------------------------------------
def _rvq(x, books):
    """Kernel codes [n_q, T] and final residual [dim, T] from the hook."""
    L, lib = _lib()
    n_q, _, dim = books.shape
    T = x.shape[1]
    codes = torch.full((n_q, T), -1, dtype=torch.int32, device=DEV)
    res = torch.full((dim, T), float("nan"), device=DEV)
    L.check(lib.mvb_enc_op_test(2, x.data_ptr(), dim, T, T, books.data_ptr(), None, 0, n_q, 0, res.data_ptr(), codes.data_ptr(),
                                _st()))
    return codes, res


def rvq_check(x, books, codes, res, label):
    """Verifies the kernel's choices codebook by codebook on the fp32 residual chain it must hold; returns the number of
    (frame, codebook) choices inside the rounding band and the chain's final residual."""
    n_q, n_bins, dim = books.shape
    r = x.t().contiguous()                                  # fp32 [T, dim]
    in_band = 0
    for q in range(n_q):
        E = books[q]
        Ed, rd = E.double(), r.double()
        nrm = (Ed * Ed).sum(1)
        s = nrm[None] - 2 * rd @ Ed.t()                      # [T, bins]
        ds = U * nrm[None] + 2 * dim * U * (rd.abs() @ Ed.abs().t()) + U * s.abs()
        c = codes[q].long()
        best = torch.argmin(s, dim=1)                       # first minimal index
        ar = torch.arange(s.shape[0], device=DEV)
        gap = s[ar, c] - s[ar, best]
        band = ds[ar, c] + ds[ar, best]
        assert ((c >= 0) & (c < n_bins)).all()
        wrong = (c != best) & (gap > band)
        assert not wrong.any(), f"{label} q={q}: {int(wrong.sum())} choices outside the band"
        in_band += int((c != best).sum())
        r = r - E[c]                                        # fp32 subtraction of the chosen rows
    assert torch.equal(res.t(), r), f"{label}: final residual is not the fp32 chain over the chosen rows"
    print(f"{label}: {in_band} choices inside the rounding band")
    return in_band


def _books(kind, n_q, dim, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    if kind == "synthetic":                                 # the checkpoint's N(0, 1) rows
        return torch.randn(n_q, 1024, dim, generator=g, device=DEV)
    b = 0.03 * torch.randn(n_q, 1024, dim, generator=g, device=DEV)   # the embeddings' scale
    if kind == "duplicates":                                # rows 2j + 1 copy rows 2j; also copies far apart
        b[:, 1::2] = b[:, 0::2]
        b[:, 1000:1024] = b[:, 3:27]
    elif kind == "ulps":                                    # rows 2j + 1 differ from 2j by one ulp in one element
        b[:, 1::2] = b[:, 0::2]
        b[:, 1::2, 5] = torch.nextafter(b[:, 0::2, 5], torch.full_like(b[:, 0::2, 5], 1.0))
    return b.contiguous()


@pytest.mark.parametrize("kind", ["synthetic", "scaled", "duplicates", "ulps"])
@pytest.mark.parametrize("n_q,dim,T", [(8, 128, 375), (32, 128, 33), (3, 100, 64)])
def test_rvq_encode(kind, n_q, dim, T):
    g = torch.Generator(device=DEV).manual_seed(T + n_q)
    x = 0.027 * torch.randn(dim, T, generator=g, device=DEV)
    books = _books(kind, n_q, dim, seed=n_q * 10 + dim)
    if kind in ("duplicates", "ulps"):                      # embeddings on top of codebook rows: ties are decisive
        x[:, ::3] = books[0, torch.arange(0, 1024, 7, device=DEV)[: x[:, ::3].shape[1]]].t()
    codes, res = _rvq(x, books)
    rvq_check(x, books, codes, res, f"k_rvq_encode {kind} n_q={n_q} dim={dim} T={T}")
    if kind == "duplicates":
        # exact duplicates score identically in fp32: the lower copy must win every time
        c = codes.long()
        assert not ((c % 2 == 1) & (c < 1000)).any(), "the higher copy of a duplicate row was chosen"
        assert not (c >= 1000).any(), "a far copy (rows 1000..1023 duplicate rows 3..26) was chosen"


def test_rvq_encode_sensitivity():
    """The highest index on ties, and a residual never updated, must differ from the kernel."""
    n_q, dim, T = 4, 128, 96
    g = torch.Generator(device=DEV).manual_seed(9)
    books = _books("duplicates", n_q, dim, seed=9)
    x = 0.027 * torch.randn(dim, T, generator=g, device=DEV)
    x[:, ::2] = books[0, torch.arange(0, 96, 2, device=DEV)].t()
    codes, res = _rvq(x, books)
    rvq_check(x, books, codes, res, "sensitivity")
    r = x.t().double()
    highest, stale = [], []
    for q in range(n_q):
        s = (books[q].double() ** 2).sum(1)[None] - 2 * r @ books[q].double().t()
        highest.append(s.shape[1] - 1 - torch.argmin(s.flip(1), dim=1))
        s0 = (books[q].double() ** 2).sum(1)[None] - 2 * x.t().double() @ books[q].double().t()
        stale.append(torch.argmin(s0, dim=1))
        r = r - books[q].double()[torch.argmin(s, dim=1)]
    highest, stale = torch.stack(highest), torch.stack(stale)
    n_hi, n_st = int((highest != codes.long()).sum()), int((stale != codes.long()).sum())
    print(f"highest index on ties: {n_hi} codes differ; residual not updated: {n_st} codes differ")
    assert n_hi > 0 and n_st > 0
