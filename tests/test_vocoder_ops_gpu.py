"""GPU: the EnCodec decoder kernels of csrc/vocoder.cu one at a time (hook `mvb_voc_op_test`: each kernel launched with
a single segment, the kernels single and batched decodes both run; `k_rvq_decode` through `mvb_voc_decode_latent`) against
float64 references of the same operations on the kernels' own fp32 inputs.  u = 2^-23.

k_rvq_decode   latent[c][t] = sum_q book_q[code[q][t]][c], summed in fp32 in codebook order: bit-identical to that sum.
k_conv1d<K>    causal conv, reflect left padding x[-j] = x[j], optional ELU on every input sample (halo included), bias,
               optional accumulation into y.  One fmaf per product (Cin K of them), then + bias and + y_prev:
                 |err| <= (Cin K + 2) u conv(|e|, |W|) + conv(|de|, |W|) + 2u (|b| + |y_prev|),
               de = u |e| on the ELU branch (expm1f: 1 ulp).
k_convtr1d     ELU, ConvTranspose1d(k = 2r, stride r), trimmed by r on the right; 2 Cin fmaf + the bias:
                 |err| <= (2 Cin + 1) u (convtr(|e|, |W|) + |b|) + convtr(|de|, |W|).
k_lstm_layer   gate order i, f, g, o, zero initial state.  Teacher-forced: every step of the float64 reference starts
               from the kernel's own h_{t-1}.  Pre-activation a: H/8 fmaf per lane, 3 shuffle adds, + pre:
                 |da| <= (H/8 + 4) u (sum |w||h| + |pre|).
               sigma = 1 / (1 + expf(-a)) (expf 2 ulp, one add, one division): |dsigma| <= |da| / 4 + 5u sigma;
               tanhf (2 ulp): |dtanh| <= |da| + 2u |tanh|.  Cell: local error
                 eps_t = |df| |c| + |di| |g| + i |dg| + 2u (|f c| + |i g|)   (one fmaf and one product),
               drift D_t = (f_t + |df_t|) D_{t-1} + eps_t (the forget gate damps it, f < 1), and
                 |dh_t| <= |do| |tanh c| + o (D_t + 2u |tanh c|) + u |h|.
               A free-running float64 LSTM is compared normwise at weights scaled so the recurrence contracts.
Each output buffer has NaN guards on both sides (the kernel writes all of [Cout, Tout] and nothing else), and every
check also asserts ||err||_F / ||ref||_F < 1e-4.  The whole decode is compared normwise with the oracle port run in
float64.  Sensitivity: zero padding instead of reflect, no ELU on the reflected halo, the convtr reference without the e[t-1] tap
at the first output of each 32-frame tile, f and g swapped, the LSTM skip dropped -- each must break its bound."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
NORMWISE = 1e-4
GUARD = 1024
DEV = "cuda"
RATIOS = (8, 5, 4, 2)


def _lib():
    from mvb200 import _lib as L
    return L, L.load()


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _guarded(n, init=None):
    buf = torch.full((2 * GUARD + n,), float("nan"), device=DEV)
    if init is not None:
        buf[GUARD:GUARD + n] = init.reshape(-1)
    return buf, buf[GUARD:GUARD + n]


def _check_guards(buf, n):
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + n:]).all(), "write outside the output"
    assert not torch.isnan(buf[GUARD:GUARD + n]).any(), "output not fully written"


def _op(op, x, Cin, T, w, b, Cout, k, elu=0, acc=0, skip=None, y0=None, Tout=None):
    L, lib = _lib()
    n = Cout * (Tout or T)
    buf, y = _guarded(n, y0)
    ptr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    L.check(lib.mvb_voc_op_test(op, x.data_ptr(), Cin, T, w.data_ptr(), ptr(b), Cout, k, elu, acc, ptr(skip), y.data_ptr(), _st()))
    _check_guards(buf, n)
    return y.view(Cout, Tout or T).double()


def _elu(x):
    """float64 ELU of fp32 x and the expm1f error bound of the kernel's fp32 ELU (1 ulp on the negative branch)."""
    xd = x.double()
    e = torch.where(xd > 0, xd, torch.expm1(xd))
    return e, torch.where(xd > 0, torch.zeros_like(xd), U * e.abs())


def _report(label, got, ref, bound):
    err = (got - ref).abs()
    ratio, nw = float((err / bound).max()), float(err.norm() / ref.norm().clamp_min(1e-300))
    print(f"{label}: max |err|/bound {ratio:.2e}, normwise {nw:.2e}")
    bad = (err > bound).nonzero()
    assert bad.numel() == 0, f"{label}: {bad.shape[0]} elements over the bound, first at {bad[0].tolist()}"
    assert nw < NORMWISE, f"{label}: normwise {nw:.2e}"
    return ratio


def _over(got, ref, bound):
    return int(((got - ref).abs() > bound).sum())


# ---- k_rvq_decode -------------------------------------------------------------------------------------------------------
def _voc_engine(n_q, dim, max_frames, seed=0):
    """An EncodecDecodeEngine-shaped handle whose codebooks the test chooses (the decoder weights are zeros)."""
    from mvb200 import _lib as L
    lib = L.load()
    g = torch.Generator().manual_seed(seed)
    books = [torch.randn(1024, dim, generator=g) * 0.7 for _ in range(n_q)]
    top, shapes = 512, []
    shapes += [(top, dim, 7), (top,)]
    shapes += [(4 * top, top), (4 * top, top), (4 * top,)] * 2
    ch = top
    for r in RATIOS:
        shapes += [(ch, ch // 2, 2 * r), (ch // 2,), (ch // 4, ch // 2, 3), (ch // 4,), (ch // 2, ch // 4, 1), (ch // 2,),
                   (ch // 2, ch // 2, 1), (ch // 2,)]
        ch //= 2
    shapes += [(1, ch, 7), (1,)]
    tensors = books + [torch.zeros(s) for s in shapes]
    offs, total = [], 0
    for t in tensors:
        offs.append(total)
        total = (total + t.numel() * 4 + 255) // 256 * 256
    arena = torch.zeros(total // 4)
    for t, o in zip(tensors, offs):
        arena[o // 4:o // 4 + t.numel()] = t.reshape(-1)
    arena = arena.to(DEV)
    cfg = L.VocConfig()
    cfg.n_q, cfg.hidden, cfg.n_filters, cfg.n_ratios = n_q, dim, 32, len(RATIOS)
    for k, r in enumerate(RATIOS):
        cfg.ratios[k] = r
    cfg.kernel, cfg.res_kernel, cfg.last_kernel, cfg.compress, cfg.max_frames = 7, 3, 7, 2, max_frames
    ws = torch.zeros(lib.mvb_voc_workspace_bytes(C.byref(cfg)), dtype=torch.uint8, device=DEV)
    h = C.c_void_p()
    L.check(lib.mvb_voc_create(C.byref(cfg), arena.data_ptr(), arena.numel() * 4, (C.c_uint64 * len(offs))(*offs), ws.data_ptr(),
                               C.byref(h)))
    return h, books, (arena, ws)


@pytest.mark.parametrize("n_q", [1, 8, 32])
@pytest.mark.parametrize("dim", [128, 100])
def test_rvq_decode_bit_identical(n_q, dim):
    L, lib = _lib()
    h, books, keep = _voc_engine(n_q, dim, 2048, seed=n_q * dim)
    try:
        for T in (1, 31, 32, 33, 2048):
            g = torch.Generator().manual_seed(T)
            codes = torch.randint(0, 1024, (n_q, T), generator=g, dtype=torch.int32)
            codes[:, 0] = 0
            codes[:, -1] = 1023
            buf, lat = _guarded(dim * T)
            cd = codes.to(DEV)
            L.check(lib.mvb_voc_decode_latent(h, cd.data_ptr(), T, lat.data_ptr(), _st()))
            torch.cuda.synchronize()
            _check_guards(buf, dim * T)
            want = torch.zeros(T, dim)
            for q in range(n_q):           # fp32, codebook order
                want = want + books[q][codes[q].long()]
            assert torch.equal(lat.view(dim, T).cpu(), want.t()), f"n_q={n_q} dim={dim} T={T}"
    finally:
        lib.mvb_voc_destroy(h)


# ---- k_conv1d<K> --------------------------------------------------------------------------------------------------------
def conv_ref(x, w, b, K, elu, y0=None, pad="reflect", halo_elu=True):
    """(ref, bound) of k_conv1d<K> in float64."""
    e, de = _elu(x) if elu else (x.double(), torch.zeros_like(x, dtype=torch.float64))
    if elu and not halo_elu:
        raw = x.double()
    wd = w.double()

    def padded(v, raw_halo=None):
        if K == 1:
            return v
        p = F.pad(v[None], (K - 1, 0), mode=pad)[0] if pad == "reflect" else F.pad(v, (K - 1, 0))
        if raw_halo is not None:
            p[:, :K - 1] = F.pad(raw_halo[None], (K - 1, 0), mode="reflect")[0][:, :K - 1]
        return p

    ep = padded(e, raw if elu and not halo_elu else None)
    ref = F.conv1d(ep[None], wd)[0]
    A = F.conv1d(padded(e.abs())[None], wd.abs())[0]
    dA = F.conv1d(padded(de)[None], wd.abs())[0]
    extra = torch.zeros_like(ref)
    if b is not None:
        ref = ref + b.double()[:, None]
        extra = extra + b.double().abs()[:, None]
    if y0 is not None:
        ref = ref + y0.double()
        extra = extra + y0.double().abs()
    bound = (w.shape[1] * K + 2) * U * A + dA + 2 * U * extra + 1e-300
    return ref, bound


def _conv_case(label, Cin, Cout, K, T, elu, acc, bias=True, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(Cin, T, generator=g, device=DEV) * 0.8
    w = torch.randn(Cout, Cin, K, generator=g, device=DEV) / (Cin * K) ** 0.5
    b = 0.1 * torch.randn(Cout, generator=g, device=DEV) if bias else None
    y0 = torch.randn(Cout, T, generator=g, device=DEV) if acc else None
    got = _op(0, x, Cin, T, w, b, Cout, K, elu, acc, y0=y0)
    ref, bound = conv_ref(x, w, b, K, elu, y0)
    return _report(f"k_conv1d<{K}> {label} {Cin}->{Cout} T={T} elu={elu} acc={acc}", got, ref, bound), (x, w, b, got)


def _production_convs(T):
    """(label, Cin, Cout, K, T, elu, acc) of every k_conv1d launch of mvb_voc_decode at T frames."""
    out = [("conv_in", 128, 512, 7, T, 0, 0), ("lstm pre", 512, 2048, 1, T, 0, 0)]
    ch, Tl = 512, T
    for r in RATIOS:
        ch, Tl = ch // 2, Tl * r
        out += [(f"r{r} res conv3", ch, ch // 2, 3, Tl, 1, 0), (f"r{r} res conv1", ch // 2, ch, 1, Tl, 1, 1),
                (f"r{r} shortcut", ch, ch, 1, Tl, 0, 0)]
    out.append(("conv_out", 32, 1, 7, Tl, 1, 0))
    return out


@pytest.mark.parametrize("T", [8, 375, 2048])
def test_conv1d_production_layers(T):
    for i, (label, cin, cout, K, t, elu, acc) in enumerate(_production_convs(T)):
        _conv_case(label, cin, cout, K, t, elu, acc, seed=100 * T + i)


@pytest.mark.parametrize("K", [1, 3, 7])
def test_conv1d_tile_seams_load_paths_and_ragged_channels(K):
    """T = 255 / 256 / 257 / 259 / 260 around the 256-sample tile (T % 4 == 0: 128-bit path, else scalar), partial
    16-channel passes (Cin 17 / 33) and partial 32-channel output tiles (Cout 1 / 31 / 33), no bias."""
    for T in (255, 256, 257, 259, 260):
        _conv_case("seam", 33, 33, K, T, 1, 1, seed=T * K)
    for cin, cout in ((17, 1), (33, 31), (17, 33)):
        _conv_case("ragged", cin, cout, K, 259, 1, 0, bias=False, seed=cin * cout + K)
        _conv_case("ragged", cin, cout, K, 260, 0, 1, seed=cin * cout + K + 1)


def test_conv1d_padding_and_halo_elu_sensitivity():
    """Zero padding instead of reflect, and reflect padding without the ELU on the halo samples, must break the bound
    (the first K - 1 outputs of every channel differ)."""
    for T in (259, 260):          # scalar and 128-bit load paths
        _, (x, w, b, got) = _conv_case("sensitivity", 32, 32, 7, T, 1, 0, seed=7 + T)
        _, bound = conv_ref(x, w, b, 7, 1)
        zero, _ = conv_ref(x, w, b, 7, 1, pad="constant")
        no_halo_elu, _ = conv_ref(x, w, b, 7, 1, halo_elu=False)
        n1, n2 = _over(got, zero, bound), _over(got, no_halo_elu, bound)
        print(f"T={T}: zero padding {n1}, halo without ELU {n2} elements over the bound")
        assert n1 > 0 and n2 > 0


# ---- k_convtr1d ---------------------------------------------------------------------------------------------------------
def convtr_ref(x, w, b, r, drop_seam_tap=False):
    e, de = _elu(x)
    wd = w.double()
    T = x.shape[1]
    ct = lambda v, ww: F.conv_transpose1d(v[None], ww, stride=r)[0][:, :T * r]   # noqa: E731
    ref = ct(e, wd) + b.double()[:, None]
    bound = (2 * x.shape[0] + 1) * U * (ct(e.abs(), wd.abs()) + b.double().abs()[:, None]) + ct(de, wd.abs()) + 1e-300
    if drop_seam_tap:             # e[t-1] of the first output frame t of every 32-frame tile (t = 32, 64, ...)
        sel = torch.zeros_like(e)
        sel[:, 31:T - 1:32] = e[:, 31:T - 1:32]
        w2 = wd.clone()
        w2[:, :, :r] = 0
        ref = ref - ct(sel, w2)
    return ref, bound


def _convtr_case(label, Cin, Cout, r, T, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(Cin, T, generator=g, device=DEV) * 0.8
    w = torch.randn(Cin, Cout, 2 * r, generator=g, device=DEV) / (2 * Cin) ** 0.5
    b = 0.1 * torch.randn(Cout, generator=g, device=DEV)
    got = _op(1, x, Cin, T, w, b, Cout, r, Tout=T * r)
    assert got.shape == (Cout, T * r)
    ref, bound = convtr_ref(x, w, b, r)
    _report(f"k_convtr1d {label} {Cin}->{Cout} r={r} T={T}", got, ref, bound)
    return x, w, b, got


@pytest.mark.parametrize("stage", range(4))
def test_convtr1d_production(stage):
    cin, r = 512 >> stage, RATIOS[stage]
    up = 1
    for q in RATIOS[:stage]:
        up *= q
    for T in (1, 31, 32, 33, 375, 2048 * up):
        _convtr_case("production", cin, cin // 2, r, T, seed=stage * 10000 + T)


@pytest.mark.parametrize("r", [1, 3, 6, 7])
def test_convtr1d_other_ratios(r):
    for T in (1, 31, 32, 33, 375):
        _convtr_case("ratio", 48, 33, r, T, seed=r * 1000 + T)


def test_convtr1d_seam_tap_sensitivity():
    x, w, b, got = _convtr_case("sensitivity", 64, 32, 4, 200, seed=3)
    _, bound = convtr_ref(x, w, b, 4)
    bad, _ = convtr_ref(x, w, b, 4, drop_seam_tap=True)
    n = _over(got, bad, bound)
    print(f"convtr without the e[t-1] tap at tile seams: {n} elements over the bound")
    assert n > 0


# ---- k_lstm_layer -------------------------------------------------------------------------------------------------------
def _lstm_run(H, T, seed, scale, skip=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    pre = torch.randn(4 * H, T, generator=g, device=DEV) * 1.5
    whh = torch.randn(4 * H, H, generator=g, device=DEV) * (scale / H ** 0.5)
    sk = torch.randn(H, T, generator=g, device=DEV) if skip else None
    out = _op(2, pre, H, T, whh, None, H, 0, skip=sk)
    return pre, whh, sk, out


def lstm_teacher_forced(pre, whh, h_kernel, swap_fg=False):
    """float64 steps driven by the kernel's own h_{t-1} -> (h_ref, bound), both [H, T]."""
    H, T = whh.shape[1], pre.shape[1]
    P, Wd = pre.double(), whh.double()
    hk = h_kernel.double()
    c = torch.zeros(H, dtype=torch.float64, device=DEV)
    D = torch.zeros_like(c)
    hs, bs = [], []
    sig = torch.sigmoid
    for t in range(T):
        hp = hk[:, t - 1] if t else torch.zeros_like(c)
        a = P[:, t] + Wd @ hp
        da = (H / 8 + 4) * U * (Wd.abs() @ hp.abs() + P[:, t].abs())
        ai, af, ag, ao = a.split(H)
        if swap_fg:
            af, ag = ag, af
        di, df, dg, do = da.split(H)
        i, f, gg, o = sig(ai), sig(af), torch.tanh(ag), sig(ao)
        di, df, do = di / 4 + 5 * U * i, df / 4 + 5 * U * f, do / 4 + 5 * U * o
        dg = dg + 2 * U * gg.abs()
        eps = df * c.abs() + di * gg.abs() + i * dg + 2 * U * ((f * c).abs() + (i * gg).abs())
        c = f * c + i * gg
        D = (f + df) * D + eps
        tc = torch.tanh(c)
        h = o * tc
        hs.append(h)
        bs.append(do * tc.abs() + o * (D + 2 * U * tc.abs()) + U * h.abs() + 1e-300)
    return torch.stack(hs, 1), torch.stack(bs, 1)


def lstm_free(pre, whh):
    H, T = whh.shape[1], pre.shape[1]
    P, Wd = pre.double(), whh.double()
    h = torch.zeros(H, dtype=torch.float64, device=DEV)
    c = torch.zeros_like(h)
    hs = []
    for t in range(T):
        ai, af, ag, ao = (P[:, t] + Wd @ h).split(H)
        c = torch.sigmoid(af) * c + torch.sigmoid(ai) * torch.tanh(ag)
        h = torch.sigmoid(ao) * torch.tanh(c)
        hs.append(h)
    return torch.stack(hs, 1)


@pytest.mark.parametrize("H", [32, 128, 512])
def test_lstm_teacher_forced_and_free_running(H):
    for T in (1, 2, 8, 375, 2048):
        pre, whh, _, got = _lstm_run(H, T, seed=H * 7 + T, scale=1.0)
        ref, bound = lstm_teacher_forced(pre, whh, got)
        _report(f"k_lstm_layer H={H} T={T} teacher-forced", got, ref, bound)
        pre, whh, _, got = _lstm_run(H, T, seed=H * 7 + T + 1, scale=0.5)
        free = lstm_free(pre, whh)
        nw = float((got - free).norm() / free.norm())
        print(f"k_lstm_layer H={H} T={T} free-running (contracting W_hh): normwise {nw:.2e}")
        assert nw < NORMWISE


def test_lstm_skip_and_sensitivity():
    """The skip is added to the stored output (fp32 add of the same h); a reference without it, and one with the f and
    g gates swapped, must break the bound."""
    H, T = 128, 375
    pre, whh, sk, got_skip = _lstm_run(H, T, seed=5, scale=1.0, skip=True)
    got = _op(2, pre, H, T, whh, None, H, 0)
    assert torch.equal(got_skip.float(), got.float() + sk), "skip is not fl(h + skip) of the same h"
    ref, bound = lstm_teacher_forced(pre, whh, got)
    n_skip = _over(got_skip, ref, bound)
    swapped, _ = lstm_teacher_forced(pre, whh, got, swap_fg=True)
    n_swap = _over(got, swapped, bound)
    print(f"LSTM without the skip: {n_skip}, f/g swapped: {n_swap} elements over the bound")
    assert n_skip > 0 and n_swap > 0


# ---- whole decode ---------------------------------------------------------------------------------------------------------
def _oracle_f64(sd):
    from oracle import vocoder_port as V
    o = V.EncodecDecodeOracle(sd)
    d = lambda t: t.to(DEV, torch.float64)    # noqa: E731
    o.codebooks = [d(t) for t in o.codebooks]
    o.conv_in = tuple(d(t) for t in o.conv_in)
    o.lstm = [{k: d(v) for k, v in L.items()} for L in o.lstm]
    o.ups = [tuple(d(t) for t in p) for p in o.ups]
    o.res = [{k: tuple(d(t) for t in p) for k, p in blk.items()} for blk in o.res]
    o.conv_out = tuple(d(t) for t in o.conv_out)
    return o


def test_whole_decode_vs_float64_oracle():
    from mvb200 import synth
    from mvb200.vocoder import EncodecDecodeEngine
    _, sd = synth.encodec_model_and_state_dict(seed=0)
    eng = EncodecDecodeEngine(sd, device=DEV, max_frames=2048)
    o = _oracle_f64(sd)
    prev = torch.get_default_dtype()
    for T in (8, 375, 2048):
        codes = torch.randint(0, 1024, (8, T), generator=torch.Generator().manual_seed(T))
        wav = eng.decode(codes).double()
        torch.set_default_dtype(torch.float64)
        try:
            with torch.device(DEV):
                ref = o.decode(codes[None].to(DEV))[0, 0]
        finally:
            torch.set_default_dtype(prev)
        nw = float((wav - ref).norm() / ref.norm())
        print(f"mvb_voc_decode T={T}: normwise {nw:.2e} vs the float64 oracle")
        assert wav.shape == ref.shape == (T * 320,) and nw < NORMWISE
